"""Cost of perturbed-attention guidance (PAG, `pag_scale`) with synthetic weights.  Prints a table and one JSON line.

    python tools/bench_pag.py [--batch 16] [--repeat 3] [--pag 1.5]

- ms per step with and without PAG: CUDA events around whole 50-step DPM-Solver++ `sample()` calls (production path, update
  fused into the output head), alternated, best of `repeat` rounds after a warm-up round.
    config 2 (rgbd_imagenet_adm_128_large_cfg, guidance 0.5): 2N rows against 3N rows;
    the single-category small network (rgbd_singlecategory_adm_128_small, GaussianDiffusion, no classes): N against 2N.
- whole DPM-Solver++ 25-step runs with and without PAG on both networks.
- the device memory the PAG plan adds (free memory before and after its first use).
- the relative L2 distance between the PAG run and the run without it from the same x_T and seed: diagnostic drift on
  random weights, not a statement about sample quality.
Needs a GPU: there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np                                # noqa: E402
import torch                                      # noqa: E402

import bench                                      # noqa: E402  (MODELS, GUIDANCE)
import ivid_b200.backbones as backbones           # noqa: E402
import ivid_b200.frameworks as frameworks         # noqa: E402
import ivid_b200.samplers as samplers             # noqa: E402
from oracle import unet_ref                       # noqa: E402


def _card():
    info = {"torch_name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["name_power_limit_max_sm_clock_current_sm_clock"] = r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["name_power_limit_max_sm_clock_current_sm_clock"] = f"unavailable: {e}"
    return info


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def _single_category_cfg():
    # the backbone args of configs/rgbd_singlecategory_adm_128_small.json, as the test fixture stores them
    golden = np.load(os.path.join(ROOT, "tests", "golden", "unet_sampler_golden_part0.npz"))
    key = "schemacfg_rgbd_singlecategory_adm_128_small"
    if key not in golden.files:
        golden = np.load(os.path.join(ROOT, "tests", "golden", "unet_sampler_golden_part1.npz"))
    return json.loads(bytes(golden[key]).decode())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--pag", type=float, default=1.5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_pag.py needs a GPU"
    card = _card()
    B, w = args.batch, args.pag

    def timed(fn):
        torch.manual_seed(0)                         # the Philox seed of the run is drawn from torch's generator
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    cases = []
    for name, cfg, fw_cls, guided in (("config2_cfg", bench.MODELS["L"], frameworks.ClassifierFreeGuidance, True),
                                      ("singlecategory_small", _single_category_cfg(), frameworks.GaussianDiffusion, False)):
        net = backbones.AdmUnet2d(**cfg)
        net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234))
        fw = fw_cls(net.cuda(), timesteps=1000, beta_schedule="linear")
        dpm = samplers.DpmSolverSampler(fw)
        S = cfg["image_size"]
        x_T = torch.randn(B, 4, S, S, generator=torch.Generator().manual_seed(1000)).cuda()
        kw = dict(noise=x_T, verbose=False)
        if guided:
            kw.update(classes=torch.arange(B, device="cuda") % 1000, strength=bench.GUIDANCE)
        # memory of the PAG plan: the plan without PAG exists after the first run, the PAG plan after the first PAG step
        timed(lambda: dpm.sample(B, steps=5, **kw))
        free0 = torch.cuda.mem_get_info()[0]
        timed(lambda: dpm.sample(B, steps=5, pag_scale=w, **kw))
        free1 = torch.cuda.mem_get_info()[0]
        best = {"off": None, "pag": None}
        for rnd in range(1 + args.repeat):
            for key, pk in (("off", {}), ("pag", dict(pag_scale=w))):
                ms, _ = timed(lambda: dpm.sample(B, steps=50, **pk, **kw))
                if rnd > 0 and (best[key] is None or ms / 50 < best[key]):
                    best[key] = ms / 50
        runs = {}
        for key, pk in (("off", {}), ("pag", dict(pag_scale=w))):
            t_best, out = None, None
            for _ in range(args.repeat):
                ms, o = timed(lambda: dpm.sample(B, steps=25, **pk, **kw).samples)
                t_best = ms if t_best is None else min(t_best, ms)
                out = o
            runs[key] = (t_best, out)
        rows = 3 if guided else 2
        cases.append({"network": name, "rows": f"{rows - 1}N vs {rows}N", "ms_per_step_off": round(best["off"], 3),
                      "ms_per_step_pag": round(best["pag"], 3), "step_ratio": round(best["pag"] / best["off"], 4),
                      "dpmpp_25_ms_off": round(runs["off"][0], 1), "dpmpp_25_ms_pag": round(runs["pag"][0], 1),
                      "pag_plan_extra_mib": round((free0 - free1) / 2 ** 20, 1),
                      "rel_l2_pag_vs_off_drift_random_weights": round(_rel(runs["pag"][1], runs["off"][1]), 4)})
        del fw, net, dpm
        torch.cuda.empty_cache()
    print(f"{'network':>22} {'rows':>10} {'off ms/step':>12} {'pag ms/step':>12} {'ratio':>7} {'25-step off':>12} {'25-step pag':>12} "
          f"{'+MiB':>8} {'rel L2':>8}")
    for c in cases:
        print(f"{c['network']:>22} {c['rows']:>10} {c['ms_per_step_off']:>12.2f} {c['ms_per_step_pag']:>12.2f} {c['step_ratio']:>7.3f} "
              f"{c['dpmpp_25_ms_off']:>12.1f} {c['dpmpp_25_ms_pag']:>12.1f} {c['pag_plan_extra_mib']:>8.1f} "
              f"{c['rel_l2_pag_vs_off_drift_random_weights']:>8.4f}")
    print(json.dumps({"bench": "pag", "batch": B, "pag_scale": w, "pag_layers": ["middle_block.1"], "guidance": bench.GUIDANCE,
                      "card": card, "cases": cases, "card_after": _card()}))


if __name__ == "__main__":
    main()

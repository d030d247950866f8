"""Cost of adaptive projected guidance (APG, `apg=(eta, r, beta)`) with synthetic weights.  Prints a table and one JSON line.

    python tools/bench_apg.py [--repeat 3] [--apg 0,4,-0.5]

- ms per step with and without APG: CUDA events around whole `sample()` calls (production path, step fused into the output
  head), alternated, best of `repeat` rounds after a warm-up round.
    config 2 network (rgbd_imagenet_adm_128_large_cfg, batch 16), 50-step DPM-Solver++ at guidance 0.5 and 3.0;
    config 5 (rgbd_imagenet_adm_256_128_small_sr super-resolution, 256x256, batch 8), 50-step DDIM at guidance 0.5.
- the device memory APG adds (free memory before and after its first run).
- the relative L2 distance between the APG run and plain classifier-free guidance from the same x_T and seed: diagnostic
  drift on random weights, not a statement about sample quality.
Needs a GPU: there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--apg", default="0,4,-0.5", help="ETA[,R[,BETA]] (default: the paper's eta = 0 and beta = -0.5, r = 4)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_apg.py needs a GPU"
    apg = tuple(float(v) for v in args.apg.split(","))
    card = _card()

    def timed(fn):
        torch.manual_seed(0)                         # the Philox seed of the run is drawn from torch's generator
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    cases = []
    gen = torch.Generator().manual_seed(1000)
    for name, key, fw_cls, sampler_cls, B, guidance in (
            ("config2_dpmpp", "L", frameworks.ClassifierFreeGuidance, samplers.DpmSolverSampler, 16, bench.GUIDANCE),
            ("config2_dpmpp", "L", frameworks.ClassifierFreeGuidance, samplers.DpmSolverSampler, 16, 3.0),
            ("config5_sr_ddim", "SR", frameworks.SuperResCFG, samplers.DdimSampler, 8, bench.GUIDANCE)):
        cfg = bench.MODELS[key]
        net = backbones.AdmUnet2d(**cfg)
        net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234))
        fw = fw_cls(net.cuda(), timesteps=1000, beta_schedule="linear")
        s = sampler_cls(fw)
        S = cfg["image_size"]
        x_T = torch.randn(B, 4, S, S, generator=gen).cuda()
        kw = dict(noise=x_T, verbose=False, classes=torch.arange(B, device="cuda") % 1000, strength=guidance)
        if key == "SR":
            kw["y"] = torch.randn(B, 4, S // 2, S // 2, generator=gen).cuda()
        timed(lambda: s.sample(B, steps=5, **kw))
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        timed(lambda: s.sample(B, steps=5, apg=apg, **kw))
        torch.cuda.synchronize()
        free1 = torch.cuda.mem_get_info()[0]
        best, outs = {"off": None, "apg": None}, {}
        for rnd in range(1 + args.repeat):
            for k, ak in (("off", {}), ("apg", dict(apg=apg))):
                ms, out = timed(lambda: s.sample(B, steps=50, **ak, **kw).samples)
                outs[k] = out
                if rnd > 0 and (best[k] is None or ms / 50 < best[k]):
                    best[k] = ms / 50
        cases.append({"workload": name, "batch": B, "guidance": guidance, "ms_per_step_off": round(best["off"], 3),
                      "ms_per_step_apg": round(best["apg"], 3), "step_ratio": round(best["apg"] / best["off"], 4),
                      "apg_extra_mib": round((free0 - free1) / 2 ** 20, 1),
                      "rel_l2_apg_vs_cfg_drift_random_weights": round(_rel(outs["apg"], outs["off"]), 4)})
        del fw, net, s
        torch.cuda.empty_cache()
    print(f"{'workload':>16} {'B':>3} {'s':>5} {'off ms/step':>12} {'apg ms/step':>12} {'ratio':>7} {'+MiB':>7} {'rel L2':>8}")
    for c in cases:
        print(f"{c['workload']:>16} {c['batch']:>3} {c['guidance']:>5} {c['ms_per_step_off']:>12.3f} {c['ms_per_step_apg']:>12.3f} "
              f"{c['step_ratio']:>7.4f} {c['apg_extra_mib']:>7.1f} {c['rel_l2_apg_vs_cfg_drift_random_weights']:>8.4f}")
    print(json.dumps({"bench": "apg", "apg": apg, "card": card, "cases": cases, "card_after": _card()}))


if __name__ == "__main__":
    main()

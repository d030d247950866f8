"""Cost of classifier-free guidance restricted to an interval (`guidance_interval`) on the config-2 network
(rgbd_imagenet_adm_128_large_cfg with synthetic weights, as bench.py builds it; guidance 0.5, batch 16).  Prints tables and
one JSON line.

    python tools/bench_guidance.py [--batch 16] [--repeat 3] [--interval 100,600] [--ddpm-repeat 1]

- ms per step, guided against unguided: CUDA events around whole 50-step DPM-Solver++ `sample()` calls (production path,
  update fused into the output head) with no interval (every step guided, one batch-2N forward) and with an interval that
  excludes every model time of the grid (every step unguided, one batch-N forward); alternated, best of `repeat` rounds
  after a warm-up round.
- whole runs: DDPM 1000 steps and DPM-Solver++ 25 steps, with no interval and with `--interval`, in fp16 and in fp8.  The
  DPM-Solver++ runs take the best of `repeat` rounds; each DDPM run takes `ddpm-repeat` rounds (about a minute each).
- the device memory the batch-N plan adds (free memory before and after its first use).
- the relative L2 distance between each interval run and the fully guided run from the same x_T and seed.  Diagnostic drift
  on random weights, not a statement about sample quality.
Needs a GPU: there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch                                      # noqa: E402

import bench                                      # noqa: E402  (MODELS, GUIDANCE)
import ivid_b200.backbones as backbones           # noqa: E402
import ivid_b200.frameworks as frameworks         # noqa: E402
import ivid_b200.samplers as samplers             # noqa: E402
from ivid_b200.samplers.options import parse_interval   # noqa: E402
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
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--ddpm-repeat", type=int, default=1)
    ap.add_argument("--interval", type=parse_interval, default=(100, 600))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_guidance.py needs a GPU"
    card = _card()
    B = args.batch
    cfg = bench.MODELS["L"]
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234))
    fw = frameworks.ClassifierFreeGuidance(net.cuda(), timesteps=1000, beta_schedule="linear", p_uncond=0.1)
    ddpm, dpm = samplers.DdpmSampler(fw), samplers.DpmSolverSampler(fw)
    x_T = torch.randn(B, 4, cfg["image_size"], cfg["image_size"], generator=torch.Generator().manual_seed(1000)).cuda()
    classes = torch.arange(B, device="cuda") % 1000
    kw = dict(noise=x_T, classes=classes, strength=bench.GUIDANCE, verbose=False)
    none_of_grid = (0, 0)                            # the DPM-Solver++ grids of 5 / 25 / 50 steps start at model time 199 / 39 / 19

    def timed(fn):
        torch.manual_seed(0)                         # the Philox seed of the run is drawn from torch's generator
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    # memory of the batch-N plan: the batch-2N plan exists after the first guided run, the batch-N plan after the first
    # unguided step
    timed(lambda: dpm.sample(B, steps=5, **kw))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    timed(lambda: dpm.sample(B, steps=5, guidance_interval=none_of_grid, **kw))
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    extra_mib = (free0 - free1) / 2 ** 20

    # guided vs unguided step
    best = {"guided": None, "unguided": None}
    for rnd in range(1 + args.repeat):
        for name, gi in (("guided", None), ("unguided", none_of_grid)):
            ms, _ = timed(lambda: dpm.sample(B, steps=50, guidance_interval=gi, **kw))
            if rnd > 0 and (best[name] is None or ms / 50 < best[name]):
                best[name] = ms / 50
    step = {"guided_ms_per_step": round(best["guided"], 3), "unguided_ms_per_step": round(best["unguided"], 3),
            "unguided_over_guided": round(best["unguided"] / best["guided"], 4)}
    print(f"{'guided ms/step':>16} {'unguided ms/step':>18} {'ratio':>8}")
    print(f"{step['guided_ms_per_step']:>16.2f} {step['unguided_ms_per_step']:>18.2f} {step['unguided_over_guided']:>8.3f}")

    # whole runs
    lo, hi = args.interval
    runs = []
    for precision in ("fp16", "fp8"):
        net.set_precision(precision)
        for name, sampler, steps, rounds in (("dpmpp_25", dpm, 25, args.repeat), ("ddpm_1000", ddpm, 1000, args.ddpm_repeat)):
            if name == "dpmpp_25":
                timed(lambda: sampler.sample(B, steps=steps, **kw))                       # warm-up: plans and graphs of
                timed(lambda: sampler.sample(B, steps=steps, guidance_interval=(lo, hi), **kw))   # this precision
            res = {}
            for gi in (None, (lo, hi)):
                t_best, out = None, None
                for _ in range(rounds):
                    ms, o = timed(lambda: sampler.sample(B, steps=steps, guidance_interval=gi, **kw).samples)
                    t_best = ms if t_best is None else min(t_best, ms)
                    out = o
                res[gi] = (t_best, out)
            model_times = [t for t in range(1000)] if name == "ddpm_1000" else [1000 // steps * (i + 1) - 1 for i in range(steps)]
            guided_steps = sum(lo <= t <= hi for t in model_times)
            row = {"precision": precision, "run": name, "guided_steps": guided_steps, "steps": len(model_times),
                   "no_interval_ms": round(res[None][0], 1), "interval_ms": round(res[(lo, hi)][0], 1),
                   "speedup": round(res[None][0] / res[(lo, hi)][0], 3),
                   "rel_l2_interval_vs_guided_drift_random_weights": round(_rel(res[(lo, hi)][1], res[None][1]), 4)}
            runs.append(row)
    net.set_precision("fp16")
    print(f"{'precision':>9} {'run':>10} {'guided':>7} {'no interval ms':>15} {'interval ms':>12} {'speedup':>8} {'rel L2 (drift)':>15}")
    for r in runs:
        print(f"{r['precision']:>9} {r['run']:>10} {str(r['guided_steps']) + '/' + str(r['steps']):>7} {r['no_interval_ms']:>15.1f} "
              f"{r['interval_ms']:>12.1f} {r['speedup']:>8.3f} {r['rel_l2_interval_vs_guided_drift_random_weights']:>15.4f}")
    print(f"batch-N plan: {extra_mib:.1f} MiB of extra device memory")
    print(json.dumps({"bench": "guidance_interval", "model": "rgbd_imagenet_adm_128_large_cfg (synthetic weights)", "batch": B,
                      "guidance": bench.GUIDANCE, "interval": [lo, hi], "card": card, "step": step, "runs": runs,
                      "batch_n_plan_extra_mib": round(extra_mib, 1), "card_after": _card()}))


if __name__ == "__main__":
    main()

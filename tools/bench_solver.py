"""Convergence and speed of DPM-Solver++(2M) against DDIM on the config-2 network (rgbd_imagenet_adm_128_large_cfg with
synthetic weights, classifier-free guidance 0.5, batch 16).  Prints a table and one JSON line.

    python tools/bench_solver.py [--batch 16] [--steps 10,15,25,50] [--repeat 2]

The reference solution is a 1000-step DDIM (eta = 0) run from the same x_T.  For every step count both solvers run from that
x_T and report the relative L2 distance of their samples to it, and ms per denoising step (CUDA events around the whole
`sample()` call, the best of `repeat` timed runs after a warm-up run; production path: the update is fused into the output
head).  This measures how fast each solver converges to the ODE solution on synthetic weights.  It does not measure image
quality.  Needs a GPU: there is no fallback."""
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
from oracle import unet_ref                       # noqa: E402


def _card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_max_sm_clock_current_sm_clock"] = r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_max_sm_clock_current_sm_clock"] = f"unavailable: {e}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", default="10,15,25,50")
    ap.add_argument("--repeat", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_solver.py needs a GPU"
    B = args.batch
    cfg = bench.MODELS["L"]
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234))
    fw = frameworks.ClassifierFreeGuidance(net.cuda(), timesteps=1000, beta_schedule="linear", p_uncond=0.1)
    ddim, dpm = samplers.DdimSampler(fw), samplers.DpmSolverSampler(fw)
    x_T = torch.randn(B, 4, cfg["image_size"], cfg["image_size"], generator=torch.Generator().manual_seed(1000)).cuda()
    classes = torch.arange(B, device="cuda") % 1000
    kw = dict(noise=x_T, classes=classes, strength=bench.GUIDANCE, verbose=False)

    def timed(sampler, steps, **extra):
        best, out = None, None
        for _ in range(1 + args.repeat):              # the first run warms up this step count's plan and graph
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = sampler.sample(B, steps=steps, **kw, **extra).samples
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / steps
            best = ms if best is None or ms < best else best
        return out, best

    card = _card()
    ref = ddim.sample(B, steps=1000, eta=0.0, **kw).samples.double()
    rows = []
    for n in [int(s) for s in args.steps.split(",")]:
        row = {"steps": n}
        for name, s, extra in (("ddim", ddim, dict(eta=0.0)), ("dpmpp_2m", dpm, dict(order=2))):
            out, ms = timed(s, n, **extra)
            row[f"{name}_rel_l2"] = float((out.double() - ref).norm() / ref.norm())
            row[f"{name}_ms_per_step"] = round(ms, 3)
        rows.append(row)
    print(f"{'steps':>6} {'DDIM rel L2':>12} {'DPM++(2M) rel L2':>17} {'DDIM ms/step':>13} {'DPM++ ms/step':>14}")
    for r in rows:
        print(f"{r['steps']:>6} {r['ddim_rel_l2']:>12.3e} {r['dpmpp_2m_rel_l2']:>17.3e} {r['ddim_ms_per_step']:>13.2f} "
              f"{r['dpmpp_2m_ms_per_step']:>14.2f}")
    print(json.dumps({"bench": "solver_convergence", "model": "rgbd_imagenet_adm_128_large_cfg (synthetic weights)", "batch": B,
                      "guidance": bench.GUIDANCE, "reference": "DDIM eta=0, 1000 steps, same x_T", "card": card,
                      "card_after": _card(), "rows": rows}))


if __name__ == "__main__":
    main()

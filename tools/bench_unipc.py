"""Convergence and speed of UniPC against DDIM and DPM-Solver++(2M) on the config-2 network (rgbd_imagenet_adm_128_large_cfg
with synthetic weights, classifier-free guidance 0.5, batch 16).  Prints a table and one JSON line.

    python tools/bench_unipc.py [--batch 16] [--steps 5,10,20,25,50] [--repeat 3]

The reference solution is a 1000-step DDIM (eta = 0) run from the same x_T.  For every step count each method runs from that
x_T and reports the relative L2 distance to it of its final samples and of its x at t = 200 (a point of every grid used,
before the final step's jump to x_0; UniPC: the prediction the network sees there).  ms per denoising step: CUDA events
around the whole `sample()` call on the production path (the update fused into the output head), the methods alternated,
the best of `repeat` timed runs after a warm-up run.  The step tail (the step-state kernel and the fused output-head step
kernel, every kernel whose name holds "step_kernel") is timed separately with torch.profiler on one 10-step run per method.  This measures convergence to the ODE solution on random weights, not
image quality.  Needs a GPU: there is no fallback."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch                                      # noqa: E402

import bench                                      # noqa: E402  (MODELS, GUIDANCE)
import ivid_b200.backbones as backbones           # noqa: E402
import ivid_b200.frameworks as frameworks         # noqa: E402
import ivid_b200.samplers as samplers             # noqa: E402
from bench_solver import _card                    # noqa: E402
from oracle import unet_ref                       # noqa: E402

T_MID = 200


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", default="5,10,20,25,50")
    ap.add_argument("--repeat", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_unipc.py needs a GPU"
    B = args.batch
    cfg = bench.MODELS["L"]
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234))
    fw = frameworks.ClassifierFreeGuidance(net.cuda(), timesteps=1000, beta_schedule="linear", p_uncond=0.1)
    ddim, dpm, uni = samplers.DdimSampler(fw), samplers.DpmSolverSampler(fw), samplers.UniPcSampler(fw)
    methods = (("ddim", ddim, dict(eta=0.0)), ("dpmpp_2m", dpm, dict(order=2)), ("unipc_2", uni, dict(order=2)),
               ("unipc_3", uni, dict(order=3)))
    x_T = torch.randn(B, 4, cfg["image_size"], cfg["image_size"], generator=torch.Generator().manual_seed(1000)).cuda()
    classes = torch.arange(B, device="cuda") % 1000
    kw = dict(noise=x_T, classes=classes, strength=bench.GUIDANCE, verbose=False)
    card = _card()

    def at_mid(sampler, steps, **extra):
        """(final samples, x at t = 200) of one run with trajectories (the separate route: the same bits as the fused one)."""
        res = sampler.sample(B, steps=steps, return_trajectory=True, **kw, **extra)
        jump = 1000 // steps
        i = steps - 1 - T_MID // jump          # step i ends at t_prev = jump * (steps - 1 - i)
        mid = res.pred_x_t[i].double().clone()
        return res.samples.double(), mid

    ref, ref_mid = at_mid(ddim, 1000, eta=0.0)
    rel = lambda a, b: float((a - b).norm() / b.norm())
    rows = []
    for n in [int(s) for s in args.steps.split(",")]:
        assert (1000 // n) and T_MID % (1000 // n) == 0, f"t = {T_MID} is not on the {n}-step grid"
        row = {"steps": n}
        for name, s, extra in methods:
            final, mid = at_mid(s, n, **extra)
            row[f"{name}_rel_l2"] = rel(final, ref)
            row[f"{name}_rel_l2_t{T_MID}"] = rel(mid, ref_mid)
        best = {name: None for name, _, _ in methods}
        for rep in range(1 + args.repeat):    # rep 0 warms up this step count's plans and graphs
            for name, s, extra in methods:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                s.sample(B, steps=n, **kw, **extra)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / n
                if rep > 0 and (best[name] is None or ms < best[name]):
                    best[name] = ms
        for name in best:
            row[f"{name}_ms_per_step"] = round(best[name], 3)
        rows.append(row)

    # the step tail: device time of set_step_kernel and the fused step kernel (the output head's last node) per step
    tail = {}
    for name, s, extra in methods:
        s.sample(B, steps=10, **kw, **extra)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            s.sample(B, steps=10, **kw, **extra)
            torch.cuda.synchronize()
        us = [e.time_range.elapsed_us() for e in prof.events()
              if e.device_type == torch.autograd.DeviceType.CUDA and "step_kernel" in e.name]
        tail[name] = {"launches": len(us), "us_per_step": round(sum(us) / 10, 2) if us else None}

    hdr = f"{'steps':>5} " + " ".join(f"{name + ' L2':>14} {name + ' L2@200':>16} {name + ' ms':>12}" for name, _, _ in methods)
    print(hdr)
    for r in rows:
        print(f"{r['steps']:>5} " + " ".join(f"{r[f'{m}_rel_l2']:>14.3e} {r[f'{m}_rel_l2_t{T_MID}']:>16.3e} {r[f'{m}_ms_per_step']:>12.2f}"
                                            for m, _, _ in methods))
    print("step tail (us/step):", {k: v["us_per_step"] for k, v in tail.items()})
    print(json.dumps({"bench": "unipc_convergence", "model": "rgbd_imagenet_adm_128_large_cfg (synthetic weights)", "batch": B,
                      "guidance": bench.GUIDANCE, "reference": "DDIM eta=0, 1000 steps, same x_T", "card": card,
                      "card_after": _card(), "rows": rows, "step_tail": tail}))


if __name__ == "__main__":
    main()

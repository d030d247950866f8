"""Step cost of the stochastic DPM-Solver++(2M) (DpmSolverSampler with sde=True) against DDIM (eta 0 and 1) and the ODE
solver, on the config-2 network (rgbd_imagenet_adm_128_large_cfg with synthetic weights, classifier-free guidance 0.5,
batch 16).  Prints tables and one JSON line.

    python tools/bench_sde.py [--batch 16] [--repeat 3] [--out DIR] [--dump-ode25 DIR]

ms per denoising step: CUDA events around the whole `sample()` call (production path: the update is fused into the output
head), at 25 and 50 steps, the four samplers alternated in one process, best of `repeat` rounds after a warm-up round.

Diagnostic, not a quality claim: SDE 2M and DDIM eta = 1 at 10, 25, 50 and 100 steps, and a 1000-step DDPM set, all from the
same x_T on these random weights; for each, the per-channel mean and std of the samples over batch and pixels.

`--out DIR` writes the 25-step ODE 2M samples as DIR/dpmpp_ode_25.npy.  `--dump-ode25 DIR` writes only that file and exits,
so two builds can be compared bit for bit.  Needs a GPU: there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
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


def _moments(x):
    """Per-channel mean and std over batch and pixels."""
    x = x.double()
    return {"mean": [round(float(v), 4) for v in x.mean(dim=(0, 2, 3))], "std": [round(float(v), 4) for v in x.std(dim=(0, 2, 3))]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dump-ode25", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sde.py needs a GPU"
    B = args.batch
    cfg = bench.MODELS["L"]
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234))
    fw = frameworks.ClassifierFreeGuidance(net.cuda(), timesteps=1000, beta_schedule="linear", p_uncond=0.1)
    ddim, dpm = samplers.DdimSampler(fw), samplers.DpmSolverSampler(fw)
    x_T = torch.randn(B, 4, cfg["image_size"], cfg["image_size"], generator=torch.Generator().manual_seed(1000)).cuda()
    classes = torch.arange(B, device="cuda") % 1000
    kw = dict(noise=x_T, classes=classes, strength=bench.GUIDANCE, verbose=False)

    def run(name, steps, seed=0):
        torch.manual_seed(seed)                       # the Philox seed of the run is drawn from torch's generator
        if name == "ddim_eta0":
            return ddim.sample(B, steps=steps, eta=0.0, **kw).samples
        if name == "ddim_eta1":
            return ddim.sample(B, steps=steps, eta=1.0, **kw).samples
        if name == "dpmpp_ode":
            return dpm.sample(B, steps=steps, order=2, **kw).samples
        if name == "dpmpp_sde":
            return dpm.sample(B, steps=steps, order=2, sde=True, **kw).samples
        raise ValueError(name)

    def dump(d):
        os.makedirs(d, exist_ok=True)
        np.save(os.path.join(d, "dpmpp_ode_25.npy"), run("dpmpp_ode", 25).cpu().numpy())

    if args.dump_ode25:
        dump(args.dump_ode25)
        return
    card = _card()
    names = ("ddim_eta0", "ddim_eta1", "dpmpp_ode", "dpmpp_sde")
    step_counts = (25, 50)
    best = {(n, s): None for n in names for s in step_counts}
    for rnd in range(1 + args.repeat):                # round 0 warms up every step count's plan and graph
        for s in step_counts:
            for n in names:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(n, s)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / s
                if rnd > 0 and (best[(n, s)] is None or ms < best[(n, s)]):
                    best[(n, s)] = ms
    timing = [{"steps": s, **{f"{n}_ms_per_step": round(best[(n, s)], 3) for n in names}} for s in step_counts]
    print(f"{'steps':>6} " + " ".join(f"{n + ' ms/step':>18}" for n in names))
    for r in timing:
        print(f"{r['steps']:>6} " + " ".join(f"{r[n + '_ms_per_step']:>18.2f}" for n in names))
    if args.out:
        dump(args.out)

    torch.manual_seed(0)
    ref = samplers.DdpmSampler(fw).sample(B, **kw).samples
    diag = {"ddpm_1000": _moments(ref)}
    for s in (10, 25, 50, 100):
        for n in ("dpmpp_sde", "ddim_eta1"):
            diag[f"{n}_{s}"] = _moments(run(n, s))
    print(f"{'run':>16} " + " ".join(f"{'mean c' + str(c):>9}" for c in range(4)) + " " + " ".join(f"{'std c' + str(c):>8}" for c in range(4)))
    for k, v in diag.items():
        print(f"{k:>16} " + " ".join(f"{m:>9.4f}" for m in v["mean"]) + " " + " ".join(f"{m:>8.4f}" for m in v["std"]))
    print(json.dumps({"bench": "sde_step_cost", "model": "rgbd_imagenet_adm_128_large_cfg (synthetic weights)", "batch": B,
                      "guidance": bench.GUIDANCE, "card": card, "timing": timing,
                      "diagnostic_same_x_T_random_weights": diag, "card_after": _card()}))


if __name__ == "__main__":
    main()

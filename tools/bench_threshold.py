"""Cost of dynamic thresholding (`dynamic_threshold`) on the config-2 network (rgbd_imagenet_adm_128_large_cfg, synthetic weights,
as bench.py builds it; batch 16, guidance 0.5 and 3.0) and on config 5 (rgbd_imagenet_adm_256_128_small_sr, SuperResCFG at
256x256, batch 8, guidance 0.5).  Prints tables and one JSON line.

    python tools/bench_threshold.py [--repeat 3] [--ratio 0.995] [--profile-dir DIR]

- ms per step with and without thresholding: CUDA events around whole `sample()` calls (production path, fused route),
  DPM-Solver++ 25 steps and DDIM 50 steps, the two settings alternated, best of `repeat` rounds after a warm-up round.
- device time of the step's kernels, from torch.profiler in a separate run of 5 DPM-Solver++ steps each: the fused head step
  step_kernel<HeadTaps, Update<2>> without thresholding; with it step_kernel<HeadTaps, StoreX0> (x_0 out of the head),
  threshold_select_kernel and step_kernel<ThresholdedX0, Update<2>> (the update).
- the relative L2 distance and the largest |x| of the final samples with and without thresholding.  Diagnostic drift on random
  weights, not a statement about sample quality.
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
from oracle import unet_ref                       # noqa: E402

# every instantiation of step_kernel<Source, Sink> (not set_step_kernel), and the selection of a thresholded step
STEP_KERNELS = ("step_kernel<", "threshold_select_kernel")


def _card():
    info = {"torch_name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["name_power_limit_max_sm_clock"] = r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["name_power_limit_max_sm_clock"] = f"unavailable: {e}"
    return info


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def _timed(fn):
    torch.manual_seed(0)                             # the Philox seed of the run is drawn from torch's generator
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def _net(key, fw_cls):
    cfg = bench.MODELS[key]
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234))
    return fw_cls(net.cuda(), timesteps=1000, beta_schedule="linear", p_uncond=0.1), cfg["image_size"]


def _compare(name, run, steps, ratio, repeat):
    """Alternated best-of-`repeat` ms per step of run(threshold) with threshold None and `ratio`, after a warm-up round."""
    for th in (None, ratio):
        _timed(lambda: run(th))
    best = {None: float("inf"), ratio: float("inf")}
    outs = {}
    for _ in range(repeat):
        for th in (None, ratio):
            ms, outs[th] = _timed(lambda: run(th))
            best[th] = min(best[th], ms)
    plain, thr = best[None] / steps, best[ratio] / steps
    row = dict(workload=name, ms_per_step_plain=round(plain, 4), ms_per_step_threshold=round(thr, 4),
               overhead_pct=round(100.0 * (thr - plain) / plain, 3), drift_rel_l2=_rel(outs[ratio], outs[None]),
               max_abs_plain=float(outs[None].abs().max()), max_abs_threshold=float(outs[ratio].abs().max()))
    print(f"{name:58s} plain {plain:8.3f} ms/step  thresholded {thr:8.3f} ms/step  overhead {row['overhead_pct']:+.3f} %  "
          f"drift {row['drift_rel_l2']:.3e}  max|x| {row['max_abs_plain']:.3f} -> {row['max_abs_threshold']:.3f}")
    return row


def _profile(run, out_dir):
    """Device time per kernel name of one 5-step run, from torch.profiler (CUDA activities)."""
    run()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        run()
        torch.cuda.synchronize()
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, f"threshold_{len(os.listdir(out_dir))}.pt.trace.json"))
    times = {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA or getattr(ev, "self_device_time_total", 0) > 0:
            dt = getattr(ev, "self_device_time_total", None)
            if dt is None:
                dt = ev.self_cuda_time_total
            if dt > 0:
                times[ev.key] = (times.get(ev.key, (0.0, 0))[0] + dt / 1000.0, ev.count)
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--ratio", type=float, default=0.995)
    ap.add_argument("--profile-dir", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_threshold.py needs a GPU"
    card = _card()
    rows = []
    # config 2: batch 16, guidance 0.5 (the bench's protocol) and 3.0 (the reference CLI's default)
    fw, S = _net("L", frameworks.ClassifierFreeGuidance)
    B = 16
    x_T = torch.randn(B, 4, S, S, generator=torch.Generator().manual_seed(1000)).cuda()
    classes = torch.arange(B, device="cuda") % 1000
    dpm, ddim = samplers.DpmSolverSampler(fw), samplers.DdimSampler(fw)
    for g in (bench.GUIDANCE, 3.0):
        for name, s, steps in (("DPM-Solver++ 25", dpm, 25), ("DDIM 50", ddim, 50)):
            run = lambda th, s=s, steps=steps, g=g: s.sample(B, noise=x_T, classes=classes, steps=steps, strength=g, verbose=False,
                                                             dynamic_threshold=th).samples
            rows.append(_compare(f"config 2, {name}, guidance {g}, batch {B}", run, steps, args.ratio, args.repeat))
    prof_rows = {}
    for th in (None, args.ratio):
        times = _profile(lambda: dpm.sample(B, noise=x_T, classes=classes, steps=5, strength=bench.GUIDANCE, verbose=False,
                                            dynamic_threshold=th), args.profile_dir)
        sel = {k: v for k, v in times.items() if any(a in k for a in STEP_KERNELS)}
        prof_rows["threshold" if th else "plain"] = {k: dict(ms_total=round(v[0], 4), calls=v[1]) for k, v in sel.items()}
    print("device time, 5 DPM-Solver++ steps (torch.profiler):")
    for mode, sel in prof_rows.items():
        for k, v in sel.items():
            print(f"  {mode:9s} {k[:90]:90s} {v['ms_total']:9.4f} ms over {v['calls']} launches")
    del dpm, ddim, fw
    torch.cuda.empty_cache()
    # config 5: super-resolution at 256x256, batch 8, guidance 0.5
    fw, S = _net("SR", frameworks.SuperResCFG)
    B = 8
    x_T = torch.randn(B, 4, S, S, generator=torch.Generator().manual_seed(1001)).cuda()
    y = torch.randn(B, 4, S // 2, S // 2, generator=torch.Generator().manual_seed(1002)).cuda().clamp(-1, 1)
    classes = torch.arange(B, device="cuda") % 1000
    for name, s, steps in (("DPM-Solver++ 25", samplers.DpmSolverSampler(fw), 25), ("DDIM 50", samplers.DdimSampler(fw), 50)):
        run = lambda th, s=s, steps=steps: s.sample(B, noise=x_T, classes=classes, steps=steps, strength=bench.GUIDANCE, y=y,
                                                    verbose=False, dynamic_threshold=th).samples
        rows.append(_compare(f"config 5, {name}, guidance {bench.GUIDANCE}, batch {B}", run, steps, args.ratio, args.repeat))
    print(json.dumps(dict(card=card, ratio=args.ratio, repeat=args.repeat, rows=rows, profile=prof_rows)))


if __name__ == "__main__":
    main()

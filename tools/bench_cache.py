"""Cost of feature reuse between denoising steps (DeepCache: `cache_interval`, `cache_branch`) on the config-2 network
(rgbd_imagenet_adm_128_large_cfg with synthetic weights, as bench.py builds it; guidance 0.5, batch 16, so one guided forward
is batch 32) and the config-5 SR network (rgbd_imagenet_adm_256_128_small_sr, batch 8, guided: batch 16).  Prints tables
and one JSON line.

    python tools/bench_cache.py [--batch 16] [--sr-batch 8] [--repeat 3] [--iters 10] [--ddpm-repeat 1]

- ms per forward: CUDA events around `iters` back-to-back forwards (CUDA-graph replays) of the full forward and of the
  reuse forward at branches 0, 1 and 2, alternated; best of `repeat` rounds after a warm-up round.
- whole runs of the config-2 network (update fused into the output head): DDPM 1000 steps at cache intervals 1, 2, 3 and 5
  (branch 0) and DPM-Solver++ 25 steps at intervals 1, 2 and 3 (branch 0).  DPM-Solver++ runs take the best of `repeat`
  rounds; each DDPM run takes `ddpm-repeat` rounds (about a minute each at interval 1).
- the relative L2 distance of each cached run to the uncached run from the same x_T and seed.  Drift on random weights, not
  a statement about image quality.
Needs a GPU: there is no fallback."""
import argparse
import ctypes
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
from ivid_b200 import _lib                        # noqa: E402
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


def _net(key):
    cfg = bench.MODELS[key]
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234))
    net = net.cuda()
    net._ensure_packed()
    return cfg, net


def forward_times(key, batch, repeat, iters):
    """ms per guided forward (batch 2 x `batch`): full, and reuse at each branch."""
    cfg, net = _net(key)
    S = cfg["image_size"]
    N = 2 * batch
    g = torch.Generator().manual_seed(7)
    x = torch.randn(N, 4, S, S, generator=g).cuda()
    t = torch.full((N,), 500, dtype=torch.int64, device="cuda")
    classes = torch.cat([torch.arange(batch), torch.full((batch,), -1)]).cuda()
    eps = torch.empty(N, 4, S, S, device="cuda")
    cond, keep = None, []
    if cfg["in_channels"] == 8:                      # SuperResCFG: y at half the size, bilinear-upsampled in the input packing
        y = torch.randn(N, 4, S // 2, S // 2, generator=g).cuda()
        keep.append(y)
        cond = _lib.CondT(kind=2, y_dev=y.data_ptr())
    L = _lib.lib()
    args = (net._handle, _lib.ptr(x), N, S, S, ctypes.byref(cond) if cond is not None else None, _lib.ptr(t), _lib.ptr(classes),
            _lib.ptr(eps), N)
    stream = _lib.cur_stream()

    def run(branch):
        if branch is None:
            _lib.check(L.ivid_unet_forward_hw(*args, stream))
        else:
            _lib.check(L.ivid_unet_forward_reuse(*args, branch, stream))

    modes = [None] + list(range(min(cfg["num_res_blocks"], 2) + 1))
    best = {m: None for m in modes}
    for rnd in range(1 + repeat):
        for m in modes:
            run(None)                                 # the reuse forwards read what the last full forward stored
            run(m)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                run(m)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / iters
            if rnd > 0 and (best[m] is None or ms < best[m]):
                best[m] = ms
    row = {"network": key, "forward_batch": N, "full_ms": round(best[None], 3)}
    for m in modes[1:]:
        row[f"reuse_b{m}_ms"] = round(best[m], 3)
        row[f"reuse_b{m}_over_full"] = round(best[m] / best[None], 4)
    del net
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--sr-batch", type=int, default=8)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--ddpm-repeat", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_cache.py needs a GPU"
    card = _card()

    fwd = [forward_times("L", args.batch, args.repeat, args.iters), forward_times("SR", args.sr_batch, args.repeat, args.iters)]
    print(f"{'network':>8} {'batch':>6} {'full ms':>9} {'b0 ms':>8} {'b0/full':>8} {'b1 ms':>8} {'b1/full':>8} {'b2 ms':>8} {'b2/full':>8}")
    for r in fwd:
        print(f"{r['network']:>8} {r['forward_batch']:>6} {r['full_ms']:>9.2f} " +
              " ".join(f"{r.get(f'reuse_b{b}_ms', float('nan')):>8.2f} {r.get(f'reuse_b{b}_over_full', float('nan')):>8.3f}"
                       for b in range(3)))

    B = args.batch
    cfg, net = _net("L")
    fw = frameworks.ClassifierFreeGuidance(net, timesteps=1000, beta_schedule="linear", p_uncond=0.1)
    ddpm, dpm = samplers.DdpmSampler(fw), samplers.DpmSolverSampler(fw)
    x_T = torch.randn(B, 4, cfg["image_size"], cfg["image_size"], generator=torch.Generator().manual_seed(1000)).cuda()
    classes = torch.arange(B, device="cuda") % 1000
    kw = dict(noise=x_T, classes=classes, strength=bench.GUIDANCE, verbose=False)

    def timed(fn):
        torch.manual_seed(0)                         # the Philox seed of the run is drawn from torch's generator
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    runs = []
    for name, sampler, steps, intervals, rounds in (("dpmpp_25", dpm, 25, (1, 2, 3), args.repeat),
                                                    ("ddpm_1000", ddpm, 1000, (1, 2, 3, 5), args.ddpm_repeat)):
        if name == "dpmpp_25":
            for ci in intervals:                     # warm-up: plans and graphs
                timed(lambda: sampler.sample(B, steps=steps, cache_interval=ci, **kw))
        res = {}
        for ci in intervals:
            t_best, out = None, None
            for _ in range(rounds):
                ms, o = timed(lambda: sampler.sample(B, steps=steps, cache_interval=ci, **kw).samples)
                t_best = ms if t_best is None else min(t_best, ms)
                out = o
            res[ci] = (t_best, out)
        for ci in intervals:
            full_steps = len(range(0, steps, ci))
            runs.append({"run": name, "cache_interval": ci, "cache_branch": 0, "full_steps": full_steps, "steps": steps,
                         "ms": round(res[ci][0], 1), "speedup": round(res[1][0] / res[ci][0], 3),
                         "rel_l2_vs_uncached_drift_random_weights": round(_rel(res[ci][1], res[1][1]), 4)})
    print(f"{'run':>10} {'interval':>9} {'full steps':>11} {'ms':>10} {'speedup':>8} {'rel L2 (drift)':>15}")
    for r in runs:
        print(f"{r['run']:>10} {r['cache_interval']:>9} {str(r['full_steps']) + '/' + str(r['steps']):>11} {r['ms']:>10.1f} "
              f"{r['speedup']:>8.3f} {r['rel_l2_vs_uncached_drift_random_weights']:>15.4f}")
    print(json.dumps({"bench": "feature_cache", "model": "rgbd_imagenet_adm_128_large_cfg / rgbd_imagenet_adm_256_128_small_sr "
                      "(synthetic weights)", "batch": B, "sr_batch": args.sr_batch, "guidance": bench.GUIDANCE, "card": card,
                      "forward": fwd, "runs": runs, "card_after": _card()}))


if __name__ == "__main__":
    main()

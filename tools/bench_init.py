"""Cost of starting from a given image, on bench.py's networks (synthetic weights, guidance 0.5).  Prints tables and one
JSON line with the card's name and power limit.

    python tools/bench_init.py [--batch 16] [--repeat 5] [--ddpm-rounds 1] [--scene-batch 4] [--skip-scene]

- ivid_sampler_diffuse at the config-2 size ([batch, 4, 128, 128] fp32), with Philox and with injected noise: CUDA events
  around 200 back-to-back calls, best of `repeat`.  The op is HBM-bound: it moves 8 bytes per element (x_0 in, x_t out), 12
  with injected noise; the table gives GB/s against the H100 SXM data sheet's 3.35 TB/s.
- a DDPM run (the config-2 workload: rgbd_imagenet_adm_128_large_cfg, 1000 steps) from an image at strength 0.25 / 0.5 /
  1.0 against a plain run from x_T, CUDA events around `sample()`, after a warm-up run; best of `ddpm-rounds`.
- one 3x9 `sample_all` batch (1000 DDPM steps for view 0, 26 conditional views x 50 DDIM steps) with a given first view (no
  unconditional model) against one without; host clock around the whole generator, which ends in a device synchronise.
Needs a GPU: there is no fallback."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch                                      # noqa: E402

import bench                                      # noqa: E402  (MODELS, GUIDANCE, WARP_KW)
import ivid_b200.backbones as backbones           # noqa: E402
import ivid_b200.frameworks as frameworks         # noqa: E402
import ivid_b200.samplers as samplers             # noqa: E402
from ivid_b200 import _lib                        # noqa: E402
from ivid_b200.inference import build_modelviews, sample_all   # noqa: E402
from oracle import unet_ref                       # noqa: E402
from bench_guidance import _card                  # noqa: E402

HBM_TBS = 3.35


def _fw(key, cls):
    cfg = bench.MODELS[key]
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234))
    return cls(net.cuda(), timesteps=1000, beta_schedule="linear", p_uncond=0.1)


def timed(fn):
    torch.manual_seed(0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--ddpm-rounds", type=int, default=1)
    ap.add_argument("--scene-batch", type=int, default=4)
    ap.add_argument("--skip-scene", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_init.py needs a GPU"
    card = _card()
    B = args.batch
    fu = _fw("L", frameworks.ClassifierFreeGuidance)
    S = bench.MODELS["L"]["image_size"]
    ddpm = samplers.DdpmSampler(fu)
    gen = torch.Generator().manual_seed(1000)
    x0 = (torch.rand(B, 4, S, S, generator=gen) * 2 - 1).cuda()
    z = torch.randn(B, 4, S, S, generator=gen).cuda()
    out = torch.empty_like(x0)
    result = {"card": card, "batch": B}

    # the diffusion op
    L, st = _lib.lib(), _lib.cur_stream()
    calls = 200
    rows = []
    for name, noise, bytes_per_el in (("philox", None, 8), ("injected", z, 12)):
        call = lambda: L.ivid_sampler_diffuse(ddpm._handle, _lib.ptr(x0), _lib.ptr(noise), B, x0[0].numel(), 499, 7,
                                              _lib.ptr(out), st)
        _lib.check(call())
        best = min(timed(lambda: [call() for _ in range(calls)]) for _ in range(args.repeat)) / calls
        gbs = x0.numel() * bytes_per_el / (best * 1e-3) / 1e9
        rows.append({"noise": name, "us_per_call": round(best * 1e3, 2), "GB_per_s": round(gbs, 1),
                     "share_of_3.35TBps": round(gbs / (HBM_TBS * 1e3), 3)})
    result["diffuse"] = rows
    print(f"{'diffuse noise':>14} {'us/call':>9} {'GB/s':>8} {'of 3.35 TB/s':>13}")
    for r in rows:
        print(f"{r['noise']:>14} {r['us_per_call']:>9.2f} {r['GB_per_s']:>8.1f} {r['share_of_3.35TBps']:>13.3f}")

    # DDPM runs from an image against a plain run
    classes = torch.arange(B, device="cuda") % 1000
    kw = dict(classes=classes, strength=bench.GUIDANCE, verbose=False)
    plain = lambda: ddpm.sample(B, noise=z, **kw)
    init = lambda s: (lambda: ddpm.sample(B, noise=z, init=x0, init_strength=s, **kw))
    timed(plain)                                     # warm-up: plans and graphs
    runs = {"plain": plain, "0.25": init(0.25), "0.5": init(0.5), "1.0": init(1.0)}
    best = {}
    for _ in range(args.ddpm_rounds):
        for name, fn in runs.items():
            ms = timed(fn)
            best[name] = min(best.get(name, ms), ms)
    result["ddpm_runs_ms"] = {k: round(v, 1) for k, v in best.items()}
    print(f"{'DDPM run':>10} {'ms':>10} {'of plain':>9}")
    for name, ms in best.items():
        print(f"{name:>10} {ms:>10.1f} {ms / best['plain']:>9.3f}")

    # one 3x9 scene batch with and without a given first view
    if not args.skip_scene:
        fc = _fw("Lc", frameworks.InpaintCFG)
        nb = args.scene_batch
        mvs = build_modelviews("3x9", nb)
        views = x0[:nb].clone()
        cls = [int(c) for c in classes[:nb]]

        def scene(given):
            t0 = time.perf_counter()
            for _ in sample_all(None if given else fu, fc, nb, bench.DENOISE_STEPS, bench.COND_STEPS, mvs, classes=cls,
                                guidance=bench.GUIDANCE, batchsize=nb, init_views=views if given else None, **bench.WARP_KW):
                pass
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        scene(True)                                  # warm-up: the conditional plans and the warp
        t_plain, t_given = scene(False), scene(True)
        result["scene_3x9_s"] = {"batch": nb, "generated_first_view": round(t_plain, 2), "given_first_view": round(t_given, 2),
                                 "given_over_generated": round(t_given / t_plain, 4)}
        print(f"3x9 batch of {nb}: generated first view {t_plain:.2f} s, given first view {t_given:.2f} s "
              f"({t_given / t_plain:.3f}x)")
    print(json.dumps(result))


if __name__ == "__main__":
    main()

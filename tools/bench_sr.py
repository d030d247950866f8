#!/usr/bin/env python
"""Cost of the super-resolution stage of the multiview pipeline (inference/superres.py) on one GPU, synthetic weights.

    python tools/bench_sr.py [--batch 8] [--steps 50] [--viewsets random,3x9] [--out FILE.json]

Networks: bench.py's config-5 SR network (rgbd_imagenet_adm_256_128_small_sr, 128^2 -> 256^2) and, for the 128^2 pipeline
beside it, the config-2 / 3 networks (rgbd_imagenet_adm_128_large_cfg / _cond), all on seeded synthetic weights.  Inputs:
smooth synthetic RGBD views at 128^2 (a random-weight sampler's depth is noise).  Guidance 3.0 (the stage's default; the
cost does not depend on it).

Reported, measured with device synchronisation on this card:
  sr_step_ms          one DDIM step of the SR network with classifier-free guidance at the batch (view 0 of a run, steps/run)
  warp_ms_per_view    add_view + aggregate of one view at 256^2 (768^2 render) over the 3x9 camera sequence, CUDA events
  stage_s_per_scene   superresolve_views over all V views of a batch, wall clock / batch, per view set, after a set-up run
                      (one step per view) that allocates the batch's warp and the samplers in the same cache; the
                      breakdown prints the steps, the warps and the host draw of the seeded x_T that each run includes
and, computed from measured step times (not a run of the whole pipeline):
  lowres_s_per_scene  (1000 t_uncond + (V - 1) (50 t_cond + t_warp128)) / batch: the 128^2 pipeline's time per scene, with
                      t_uncond a guided DDIM step of the unconditional network standing in for its DDPM step (same forward)
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import MODELS, WARP_KW, synth_rgbd  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:       # the numbers are still printed, without the card
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--viewsets", default="random,3x9")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sr measures on the GPU"
    import ivid_b200.backbones as backbones
    import ivid_b200.frameworks as frameworks
    import ivid_b200.samplers as samplers
    from ivid_b200.inference import build_modelviews, superresolve_views
    from ivid_b200.rgbd_3d import DeviceWarp
    from oracle import unet_ref

    dev = torch.device("cuda", 0)
    B, steps = args.batch, args.steps

    def net(key, seed):
        n = backbones.AdmUnet2d(**MODELS[key])
        n.load_state_dict(unet_ref.make_synthetic_state_dict(MODELS[key], seed=seed))
        return n.to(dev)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    rng = np.random.default_rng(7)
    classes = torch.arange(B, device=dev) % 1000
    res = {"card": card(), "batch": B, "steps": steps}

    # ---- SR step
    fw_sr = frameworks.SuperResCFG(net("SR", 4321), timesteps=1000, beta_schedule="linear")
    s_sr = samplers.DdimSampler(fw_sr)
    y = torch.from_numpy(np.stack([synth_rgbd(rng).transpose(2, 0, 1) * 2 - 1 for _ in range(B)])).float().to(dev)
    run = lambda: s_sr.sample(B, y=y, classes=classes, steps=steps, strength=3.0, verbose=False, image_size=256)
    run()
    t, _ = timed(run)
    res["sr_step_ms"] = 1e3 * t / steps

    # ---- warp at 256^2 (and 128^2 for the pipeline beside it)
    views = build_modelviews("3x9", 1)

    def warp_ms(n):
        w = DeviceWarp(B, image_size=n, ssaa=3, max_views=27)
        src = [torch.from_numpy(np.stack([synth_rgbd(rng, n).transpose(2, 0, 1) * 2 - 1 for _ in range(B)])).float().to(dev)
               for _ in range(4)]
        ms = []
        for rep in range(2):                # the first pass warms up
            w.reset()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            for j in range(26):
                w.add_view(src[j % 4], views[j], **WARP_KW)
                w.aggregate(views[j + 1], **WARP_KW)
            ev[1].record()
            torch.cuda.synchronize()
            ms.append(ev[0].elapsed_time(ev[1]) / 26)
        return ms[-1]
    res["warp_ms_per_view"] = warp_ms(256)
    warp128 = warp_ms(128)

    # ---- the stage per view set
    res["stage_s_per_scene"] = {}
    for vs in args.viewsets.split(","):
        mvs = build_modelviews(vs, B, rng=np.random.default_rng(3)) if vs == "random" else build_modelviews(vs, 1)
        V = len(mvs[0]) if vs == "random" else len(mvs)
        low = torch.from_numpy(np.stack([np.stack([synth_rgbd(rng).transpose(2, 0, 1) * 2 - 1 for _ in range(V)]) for _ in range(B)]))
        low = low.float().to(dev)
        cache = {}
        kw = dict(classes=classes, guidance=3.0, seeds=list(range(B)), cache=cache, **WARP_KW)
        # set-up: the first run (one step per view) allocates the batch's warp and the samplers into the timed run's cache
        t_setup, _ = timed(lambda: superresolve_views(fw_sr, low, mvs, steps=1, **kw))
        t, _ = timed(lambda: superresolve_views(fw_sr, low, mvs, steps=steps, **kw))
        # part of every run: the seeded x_T, drawn on the host and copied to the device
        t_noise, _ = timed(lambda: torch.stack([torch.randn(V, 4, 256, 256, generator=torch.Generator().manual_seed(sd))
                                                for sd in range(B)]).to(dev))
        res["stage_s_per_scene"][vs] = t / B
        res.setdefault("stage_s_per_batch", {})[vs] = t
        res.setdefault("setup_s_per_batch", {})[vs] = t_setup
        res.setdefault("seeded_noise_s_per_batch", {})[vs] = t_noise
        res.setdefault("views", {})[vs] = V

    # ---- the 128^2 pipeline's step times
    fw_u = frameworks.ClassifierFreeGuidance(net("L", 1234), timesteps=1000, beta_schedule="linear")
    fw_c = frameworks.InpaintCFG(net("Lc", 4321), timesteps=1000, beta_schedule="linear")
    w = DeviceWarp(B, image_size=128, ssaa=3, max_views=2)
    src = torch.from_numpy(np.stack([synth_rgbd(rng).transpose(2, 0, 1) * 2 - 1 for _ in range(B)])).float().to(dev)
    w.add_view(src, views[0], **WARP_KW)
    c7 = w.aggregate(views[1], **WARP_KW)
    yc = c7[:, 0:4] * 2 - 1
    ckw = dict(y=yc, mask=c7[:, 4:5], mask_rgb=c7[:, 5:6], replace_rgb=(0.1, yc[:, :3], c7[:, 5:6]),
               replace_depth=(0.2, yc[:, 3:], c7[:, 4:5]), constrain_depth=(0.5, c7[:, 6:7] * 2 - 1))
    k = 20
    su, sc = samplers.DdimSampler(fw_u), samplers.DdimSampler(fw_c)
    ru = lambda: su.sample(B, classes=classes, steps=k, strength=0.5, verbose=False)
    rc = lambda: sc.sample(B, classes=classes, steps=k, strength=0.5, verbose=False, **ckw)
    ru(); rc()
    t_u = timed(ru)[0] / k
    t_c = timed(rc)[0] / k
    res["lowres_step_ms"] = {"uncond": 1e3 * t_u, "cond": 1e3 * t_c, "warp128_per_view": warp128}
    res["lowres_s_per_scene"] = {vs: (1000 * t_u + (V - 1) * (50 * t_c + warp128 / 1e3)) / B for vs, V in res["views"].items()}
    res["estimate_3x9_s_per_batch"] = 27 * 50 * 32.7e-3        # the estimate from the config-5 step time, not a measurement
    print(f"[bench_sr] card: {res['card']}")
    print(f"[bench_sr] SR step (batch {B}, CFG): {res['sr_step_ms']:.2f} ms; warp at 256^2: {res['warp_ms_per_view']:.2f} ms / view "
          f"(128^2: {warp128:.2f})")
    for vs, V in res["views"].items():
        t_steps = V * steps * res["sr_step_ms"] / 1e3
        t_warps = (V - 1) * res["warp_ms_per_view"] / 1e3
        print(f"[bench_sr] {vs}: {res['stage_s_per_batch'][vs]:.2f} s / batch = steps {t_steps:.2f} s + warps {t_warps:.2f} s + seeded "
              f"x_T {res['seeded_noise_s_per_batch'][vs]:.2f} s + rest {res['stage_s_per_batch'][vs] - t_steps - t_warps - res['seeded_noise_s_per_batch'][vs]:.2f} s; "
              f"set-up run (1 step / view, not in the stage time) {res['setup_s_per_batch'][vs]:.2f} s")
        print(f"[bench_sr] {vs} ({V} views, {steps} steps): stage {res['stage_s_per_scene'][vs]:.2f} s / scene "
              f"({res['stage_s_per_scene'][vs] * B:.1f} s / batch of {B}); 128^2 pipeline {res['lowres_s_per_scene'][vs]:.2f} s / scene "
              f"(computed from step times)")
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

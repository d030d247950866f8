"""The fp8 (e4m3) precision mode of the ResBlock convs against fp16, in one run.  Prints one JSON line.

    python tools/bench_fp8.py [--steps K] [--warmup W] [--reps R] [--no-distance]

per_shape    the conv shapes of tools/bench_conv.py at batch 32 (the 3x3 ones: the convs fp8 applies to), kernel ms of the
             fp16 kernel (ivid_op_conv2d) and the e4m3 kernel (ivid_op_conv2d_e4m3) from torch.profiler, each in a run of its
             own, with algorithmic TFLOP/s (2 M Cout K, real channels).
per_step     ms per denoising step of bench.py's config 2 (large model, DDPM step, batch 16, CFG) and config 5 (SR model,
             DDIM step, batch 8), networks built as bench.py builds them, fp16 and fp8 alternated on the same network
             (fp16, fp8, fp16, fp8), CUDA events around K steps after W warm-up steps; then one profiled step per precision
             with the conv_gemm and gn_apply family times of the plan's roofline profile.
distance     relative L2 between the fp8 and fp16 samples from the same x_T on config 2's network (synthetic weights, batch
             16, guidance 0.5): DPM-Solver++ 25 steps, DDIM 50 steps, DDPM 1000 steps.  Drift on random weights, not image
             quality.
The card's name, power limit and max SM clock are read in the same run.  Needs a GPU: there is no fallback."""
import argparse
import ctypes
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch                                      # noqa: E402

import bench                                      # noqa: E402
import bench_conv                                 # noqa: E402
from ivid_b200 import _lib                        # noqa: E402


def per_shape(reps, warmup):
    L = _lib.lib()
    stream = _lib.cur_stream()
    N = bench_conv.N
    rows = []
    for tag, H, Cin, Cout, k, Cin2, out16, residual in bench_conv.SHAPES:
        if k != 3:
            continue
        W = H
        g = torch.Generator(device="cuda").manual_seed(H * Cin + Cout)
        x = torch.randn(N, H, W, Cin, device="cuda", generator=g)
        x16 = x.half()
        x8 = x.clamp(-448, 448).to(torch.float8_e4m3fn)
        x2 = torch.randn(N, H, W, Cin2, device="cuda", generator=g).half() if Cin2 else None
        w = (torch.randn(Cout, Cin, k, k, generator=torch.Generator().manual_seed(Cout)) / math.sqrt(Cin * k * k)).contiguous()
        w2 = (torch.randn(Cout, Cin2) / math.sqrt(max(Cin2, 1))).contiguous() if Cin2 else None
        b = torch.zeros(Cout)
        res = torch.randn(N, H, W, Cout, device="cuda", generator=g) if residual else None
        out = torch.empty(N, H, W, Cout, device="cuda", dtype=torch.float16 if out16 else torch.float32)
        e = ctypes.c_int()
        calls = {
            "fp16": lambda: _lib.check(L.ivid_op_conv2d(_lib.ptr(x16), N, H, W, Cin, _lib.ptr(w), _lib.ptr(b), Cout, k, _lib.ptr(x2),
                                                        Cin2, _lib.ptr(w2), _lib.ptr(b if Cin2 else None), _lib.ptr(res),
                                                        _lib.ptr(out), 1 if out16 else 0, stream)),
            "e4m3": lambda: _lib.check(L.ivid_op_conv2d_e4m3(_lib.ptr(x8), N, H, W, Cin, _lib.ptr(w), _lib.ptr(b), Cout, k,
                                                             _lib.ptr(x2), Cin2, _lib.ptr(w2), _lib.ptr(b if Cin2 else None),
                                                             _lib.ptr(res), _lib.ptr(out), 1 if out16 else 0, ctypes.byref(e),
                                                             stream)),
        }
        flop = 2.0 * N * H * W * Cout * (k * k * Cin + Cin2)
        row = dict(shape=tag)
        for name, call in calls.items():
            for _ in range(warmup):
                call()
            ms = bench_conv._kernel_ms(call, reps)
            row[f"{name}_ms"] = round(ms, 4)
            row[f"{name}_tflops"] = round(flop / ms / 1e9, 1)
        row["speedup"] = round(row["fp16_ms"] / row["e4m3_ms"], 3)
        rows.append(row)
    return rows


def _families(net, step):
    L = _lib.lib()
    _lib.check(L.ivid_unet_profile_begin(net._handle))
    step()
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(L.ivid_unet_profile_end(net._handle, buf, len(buf)))
    fam = json.loads(buf.value.decode())
    keep = {k: round(v["ms"], 3) for k, v in fam.items() if k.startswith(("conv_gemm", "gn_apply"))}
    keep["conv_gemm_total"] = round(sum(v["ms"] for k, v in fam.items() if k.startswith("conv_gemm")), 3)
    return keep


def per_step(config, steps, warmup):
    import ivid_b200.backbones as backbones
    import ivid_b200.frameworks as frameworks
    import ivid_b200.samplers as samplers
    from oracle import unet_ref
    wl = bench.WORKLOADS[config]
    B = wl["batch"]
    key = wl["uncond"] or wl["cond"]
    cfg = bench.MODELS[key]
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234 if wl["uncond"] else 4321))
    net = net.cuda()
    gen = torch.Generator().manual_seed(1000)
    classes = (torch.arange(B) % 1000).cuda()
    S = cfg["image_size"]
    x = torch.randn(B, 4, S, S, generator=gen).cuda()
    kw = {"strength": bench.GUIDANCE}
    if config == 2:
        s = samplers.DdpmSampler(frameworks.ClassifierFreeGuidance(net, timesteps=1000, beta_schedule="linear", p_uncond=0.1))
        step = lambda xc, i: s._native_step(xc, (bench.DENOISE_STEPS - 1 - i) % bench.DENOISE_STEPS, 0, classes, False, 0.0, kw,
                                            None, None).pred_x_prev
    else:
        s = samplers.DdimSampler(frameworks.SuperResCFG(net, timesteps=1000, beta_schedule="linear"))
        ckw = dict(kw, y=torch.randn(B, 4, S // 2, S // 2, generator=gen).cuda())
        step = lambda xc, i: s._native_step(xc, 1000 - 20 * (i % 50), 980 - 20 * (i % 50), classes, False, 0.0, ckw, None,
                                            None).pred_x_prev
    out = {"ms_per_step": {"fp16": [], "fp8": []}}
    for prec in ("fp16", "fp8", "fp16", "fp8"):
        net.set_precision(prec)
        xc = x
        for i in range(warmup):
            xc = step(xc, i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            xc = step(xc, warmup + i)
        e1.record()
        torch.cuda.synchronize()
        out["ms_per_step"][prec].append(round(e0.elapsed_time(e1) / steps, 3))
    for prec in ("fp16", "fp8"):
        net.set_precision(prec)
        step(x, 0)
        out[f"families_{prec}_ms"] = _families(net, lambda: step(x, 1))
    return out


def distance():
    import ivid_b200.backbones as backbones
    import ivid_b200.frameworks as frameworks
    import ivid_b200.samplers as samplers
    from oracle import unet_ref
    cfg = bench.MODELS["L"]
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=1234))
    net = net.cuda()
    fw = frameworks.ClassifierFreeGuidance(net, timesteps=1000, beta_schedule="linear", p_uncond=0.1)
    B = 16
    x = torch.randn(B, 4, 128, 128, generator=torch.Generator().manual_seed(5)).cuda()
    classes = (torch.arange(B) % 1000).cuda()
    runs = {"dpmpp_25": (samplers.DpmSolverSampler, dict(steps=25)), "ddim_50": (samplers.DdimSampler, dict(steps=50)),
            "ddpm_1000": (samplers.DdpmSampler, {})}
    res = {}
    for name, (S, kw) in runs.items():
        outs = {}
        for prec in ("fp16", "fp8"):
            net.set_precision(prec)
            torch.manual_seed(77)
            outs[prec] = S(fw).sample(B, noise=x, classes=classes, strength=bench.GUIDANCE, verbose=False, **kw).samples.double()
            torch.cuda.synchronize()
        d = float((outs["fp8"] - outs["fp16"]).norm() / outs["fp16"].norm())
        res[name] = dict(rel_l2_fp8_vs_fp16=round(d, 5), finite=bool(torch.isfinite(outs["fp8"]).all()))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-distance", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 needs a CUDA device")
    result = dict(bench="fp8", card=bench_conv._card(), per_shape=per_shape(a.reps, 3),
                  per_step={f"config{c}": per_step(c, a.steps, a.warmup) for c in (2, 5)})
    if not a.no_distance:
        result["distance_config2_b16_g0.5"] = distance()
    print(json.dumps(result))


if __name__ == "__main__":
    main()

"""Micro-benchmark of the implicit-GEMM conv kernel (conv_gemm_kernel<BN>) at the conv shapes of the large model
(bench.py config 2) at batch 32.  Prints one JSON line.

    python tools/bench_conv.py [--reps R] [--warmup W]

kernel_ms: device time of the conv kernel per call (torch.profiler, CUDA activity, only the kernels whose name contains
`conv_gemm`), warm, in a run of its own.  The C entry point (ivid_op_conv2d) packs the weights on the host and copies them
to the device on every call; the profiler separates that from the kernel.  TFLOP/s are algorithmic, 2 M Cout K with the
real channel counts.  l2_smem_TBs is the operand traffic the tiles load, over kernel time.  Every CTA (128 pixels x BN
columns) loads one BN x 64 weight box (BN * 128 B) per k-block.  Per-tap segments (k_order "tap"): one 128 x 64 activation
box (16 KB) per k-block.  Slab segments (k_order "slab", the 3x3 segments of one-sample tiles with TW >= 8): one
TW x (TH + 2) x 64 slab per (chunk, dx), serving the three dy k-blocks, so a 3x3 segment of `chunks` chunks loads
chunks * 3 * TW * (TH + 2) * 128 B of activations; its 1x1 skip segment still loads 16 KB per k-block.  Needs a GPU: there
is no fallback."""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch                                      # noqa: E402
from torch.profiler import ProfilerActivity, profile   # noqa: E402

from ivid_b200 import _lib                        # noqa: E402

N = 32
# tag, H (= W), Cin, Cout, k, Cin2 (1x1 skip segment), out_fp16, residual
SHAPES = [
    ("128^2 3x3 256->256, fp16 out", 128, 256, 256, 3, 0, True, False),
    ("128^2 3x3 256 + 1x1 skip 512 -> 256, fp32 out", 128, 256, 256, 3, 512, False, False),
    ("128^2 3x3 256->256, residual, fp32 out", 128, 256, 256, 3, 0, False, True),
    ("64^2 3x3 256->256", 64, 256, 256, 3, 0, False, False),
    ("32^2 3x3 512->512", 32, 512, 512, 3, 0, False, False),
    ("16^2 3x3 768->768", 16, 768, 768, 3, 0, False, False),
    ("8^2 3x3 1024->1024", 8, 1024, 1024, 3, 0, False, False),
    ("32^2 1x1 qkv 512->1536, fp16 out", 32, 512, 1536, 1, 0, True, False),
]


def _kernel_ms(fn, reps):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "conv_gemm" in e.name]
    assert len(ev) == reps, f"expected {reps} conv kernels in the trace, found {len(ev)}"
    return sum(e.device_time for e in ev) / 1e3 / reps


def _card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def _tile_bytes(H, W, Cin, Cout, k, Cin2):
    tw, th, tn, fused = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.lib().ivid_conv_tile(H, W, ctypes.byref(tw), ctypes.byref(th), ctypes.byref(tn), ctypes.byref(fused)))
    tw, th, tn = tw.value, th.value, tn.value
    cout_pad = -(-Cout // 64) * 64
    bn = 128 if cout_pad % 128 == 0 else 64
    ctas = math.ceil(N / tn) * (H // th) * (W // tw) * (cout_pad // bn)
    chunks, chunks2 = math.ceil(Cin / 64), math.ceil(Cin2 / 64)
    kblocks = k * k * chunks + chunks2
    slab = k == 3 and tn == 1 and tw >= 8              # conv_launch_create's rule
    act = chunks * 3 * tw * (th + 2) * 128 + chunks2 * 128 * 64 * 2 if slab else kblocks * 128 * 64 * 2
    return ctas, kblocks, slab, ctas * (act + kblocks * bn * 64 * 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv needs a CUDA device")
    L = _lib.lib()
    stream = _lib.cur_stream()
    rows = []
    for tag, H, Cin, Cout, k, Cin2, out16, residual in SHAPES:
        W = H
        g = torch.Generator(device="cuda").manual_seed(H * Cin + Cout)
        x = torch.randn(N, H, W, Cin, device="cuda", generator=g).half()
        x2 = torch.randn(N, H, W, Cin2, device="cuda", generator=g).half() if Cin2 else None
        w = (torch.randn(Cout, Cin, k, k, generator=torch.Generator().manual_seed(Cout)) / math.sqrt(Cin * k * k)).contiguous()
        w2 = (torch.randn(Cout, Cin2) / math.sqrt(max(Cin2, 1))).contiguous() if Cin2 else None
        b = torch.zeros(Cout)
        res = torch.randn(N, H, W, Cout, device="cuda", generator=g) if residual else None
        out = torch.empty(N, H, W, Cout, device="cuda", dtype=torch.float16 if out16 else torch.float32)
        call = lambda: _lib.check(L.ivid_op_conv2d(_lib.ptr(x), N, H, W, Cin, _lib.ptr(w), _lib.ptr(b), Cout, k,
                                                   _lib.ptr(x2), Cin2, _lib.ptr(w2), _lib.ptr(b if Cin2 else None),
                                                   _lib.ptr(res), _lib.ptr(out), 1 if out16 else 0, stream))
        for _ in range(a.warmup):
            call()
        ms = _kernel_ms(call, a.reps)
        flop = 2.0 * N * H * W * Cout * (k * k * Cin + Cin2)
        ctas, kblocks, slab, tile_bytes = _tile_bytes(H, W, Cin, Cout, k, Cin2)
        rows.append(dict(shape=tag, ctas=ctas, k_blocks=kblocks, k_order="slab" if slab else "tap", kernel_ms=round(ms, 4),
                         tflops=round(flop / ms / 1e9, 1), l2_smem_TBs=round(tile_bytes / ms / 1e9, 2)))
    print(json.dumps(dict(bench="conv", batch=N, card=_card(), reps=a.reps, rows=rows)))


if __name__ == "__main__":
    main()

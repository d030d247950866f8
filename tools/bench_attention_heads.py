"""Micro-benchmark of ivid_op_attention_heads (attention_kernel at d = 64, attention_hd_kernel otherwise) at user-sized shapes,
with torch.nn.functional.scaled_dot_product_attention on the same fp16 data as a reference point.  Prints one JSON line.

    python tools/bench_attention_heads.py [--reps R]

kernel_ms: device time of the kernels per call (torch.profiler, CUDA activity), warm.  call_ms: CUDA events around R back-to-back
calls of the C entry point, which also builds the launch (tensor maps) and synchronises each time.  TFLOP/s are algorithmic,
4 N T^2 C (the count the UNet plan tags attention with); the sliced path (d > 256) executes more (see attention_hd.cuh).
Needs a GPU: there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch                                      # noqa: E402
import torch.nn.functional as F                   # noqa: E402
from torch.profiler import ProfilerActivity, profile   # noqa: E402

from ivid_b200 import _lib                        # noqa: E402

SHAPES = [(32, 1024, 512, d) for d in (64, 128, 256, 512)] + [(32, 256, 768, d) for d in (64, 192, 768)] + \
         [(8, 4096, 256, d) for d in (64, 128, 256)]


def _kernel_ms(fn, reps):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    return us / 1e3 / reps


def _events_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def _card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention_heads needs a CUDA device")
    L = _lib.lib()
    stream = _lib.cur_stream()
    rows = []
    for N, T, C, d in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(N * T + d)
        qkv = torch.randn(N, T, 3 * C, device="cuda", generator=g).half()       # [N][T][3C], head-major q|k|v
        out = torch.empty(N, T, C, device="cuda", dtype=torch.float16)
        ours = lambda: _lib.check(L.ivid_op_attention_heads(_lib.ptr(qkv), N, T, C, d, _lib.ptr(out), stream))
        h = C // d
        q, k, v = (t.permute(0, 2, 1, 3).contiguous() for t in qkv.view(N, T, h, 3 * d).split(d, dim=-1))   # [N][h][T][d]
        sdpa = lambda: F.scaled_dot_product_attention(q, k, v)
        for _ in range(a.warmup):
            ours(); sdpa()
        flop = 4.0 * N * T * T * C
        k_ms = _kernel_ms(ours, a.reps)
        s_ms = _kernel_ms(sdpa, a.reps)
        rows.append(dict(N=N, T=T, C=C, d=d, heads=h, kernel_ms=round(k_ms, 4), tflops=round(flop / k_ms / 1e9, 1),
                         call_ms=round(_events_ms(ours, a.reps), 4),
                         sdpa_kernel_ms=round(s_ms, 4), sdpa_tflops=round(flop / s_ms / 1e9, 1),
                         sdpa_max_abs_diff=float((out.view(N, T, h, d).permute(0, 2, 1, 3).float() - sdpa().float()).abs().max())))
    print(json.dumps(dict(bench="attention_heads", card=_card(), reps=a.reps, rows=rows)))


if __name__ == "__main__":
    main()

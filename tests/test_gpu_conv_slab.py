"""GPU: the 3x3 conv's slab K order against a float64 conv of the same fp16 operands.

At tiles of one sample with TW >= 8 the conv kernel loads one (TH + 2)-row activation slab per (64-channel chunk, dx) and
reads the three dy taps from it at row offsets 0, TW and 2 TW; K then runs chunk slow, dx, dy fast.  These cases cover each
level class that takes that path (TW = 16 and TW = 8 slabs, one-row shifts of two and one 1024-byte swizzle atoms), a 3x3
segment followed by 1x1 skip segments over two tensors, widths that are not multiples of 64, non-square inputs, and the
TN = 2 levels that keep one activation box per tap.

Bar, per output element: the kernel reads fp16 operands exactly and sums K = 9 * C0p + C1p + C2p products (padded channel
counts) into an fp32 accumulator, then adds the fp32 bias.  Each of those K + 1 additions can lose up to one fp32 ulp of a
running sum bounded by S = sum |a w| + |b| if the tensor cores truncate rather than round, so |y - y64| <= (K + 1) 2^-23 S.
A wrong tap, row shift or weight column moves an output by a sizeable fraction of S and fails it by orders of magnitude."""
import math

import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
from ivid_b200 import _lib

pytestmark = pytest.mark.gpu

U23 = 2.0 ** -23

# N, H, W, C0 (3x3), Cout, C1, C2 (1x1 skip over [x1 | x2]), expected tile TWxTHxTN
CASES = [
    (1, 128, 128, 128, 128, 0, 0, "16x8x1"),        # 128^2 level
    (2, 64, 64, 256, 128, 0, 0, "16x8x1"),          # 64^2
    (2, 32, 32, 512, 128, 0, 0, "16x8x1"),          # 32^2
    (2, 16, 16, 768, 256, 0, 0, "16x8x1"),          # 16^2
    (2, 32, 32, 128, 128, 96, 160, "16x8x1"),       # up-path conv2: 3x3 + 1x1 skip over two tensors
    (2, 64, 64, 96, 160, 0, 0, "16x8x1"),           # widths that are not multiples of 64
    (2, 32, 32, 160, 96, 0, 0, "16x8x1"),
    (2, 32, 48, 128, 128, 0, 0, "16x8x1"),          # non-square, TW = 16 slab
    (3, 16, 8, 128, 128, 0, 0, "8x16x1"),           # TW = 8 slab: the row shift is exactly one swizzle atom
    (3, 16, 8, 96, 64, 64, 0, "8x16x1"),
    (3, 8, 8, 256, 128, 0, 0, "8x8x2"),             # TN = 2: per-tap boxes, batch tail
    (3, 24, 40, 128, 160, 0, 0, "8x8x2"),
]


def _case_id(c):
    N, H, W, C0, Cout, C1, C2, tile = c
    skip = f"+skip{C1}" + (f"|{C2}" if C2 else "") if C1 else ""
    return f"{tile}-{H}x{W}-N{N}-{C0}{skip}to{Cout}"


def _gen(tag):
    return torch.Generator().manual_seed(sum(ord(ch) * (i + 1) for i, ch in enumerate(tag)) % 2**31)


def _pad64(c):
    return -(-c // 64) * 64


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_conv_slab_vs_float64(case):
    N, H, W, C0, Cout, C1, C2, tile = case
    tag = _case_id(case)
    TW, TH, TN, _ = G.conv_tile(H, W)
    assert f"{TW}x{TH}x{TN}" == tile, f"{H}x{W} runs tile {TW}x{TH}x{TN}, not {tile}"
    g = _gen(tag)
    act = torch.randn(N, H, W, C0, generator=g).half()
    w = torch.randn(Cout, C0, 3, 3, generator=g) / math.sqrt(9 * C0)
    b = torch.randn(Cout, generator=g) * 0.5
    x1 = torch.randn(N, H, W, C1, generator=g).half() if C1 else None
    x2 = torch.randn(N, H, W, C2, generator=g).half() if C2 else None
    ws = torch.randn(Cout, C1 + C2, generator=g) / math.sqrt(C1 + C2) if C1 else None
    bs = torch.randn(Cout, generator=g) * 0.5 if C1 else None
    out = G.nan_like_buffer((N, H, W, Cout), torch.float32)
    rc, _ = G.conv_ex(act.cuda(), w, b, 3, out, 0, act1=x1.cuda() if C1 else None, act2=x2.cuda() if C2 else None,
                      wskip=ws, bskip=bs)
    _lib.check(rc)
    got = out.cpu().double()
    assert bool(torch.isfinite(got).all()), f"{tag}: an output was not written"

    a64, w64 = act.double().permute(0, 3, 1, 2), w.half().double()
    want = F.conv2d(a64, w64, b.double(), padding=1)
    S = F.conv2d(a64.abs(), w64.abs(), b.double().abs(), padding=1)
    if C1:
        x = torch.cat([x1, x2], -1) if C2 else x1
        x64, ws64 = x.double().permute(0, 3, 1, 2), ws.half().double()[:, :, None, None]
        want = want + F.conv2d(x64, ws64, bs.double())
        S = S + F.conv2d(x64.abs(), ws64.abs(), bs.double().abs())
    want, S = want.permute(0, 2, 3, 1), S.permute(0, 2, 3, 1)
    K = 9 * _pad64(C0) + _pad64(C1) + _pad64(C2)
    ratio = float(((got - want).abs() / ((K + 1) * U23 * S)).max())
    G.report(f"slab {tag}", got, want)
    print(f"[slab] {tag}: max |err| / bound {ratio:.3e}")
    assert ratio <= 1.0, f"{tag}: error {ratio:.3g}x the fp32-accumulation bound"

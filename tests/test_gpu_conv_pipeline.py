"""GPU parity of the conv kernel's operand pipeline at its edges: the producer warp runs STAGES k-blocks ahead of the two
consumer warpgroups, which keep one wgmma group in flight and release a ring slot one k-block late.  Each case is held to
the bars of test_gpu_ops.py (2e-5 relative L2 against fp32 math on the same fp16-rounded operands, 5e-4 for an fp16
output) and must be bitwise reproducible run to run.  The three-segment K walk (3x3 conv + two 1x1 skip segments of the
up path) runs inside the UNet and is covered by its parity tests."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gpu_util as G

pytestmark = pytest.mark.gpu


def _t(rng, *shape, scale=1.0):
    return torch.from_numpy((rng.standard_normal(shape) * scale).astype(np.float32))


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().cuda()


def _check(tag, N, H, W, Cin, Cout, k, seed, Cin2=0, out_fp16=False, residual=False):
    rng = np.random.default_rng(seed)
    x = _t(rng, N, Cin, H, W).half()
    w = _t(rng, Cout, Cin, k, k, scale=1 / math.sqrt(Cin * k * k))
    b = _t(rng, Cout, scale=0.1)
    ref = F.conv2d(x.float(), w.half().float(), b, padding=k // 2)
    kw = {"out_fp16": out_fp16}
    if Cin2:
        x2 = _t(rng, N, Cin2, H, W).half()
        ws = _t(rng, Cout, Cin2, 1, 1, scale=1 / math.sqrt(Cin2)); bs = _t(rng, Cout, scale=0.1)
        ref = ref + F.conv2d(x2.float(), ws.half().float(), bs)
        kw.update(act2=_nhwc(x2), w2=ws, b2=bs)
    if residual:
        res = _t(rng, N, Cout, H, W)
        ref = ref + res
        kw["residual"] = _nhwc(res)
    xn = _nhwc(x)
    out = G.conv2d(xn, w, b, k, **kw)
    again = G.conv2d(xn, w, b, k, **kw)
    assert torch.equal(out, again), f"{tag}: not reproducible run to run"
    r = G.report(tag, out.float().permute(0, 3, 1, 2), ref)
    assert r < (5e-4 if out_fp16 else 2e-5)


def test_conv_single_k_block():
    """1x1 over 64 channels: one k-block, fewer than the ring's stages; the only release is the one after the loop."""
    _check("1x1 64->128, one k-block", 2, 16, 16, 64, 128, 1, 11)
    _check("1x1 64->64, one k-block, fp16 out", 3, 8, 8, 64, 64, 1, 12, out_fp16=True)


def test_conv_two_k_blocks_and_uneven_segments():
    """Two k-blocks (one fewer than the stages), and a 3x3 segment of 3 chunks followed by a 1x1 segment of 5."""
    _check("1x1 128->256, two k-blocks", 2, 16, 16, 128, 256, 1, 21)
    _check("3x3 192 + 1x1 320 -> 256, residual", 2, 32, 32, 192, 256, 3, 22, Cin2=320, residual=True)


@pytest.mark.parametrize("Cout", [256, 384])
def test_conv_even_and_odd_column_blocks(Cout):
    """Two and three 128-wide column blocks over the same pixel tiles."""
    _check(f"3x3 256->{Cout}", 2, 32, 32, 256, Cout, 3, 31)


def test_conv_batch_tail_with_several_samples_per_tile():
    """8x8 images: TN = 2 samples per 128-pixel tile, and an odd batch leaves the last tile half empty."""
    _check("8x8 N5 3x3 512->512", 5, 8, 8, 512, 512, 3, 41)
    _check("4x4 N3 3x3 256->256 + skip, fp16 out", 3, 4, 4, 256, 256, 3, 42, Cin2=128, out_fp16=True)


def test_conv_grid_not_a_multiple_of_resident_ctas():
    """7 x 64 x 64 pixels and two column blocks: 448 CTAs, not a whole number of waves of two CTAs per SM."""
    _check("64x64 N7 3x3 256->256 + residual", 7, 64, 64, 256, 256, 3, 51, residual=True)

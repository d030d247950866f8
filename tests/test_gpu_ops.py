"""GPU parity of the individual sm_90a kernels against fp32 torch on the CPU (through the op-level C ABI).

Tolerances: tensor-core operands are fp16 (10-bit mantissa, like the TF32 path the reference's cuDNN convs took on
A100) with fp32 accumulation, so a single conv/GEMM is compared at 2e-3 relative L2 against the fp32 result of the SAME
fp16-rounded operands at 2e-5 (accumulation-order only)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gpu_util as G

pytestmark = pytest.mark.gpu


def _rng(seed):
    return np.random.default_rng(seed)


def _t(rng, *shape, scale=1.0):
    return torch.from_numpy((rng.standard_normal(shape) * scale).astype(np.float32))


CONV_CASES = [
    # N, H, W, Cin, Cout, k
    (2, 16, 16, 64, 64, 3),
    (1, 32, 32, 128, 256, 3),
    (3, 8, 8, 256, 128, 3),      # TN=2 tiles with odd batch (batch tail masked)
    (2, 16, 16, 192, 384, 1),    # 1x1, BN=128
    (1, 4, 4, 64, 64, 3),        # tiny spatial: TN=8 with N=1
    (2, 64, 64, 64, 16, 3),      # narrow Cout (BN=16 path, output head shape)
    (1, 128, 128, 256, 256, 3),  # the dominant shape of the large model
    (2, 64, 64, 64, 768, 3),     # 6 column blocks, more than one wave of resident CTAs
    # low-resolution levels: several samples per pixel tile, several column blocks per tile
    (4, 8, 8, 256, 512, 3),      # TN=2, 4 column blocks
    (8, 8, 8, 128, 256, 3),      # TN=2, 2 column blocks
    (32, 8, 8, 1024, 1024, 3),   # the 8x8 level of the large model at the benchmark batch: 16 K chunks per tap, 8 column blocks
    (6, 16, 16, 128, 384, 1),    # 1x1 on 16x16 images, 3 column blocks (odd)
    (4, 16, 16, 64, 640, 3),     # 5 column blocks (odd)
    (5, 32, 32, 192, 512, 3),    # odd batch, 3 channel chunks, 4 column blocks
    (13, 16, 16, 128, 768, 3),   # 16x16 images, odd batch of 13, 6 column blocks
]


@pytest.mark.parametrize("N,H,W,Cin,Cout,k", CONV_CASES)
@pytest.mark.parametrize("epilogue", ["default", "fp16_out", "residual", "skip"])
def test_conv_matches_torch(N, H, W, Cin, Cout, k, epilogue):
    """Every conv case through each epilogue / K path of the kernel: "default" = fp32 NHWC output, "fp16_out" = fp16 output,
    "residual" = fp32 identity residual added in the epilogue, "skip" = a 1x1 skip segment over a second tensor of Cin
    channels as extra K chunks (ResBlock tail)."""
    rng = _rng(hash((N, H, W, Cin, Cout, k)) % 2**31)
    x = _t(rng, N, Cin, H, W)
    w = _t(rng, Cout, Cin, k, k, scale=1 / math.sqrt(Cin * k * k))
    b = _t(rng, Cout, scale=0.1)
    xh = x.half()
    ref16 = F.conv2d(xh.float(), w.half().float(), b, padding=k // 2)       # same rounded operands, fp32 math
    ref32 = F.conv2d(x, w, b, padding=k // 2)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().cuda()
    kw = {}
    if epilogue == "fp16_out":
        kw["out_fp16"] = True
    elif epilogue == "residual":
        res = _t(rng, N, Cout, H, W)
        ref16 = ref16 + res; ref32 = ref32 + res
        kw["residual"] = nhwc(res)
    elif epilogue == "skip":
        x2 = _t(rng, N, Cin, H, W)
        ws = _t(rng, Cout, Cin, 1, 1, scale=1 / math.sqrt(Cin)); bs = _t(rng, Cout, scale=0.1)
        ref16 = ref16 + F.conv2d(x2.half().float(), ws.half().float(), bs)
        ref32 = ref32 + F.conv2d(x2, ws, bs)
        kw.update(act2=nhwc(x2.half()), w2=ws, b2=bs)
    out = G.conv2d(nhwc(xh), w, b, k, **kw)
    got = out.float().permute(0, 3, 1, 2).cpu()
    tag = f"conv N{N} {H}x{W} {Cin}->{Cout} k{k} {epilogue}"
    r16 = G.report(f"{tag} (vs fp16-rounded operands)", got, ref16)
    r32 = G.report(f"{tag} (vs fp32)", got, ref32)
    assert r16 < (5e-4 if epilogue == "fp16_out" else 2e-5)      # fp16 output: one rounding of the result
    assert r32 < 2e-3


def test_conv_skip_segment_residual_and_fp16_out():
    """out_layers conv + 1x1 skip conv as extra K slabs (ResBlock tail, adm.py:222), identity residual, fp16 output."""
    rng = _rng(5)
    N, H, W, C, Cx = 2, 16, 16, 128, 192
    a = _t(rng, N, C, H, W); x = _t(rng, N, Cx, H, W)
    w = _t(rng, C, C, 3, 3, scale=1 / math.sqrt(9 * C)); b = _t(rng, C, scale=0.1)
    ws = _t(rng, C, Cx, 1, 1, scale=1 / math.sqrt(Cx)); bs = _t(rng, C, scale=0.1)
    ref = F.conv2d(a.half().float(), w.half().float(), b, padding=1) + F.conv2d(x.half().float(), ws.half().float(), bs)
    out = G.conv2d(a.half().permute(0, 2, 3, 1).contiguous().cuda(), w, b, 3,
                   act2=x.half().permute(0, 2, 3, 1).contiguous().cuda(), w2=ws, b2=bs)
    assert G.report("conv3x3 + 1x1 skip segment", out.permute(0, 3, 1, 2), ref) < 2e-5
    res = _t(rng, N, C, H, W)
    ref2 = F.conv2d(a.half().float(), w.half().float(), b, padding=1) + res
    out2 = G.conv2d(a.half().permute(0, 2, 3, 1).contiguous().cuda(), w, b, 3, residual=res.permute(0, 2, 3, 1).contiguous().cuda())
    assert G.report("conv3x3 + identity residual", out2.permute(0, 3, 1, 2), ref2) < 2e-5
    out3 = G.conv2d(a.half().permute(0, 2, 3, 1).contiguous().cuda(), w, b, 3, out_fp16=True)
    assert G.report("conv3x3 fp16 out", out3.float().permute(0, 3, 1, 2), F.conv2d(a.half().float(), w.half().float(), b, padding=1)) < 5e-4


def test_conv_skip_segment_residual_and_fp16_out_4_column_blocks():
    """The paths of test_conv_skip_segment_residual_and_fp16_out on a layer of 4 column blocks and 128 pixel tiles: a 1x1
    skip segment over a second tensor (9-tap and 1-tap segments share the ring), the identity residual and the fp16 output."""
    rng = _rng(31)
    N, H, W, C, Cx = 4, 64, 64, 128, 192
    Co = 512
    a = _t(rng, N, C, H, W); x = _t(rng, N, Cx, H, W); res = _t(rng, N, Co, H, W)
    w = _t(rng, Co, C, 3, 3, scale=1 / math.sqrt(9 * C)); b = _t(rng, Co, scale=0.1)
    ws = _t(rng, Co, Cx, 1, 1, scale=1 / math.sqrt(Cx)); bs = _t(rng, Co, scale=0.1)
    base = F.conv2d(a.half().float(), w.half().float(), b, padding=1)
    skip = F.conv2d(x.half().float(), ws.half().float(), bs)
    an = a.half().permute(0, 2, 3, 1).contiguous().cuda()
    xn = x.half().permute(0, 2, 3, 1).contiguous().cuda()
    rn = res.permute(0, 2, 3, 1).contiguous().cuda()
    out = G.conv2d(an, w, b, 3, act2=xn, w2=ws, b2=bs)
    assert G.report("conv3x3 + 1x1 skip segment", out.permute(0, 3, 1, 2), base + skip) < 2e-5
    out2 = G.conv2d(an, w, b, 3, residual=rn)
    assert G.report("conv3x3 + identity residual", out2.permute(0, 3, 1, 2), base + res) < 2e-5
    out3 = G.conv2d(an, w, b, 3, out_fp16=True)
    assert G.report("conv3x3 fp16 out", out3.float().permute(0, 3, 1, 2), base) < 5e-4


def test_conv_low_resolution_residual_fp16_out_and_skip_segment():
    """An 8x8 layer (two samples per pixel tile, 4 column blocks) through the residual epilogue, the fp16-output epilogue and
    the 1x1 skip segment."""
    rng = _rng(21)
    N, H, W, C, Cx = 8, 8, 8, 512, 256
    a = _t(rng, N, C, H, W); x = _t(rng, N, Cx, H, W); res = _t(rng, N, C, H, W)
    w = _t(rng, C, C, 3, 3, scale=1 / math.sqrt(9 * C)); b = _t(rng, C, scale=0.1)
    ws = _t(rng, C, Cx, 1, 1, scale=1 / math.sqrt(Cx)); bs = _t(rng, C, scale=0.1)
    base = F.conv2d(a.half().float(), w.half().float(), b, padding=1)
    an = a.half().permute(0, 2, 3, 1).contiguous().cuda()
    out = G.conv2d(an, w, b, 3, residual=res.permute(0, 2, 3, 1).contiguous().cuda())
    assert G.report("8x8: conv3x3 + residual", out.permute(0, 3, 1, 2), base + res) < 2e-5
    out16 = G.conv2d(an, w, b, 3, out_fp16=True)
    assert G.report("8x8: conv3x3 fp16 out", out16.float().permute(0, 3, 1, 2), base) < 5e-4
    outs = G.conv2d(an, w, b, 3, act2=x.half().permute(0, 2, 3, 1).contiguous().cuda(), w2=ws, b2=bs)
    assert G.report("8x8: conv3x3 + 1x1 skip segment", outs.permute(0, 3, 1, 2),
                    base + F.conv2d(x.half().float(), ws.half().float(), bs)) < 2e-5


def test_conv_many_column_blocks_residual_and_fp16_out():
    """Layer with 768 output channels at 64x64 (6 column blocks, 384 tiles: more than one wave of resident CTAs on 132 SMs) through the
    residual epilogue and the fp16-output epilogue."""
    rng = _rng(11)
    N, H, W, Cin, C = 2, 64, 64, 64, 768
    a = _t(rng, N, Cin, H, W)
    w = _t(rng, C, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin)); b = _t(rng, C, scale=0.1)
    res = _t(rng, N, C, H, W)
    base = F.conv2d(a.half().float(), w.half().float(), b, padding=1)
    an = a.half().permute(0, 2, 3, 1).contiguous().cuda()
    out = G.conv2d(an, w, b, 3, residual=res.permute(0, 2, 3, 1).contiguous().cuda())
    assert G.report("768 columns: conv3x3 + residual", out.permute(0, 3, 1, 2), base + res) < 2e-5
    out16 = G.conv2d(an, w, b, 3, out_fp16=True)
    assert G.report("768 columns: conv3x3 fp16 out", out16.float().permute(0, 3, 1, 2), base) < 5e-4


@pytest.mark.parametrize("N,T,C", [(32, 256, 768), (32, 1024, 512), (8, 4096, 256)])
def test_attention_is_deterministic_under_load(N, T, C):
    """Same qkv, many launches with every SM busy: all outputs bitwise equal and equal to the fp32 reference within tolerance.
    Regression test for barrier-phase errors in the K / V ring (a wrong phase shows up as a few wrong rows in some launches)."""
    g = torch.Generator().manual_seed(T)
    qkv = (torch.randn(N, T, 3 * C, generator=g) * 1.5).half().cuda()
    ref = G.attention(qkv, C).clone()
    iters = 400 if T < 4096 else 60
    bad = 0
    for _ in range(iters):
        bad += 0 if torch.equal(G.attention(qkv, C), ref) else 1
    assert bad == 0, f"{bad} of {iters} launches differ from the first"
    # and the first one is right (one sample is enough: the op parity test covers the numerics)
    q, k, v = qkv[:1].float().cpu().reshape(1, T, C // 64, 3, 64).permute(3, 0, 2, 1, 4)
    w = torch.softmax(torch.einsum("bhtd,bhsd->bhts", q, k) / 8.0, dim=-1)
    want = torch.einsum("bhts,bhsd->bhtd", w, v).permute(0, 2, 1, 3).reshape(1, T, C)
    assert G.report(f"attention T={T} under load", ref[:1].float().cpu(), want) < 2e-3


GN_CASES = [
    # N, H, W, C0, C1, groups, silu, mode, film
    (2, 16, 16, 64, 0, 32, True, 0, False),
    (2, 16, 16, 128, 0, 32, True, 0, True),
    (3, 8, 8, 1024, 768, 32, True, 0, False),    # 1792 = 1024 (+) 768: 56 channels / group straddles the seam
    (2, 16, 16, 512, 256, 32, True, 0, False),   # 768 = 512 (+) 256: 24 / group straddles
    (2, 16, 16, 128, 0, 32, True, 1, False),     # nearest 2x upsample after GN+SiLU
    (2, 16, 16, 128, 0, 32, True, 2, False),     # 2x2 average pool after GN+SiLU
    (1, 32, 32, 512, 0, 32, False, 0, False),    # attention norm (no SiLU)
]


@pytest.mark.parametrize("N,H,W,C0,C1,groups,silu,mode,film", GN_CASES)
def test_group_norm_matches_torch(N, H, W, C0, C1, groups, silu, mode, film):
    rng = _rng(hash((N, H, W, C0, C1, mode)) % 2**31)
    C = C0 + C1
    x0 = _t(rng, N, C0, H, W) * 1.7 + 0.3
    x1 = (_t(rng, N, C1, H, W) * 0.6 - 0.2) if C1 else None
    gamma = 1 + 0.1 * _t(rng, C); beta = 0.1 * _t(rng, C)
    x = torch.cat([x0, x1], 1) if C1 else x0
    y = F.group_norm(x, groups, gamma, beta, 1e-5)
    fl = None
    if film:
        fl = 0.3 * _t(rng, N, 2 * C)
        y = y * (1 + fl[:, :C, None, None]) + fl[:, C:, None, None]
    if silu:
        y = F.silu(y)
    if mode == 1:
        y = F.interpolate(y, scale_factor=2, mode="nearest")
    elif mode == 2:
        y = F.avg_pool2d(y, 2)
    out = G.group_norm(x0.permute(0, 2, 3, 1).contiguous().cuda(), x1.permute(0, 2, 3, 1).contiguous().cuda() if C1 else None,
                       groups, gamma, beta, fl.cuda() if film else None, silu, mode)
    r = G.report(f"group_norm N{N} {H}x{W} C{C0}+{C1} silu{silu} mode{mode} film{film}", out.float().permute(0, 3, 1, 2), y)
    assert r < 6e-4     # output is rounded to fp16 (2^-11 relative)


@pytest.mark.parametrize("N,T,C", [(2, 64, 128), (1, 256, 192), (2, 1024, 128), (1, 4096, 64)])
def test_attention_matches_torch(N, T, C):
    rng = _rng(T + C)
    qkv = _t(rng, N, 3 * C, T)                     # reference layout [N, 3C, T]
    qh = qkv.half()
    heads = C // 64
    q, k, v = qh.float().reshape(N * heads, 3 * 64, T).split(64, dim=1)
    s = 1 / math.sqrt(math.sqrt(64))
    w = torch.softmax(torch.einsum("bct,bcs->bts", q * s, k * s), dim=-1)
    ref = torch.einsum("bts,bcs->bct", w, v).reshape(N, C, T)
    out = G.attention(qh.permute(0, 2, 1).contiguous().cuda(), C)     # [N, T, 3C]
    r = G.report(f"attention N{N} T{T} C{C}", out.float().permute(0, 2, 1), ref)
    assert r < 2e-3

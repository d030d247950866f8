"""GPU: the conv epilogue's fused outputs and the fp16-source GroupNorm apply against float64 references.

Every ResBlock runs conv_gemm_kernel, whose epilogue also accumulates the GroupNorm statistics of its output (and writes
the fp16 copy of a block output), and then gn_apply_h16_kernel on the fp16 tensor with those statistics.  These tests run
each half alone through ivid_op_conv2d_ex / ivid_op_group_norm_apply, which set exactly the ConvDesc / GnApplyDesc fields
the network sets, and compare with float64 computed on the CPU from the same rounded operands the kernels read.

Every output and statistics buffer is prefilled with NaN and holds one guard sample past N.  Every valid element must come
back finite and the guard must stay NaN: a write past the last pixel of the batch, or into the columns of a padded Cout
past the last channel, lands there."""
import math

import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
from ivid_b200 import _lib

pytestmark = pytest.mark.gpu

# A fused statistic passes each value through at most 12 fp32 roundings: two rows per lane, 3 shuffles, <= 8 warps, and the
# square.  12 * 2^-24 = 7.2e-7 bounds its relative error (sum: relative to sum |v|); the tests allow 1e-6.
GAMMA12 = 12 * 2.0 ** -24
STAT_BAR = 1e-6
# one conv at the bars of tests/test_gpu_ops.py (fp32 / fp16 output) and tests/test_gpu_fp8.py (e4m3 segment 0)
CONV_BAR = {"fp32": 2e-5, "fp16": 5e-4, "e4m3": 3e-3}


def _gen(tag):
    return torch.Generator().manual_seed(sum(ord(ch) * (i + 1) for i, ch in enumerate(tag)) % 2**31)


def _e4m3(t):
    return t.clamp(-448.0, 448.0).to(torch.float8_e4m3fn)


def _f64(t):
    return t.detach().cpu().double()


def _check_guard(buf, N, tag):
    b = buf.cpu()
    if b.dtype == torch.uint8:
        assert bool((b[N:] == 0x7F).all()), f"{tag}: written past sample N"
        assert not bool((b[:N] == 0x7F).any()), f"{tag}: an element was not written"
        return
    b = b.float()
    assert bool(torch.isnan(b[N:]).all()), f"{tag}: written past sample N"
    assert bool(torch.isfinite(b[:N]).all()), f"{tag}: an element was not written or is not finite"


def _check_stats(stats, vals, N, tag):
    """stats [N+1, C, 2] fp64 from the epilogue; vals [N, H, W, C] float64, the values the epilogue is specified to sum."""
    _check_guard(stats, N, f"{tag} statistics")
    st = stats[:N].to(vals.device)
    S, Q = st[..., 0], st[..., 1]
    S64, A64, Q64 = vals.sum((1, 2)), vals.abs().sum((1, 2)), (vals * vals).sum((1, 2))
    rs = float(((S - S64).abs() / A64).max())
    rq = float(((Q - Q64).abs() / Q64).max())
    print(f"[fused] {tag}: statistics |S - S64| / sum|v| max {rs:.2e}, |Q - Q64| / Q64 max {rq:.2e} (bar {STAT_BAR:.0e})")
    assert rs <= STAT_BAR and rq <= STAT_BAR, f"{tag}: fused statistics off"


def _ref_conv(act0, w0, b0, k, e4m3, e, act1=None, act2=None, wskip=None, bskip=None):
    """float64 NHWC conv of exactly the operands the kernel reads: fp16 (or e4m3 with weights e4m3(w * 2^e) * 2^-e)
    segment 0, fp16 skip weights (scaled by 2^e and back in e4m3 mode)."""
    a = act0.cpu().float().double().permute(0, 3, 1, 2)
    if e4m3:
        wq = _e4m3(w0 * 2.0 ** e).float().double() * 2.0 ** -e
    else:
        wq = w0.half().double()
    y = F.conv2d(a, wq, b0.double(), padding=k // 2)
    if act1 is not None:
        x = torch.cat([act1, act2], -1) if act2 is not None else act1
        ws = (wskip * 2.0 ** e).half().double() * 2.0 ** -e
        y = y + F.conv2d(_f64(x).permute(0, 3, 1, 2), ws[:, :, None, None], bskip.double())
    return y.permute(0, 2, 3, 1)


def _act(g, N, H, W, C, e4m3):
    a = torch.randn(N, H, W, C, generator=g)
    return (_e4m3(a * 1.5) if e4m3 else a.half()).cuda()


def _conv_weights(g, Cout, Cin, k):
    return torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k), torch.randn(Cout, generator=g) * 0.5


def _stats_buffer(N, C):
    st = G.nan_like_buffer((N + 1, C, 2), torch.float64)
    st[:N].zero_()                                   # the epilogue accumulates
    return st


# ----------------------------------------------------------------------------------------------------------------------
# a. fused statistics against the kernel's own output, at every tile class
# ----------------------------------------------------------------------------------------------------------------------
# tile TWxTHxTN, N, H, W, Cin, Cout, output form, e4m3 segment 0.  Forms: "res" fp32 + residual, "f16" fp16 output (the
# ResBlock hidden tensor), "copy" fp32 + the fp16 copy (block outputs).  Cout 96 / 160 / 40 pad to 128 / 192 / 48 (BN 128 /
# 64 / 16); 768 is six column blocks.  N = 3 at TN = 2 and N = 5, 6, 7 at TN = 4 leave a batch tail in the last tile.
STAT_CASES = [
    ("16x8x1", 2, 32, 32, 64, 96, "res", False),
    ("16x8x1", 1, 32, 32, 128, 160, "f16", False),
    ("16x8x1", 2, 48, 80, 64, 64, "copy", False),
    ("16x8x1", 2, 32, 32, 64, 768, "res", False),
    ("8x8x2", 3, 8, 8, 128, 40, "res", False),
    ("8x8x2", 3, 8, 8, 64, 96, "f16", False),
    ("8x8x2", 2, 24, 40, 64, 160, "copy", False),
    ("4x8x4", 5, 8, 4, 128, 128, "f16", False),
    ("4x8x4", 6, 8, 4, 64, 40, "res", False),
    ("4x8x4", 7, 8, 4, 64, 768, "copy", False),
    ("8x4x4", 7, 4, 8, 64, 96, "copy", False),
    ("8x4x4", 5, 4, 8, 128, 768, "f16", False),
    ("8x4x4", 6, 12, 8, 64, 160, "res", False),
    ("8x4x4", 4, 12, 8, 128, 128, "f16", False),
    ("16x8x1", 2, 32, 32, 128, 128, "f16", True),
    ("8x8x2", 3, 8, 8, 128, 40, "res", True),
    ("4x8x4", 5, 8, 4, 64, 96, "copy", True),
    ("8x4x4", 7, 12, 8, 256, 160, "f16", True),
]


def _case_id(c):
    tile, N, H, W, Cin, Cout, form, e4m3 = c
    return f"{tile}-{H}x{W}-N{N}-{Cin}to{Cout}-{form}" + ("-e4m3" if e4m3 else "")


@pytest.mark.parametrize("case", STAT_CASES, ids=[_case_id(c) for c in STAT_CASES])
def test_fused_statistics(case):
    tile, N, H, W, Cin, Cout, form, e4m3 = case
    tag = _case_id(case)
    TW, TH, TN, fused = G.conv_tile(H, W)
    assert fused and f"{TW}x{TH}x{TN}" == tile, f"{H}x{W} runs tile {TW}x{TH}x{TN}, not {tile}"
    g = _gen(tag)
    act = _act(g, N, H, W, Cin, e4m3)
    w, b = _conv_weights(g, Cout, Cin, 3)
    res = torch.randn(N, H, W, Cout, generator=g).cuda() if form == "res" else None
    out = G.nan_like_buffer((N + 1, H, W, Cout), torch.float16 if form == "f16" else torch.float32)
    out16 = G.nan_like_buffer((N + 1, H, W, Cout), torch.float16) if form == "copy" else None
    stats = _stats_buffer(N, Cout)
    rc, e = G.conv_ex(act, w, b, 3, out, 1 if form == "f16" else 0, e4m3=e4m3, residual=res, out16=out16, stats=stats)
    _lib.check(rc)
    _check_guard(out, N, tag)
    want = _ref_conv(act, w, b, 3, e4m3, e)
    if res is not None:
        want = want + _f64(res)
    got = _f64(out[:N])
    err = G.report(f"fused {tag} output", got, want)
    assert err < CONV_BAR["e4m3" if e4m3 else ("fp16" if form == "f16" else "fp32")]
    _check_stats(stats, got, N, tag)
    if out16 is not None:
        _check_guard(out16, N, f"{tag} fp16 copy")
        assert torch.equal(out16[:N].view(torch.int16), out[:N].half().view(torch.int16)), f"{tag}: fp16 copy != out.half()"


# ----------------------------------------------------------------------------------------------------------------------
# b. the epilogue's other forms
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(32, 16), (16, 48), (24, 24)])
def test_residual_through_nearest_upsample(H, W):
    """Up-path ResBlock output: conv + nearest-2x(residual [N, H/2, W/2, Cout]), with the fp16 copy and the statistics."""
    N, Cin, Cout = 3, 64, 128
    tag = f"residual_up {H}x{W}"
    g = _gen(tag)
    act = _act(g, N, H, W, Cin, False)
    w, b = _conv_weights(g, Cout, Cin, 3)
    res = torch.randn(N, H // 2, W // 2, Cout, generator=g)
    out = G.nan_like_buffer((N + 1, H, W, Cout), torch.float32)
    out16 = G.nan_like_buffer((N + 1, H, W, Cout), torch.float16)
    stats = _stats_buffer(N, Cout)
    rc, _ = G.conv_ex(act, w, b, 3, out, 0, residual=res.cuda(), residual_up=True, out16=out16, stats=stats)
    _lib.check(rc)
    _check_guard(out, N, tag)
    up = F.interpolate(res.double().permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    want = _ref_conv(act, w, b, 3, False, 0) + up
    got = _f64(out[:N])
    assert G.report(tag, got, want) < CONV_BAR["fp32"]
    _check_stats(stats, got, N, tag)
    assert torch.equal(out16[:N].view(torch.int16), out[:N].half().view(torch.int16))


@pytest.mark.parametrize("e4m3", [False, True], ids=["fp16", "e4m3"])
@pytest.mark.parametrize("C1,C2", [(192, 96), (256, 128), (64, 8)])
def test_three_segment_up_conv(C1, C2, e4m3):
    """Up-path conv2: 3x3 over a plus a 1x1 skip over the virtual concat [x0 | x1] as two more K segments, fp32 output with
    the fp16 copy and the statistics."""
    N, H, W = 2, 16, 16
    C0 = Cout = C1
    tag = f"three segments {C0} 3x3 + 1x1 over {C1}+{C2}" + (" e4m3" if e4m3 else "")
    g = _gen(tag)
    a = _act(g, N, H, W, C0, e4m3)
    x0 = torch.randn(N, H, W, C1, generator=g).half().cuda()
    x1 = torch.randn(N, H, W, C2, generator=g).half().cuda()
    w, b = _conv_weights(g, Cout, C0, 3)
    ws = torch.randn(Cout, C1 + C2, generator=g) / math.sqrt(C1 + C2)
    bs = torch.randn(Cout, generator=g) * 0.1
    out = G.nan_like_buffer((N + 1, H, W, Cout), torch.float32)
    out16 = G.nan_like_buffer((N + 1, H, W, Cout), torch.float16)
    stats = _stats_buffer(N, Cout)
    rc, e = G.conv_ex(a, w, b, 3, out, 0, e4m3=e4m3, act1=x0, act2=x1, wskip=ws, bskip=bs, out16=out16, stats=stats)
    _lib.check(rc)
    _check_guard(out, N, tag)
    want = _ref_conv(a, w, b, 3, e4m3, e, x0, x1, ws, bs)
    got = _f64(out[:N])
    assert G.report(tag, got, want) < CONV_BAR["e4m3" if e4m3 else "fp32"]
    _check_stats(stats, got, N, tag)
    assert torch.equal(out16[:N].view(torch.int16), out[:N].half().view(torch.int16))


@pytest.mark.parametrize("Cout", [3, 4, 8, 9])
def test_nchw_output(Cout):
    """The output head's direct 3x3 conv (9 * out_channels > 64): fp32 NCHW, BN 16, odd channel counts."""
    N, H, W, Cin = 2, 32, 32, 64
    tag = f"NCHW output Cout {Cout}"
    g = _gen(tag)
    act = _act(g, N, H, W, Cin, False)
    w, b = _conv_weights(g, Cout, Cin, 3)
    out = G.nan_like_buffer((N + 1, Cout, H, W), torch.float32)
    rc, _ = G.conv_ex(act, w, b, 3, out, 2)
    _lib.check(rc)
    _check_guard(out, N, tag)
    want = _ref_conv(act, w, b, 3, False, 0).permute(0, 3, 1, 2)
    assert G.report(tag, _f64(out[:N]), want) < CONV_BAR["fp32"]


def test_rejected_combinations():
    """What the network never runs is refused with IVID_ERR_INVALID_ARGUMENT before anything is launched."""
    N, Cin, Cout = 2, 64, 64
    g = _gen("rejections")
    w, b = _conv_weights(g, Cout, Cin, 3)

    def conv(H, W, out_mode=0, **kw):
        act = _act(g, N, H, W, Cin, False)
        shape = (N + 1, Cout, H, W) if out_mode == 2 else (N + 1, H, W, Cout)
        out = G.nan_like_buffer(shape, torch.float16 if out_mode == 1 else torch.float32)
        rc, _ = G.conv_ex(act, w, b, 3, out, out_mode, **kw)
        return rc, out

    res = torch.zeros(N, 16, 16, Cout, device="cuda")
    rejected = {
        "statistics at a 4x4x8 tile": conv(4, 4, stats=_stats_buffer(N, Cout)),
        "statistics with an NCHW output": conv(16, 16, 2, stats=_stats_buffer(N, Cout)),
        "residual_up at W = 8": conv(16, 8, residual=torch.zeros(N, 8, 4, Cout, device="cuda"), residual_up=True),
        "fp16 copy of an fp16 output": conv(16, 16, 1, out16=G.nan_like_buffer((N + 1, 16, 16, Cout), torch.float16)),
        "fp16 copy of an NCHW output": conv(16, 16, 2, out16=G.nan_like_buffer((N + 1, 16, 16, Cout), torch.float16)),
        "residual with an NCHW output": conv(16, 16, 2, residual=res),
    }
    C = 64
    x32 = torch.randn(N, 16, 16, C, generator=g).cuda()
    x16 = x32.half()
    gamma, beta = torch.ones(C), torch.zeros(C)

    def gn(x, mode=0, **kw):
        Ho = 32 if mode == 1 else 16
        out = G.nan_like_buffer((N + 1, Ho, Ho, C), torch.float16)
        lo = G.nan_like_buffer((N + 1, Ho, Ho, C), torch.float16)
        st = torch.zeros(N, C, 2, dtype=torch.float64, device="cuda") + 1.0
        return G.gn_apply(x, None, out, groups=32, gamma=gamma, beta=beta, stats0=st, mode=mode, out_lo=lo, **kw), out

    rejected["split output from fp32 sources"] = gn(x32)
    rejected["split output with an upsample"] = gn(x16, mode=1)
    rejected["split output with a raw copy"] = gn(x16, out_raw16=G.nan_like_buffer((N + 1, 16, 16, C), torch.float16))
    torch.cuda.synchronize()
    for name, (rc, out) in rejected.items():
        assert rc == _lib.IVID_ERR_INVALID_ARGUMENT, f"{name}: status {rc}, {_lib.last_error()}"
        assert bool(torch.isnan(out.float()).all()), f"{name}: a kernel ran"


# ----------------------------------------------------------------------------------------------------------------------
# c. GroupNorm apply from fp16 sources with exact statistics
# ----------------------------------------------------------------------------------------------------------------------
def _exact_stats(x):
    """float64 per-(sample, channel) sum / sum of squares of x [N, H, W, C] (the values the kernel reads)."""
    v = _f64(x)
    return torch.stack([v.sum((1, 2)), (v * v).sum((1, 2))], -1)


def _gn_ref(x, groups, gamma, beta, film, film_off, film_add, silu, stats=None):
    """float64 GroupNorm (+ FiLM) of x [N, H, W, C] as y = x * A + B (then SiLU).  Moments from `stats` ([N, C, 2] sums)
    when given, else exact.  Returns y, A, Bmag, and the group mean and rstd [N, groups]; Bmag [N, C] is the sum of the
    magnitudes of the terms the kernel forms B from in fp32 (beta, mean * A, the FiLM shift), which bounds B's rounding
    error where those terms cancel."""
    v = _f64(x)
    N, H, W, C = v.shape
    n = H * W * (C // groups)
    f = _f64(film) if film is not None else None
    st = _f64(stats) if stats is not None else _exact_stats(x)
    S, Q = st[..., 0], st[..., 1]
    if film_add:
        e = f[:, film_off:film_off + C]
        S, Q = S + H * W * e, Q + 2 * e * S + H * W * e * e
    mean = S.reshape(N, groups, -1).sum(-1) / n
    var = (Q.reshape(N, groups, -1).sum(-1) / n - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    r_c = rstd.repeat_interleave(C // groups, 1)
    m_c = mean.repeat_interleave(C // groups, 1)
    A = r_c * gamma.double()
    B = beta.double() - m_c * A
    Bmag = beta.double().abs() + (m_c * A).abs()
    if film is not None and film_add:
        B = B + e * A
        Bmag = Bmag + (e * A).abs()
    elif film is not None:
        sc, sh = f[:, film_off:film_off + C], f[:, film_off + C:film_off + 2 * C]
        A, B = A * (1 + sc), B * (1 + sc) + sh
        Bmag = Bmag * (1 + sc).abs() + sh.abs()
    z = v * A[:, None, None, :] + B[:, None, None, :]
    y = F.silu(z) if silu else z
    return y, A, Bmag, mean, rstd


def _slack(x, A, Bmag, silu):
    """2^-20 (|x A| + |B|), with |B| counted as Bmag (see _gn_ref): the fp32 coefficients and FMA of the apply and the
    approximate SiLU (whose slope is at most 1.1)."""
    s = 2.0 ** -20 * ((_f64(x) * A[:, None, None, :]).abs() + Bmag[:, None, None, :])
    return s * 1.1 if silu else s


def _ulp16(y):
    return torch.exp2(torch.floor(torch.log2(y.abs().clamp_min(2.0 ** -14))) - 10)


def _ulp8(y):
    return torch.exp2(torch.floor(torch.log2(y.abs().clamp(2.0 ** -6, 448.0))) - 3)


def _check_apply(out, y, slack, N, tag, e4m3=False, out_lo=None):
    _check_guard(out, N, tag)
    if e4m3:
        got = out[:N].cpu().view(torch.float8_e4m3fn).double()
        yc = y.clamp(-448.0, 448.0)
        d = (got - yc).abs()
        exact = float((out[:N].cpu() == _e4m3(y.float()).view(torch.uint8)).double().mean())
        over = float((d / (_ulp8(yc) + slack)).max())
        print(f"[fused] {tag}: e4m3 |out - y64| / (ulp + slack) max {over:.3f}, round-to-nearest-even {exact:.5f}")
        assert over <= 1.0 and exact >= 0.999, f"{tag}: e4m3 output off"
        return
    got = _f64(out[:N])
    over = float(((got - y).abs() / (_ulp16(y) + slack)).max())
    print(f"[fused] {tag}: fp16 |out - y64| / (ulp + slack) max {over:.3f}")
    assert over <= 1.0, f"{tag}: fp16 output off"
    if out_lo is not None:
        _check_guard(out_lo, N, f"{tag} low half")
        # lo is itself fp16: half its subnormal spacing (2^-25) on top
        two = got + _f64(out_lo[:N])
        over = float(((two - y).abs() / (slack + 2.0 ** -25)).max())
        print(f"[fused] {tag}: hi + lo |error| / (slack + 2^-25) max {over:.3f}")
        assert over <= 1.0, f"{tag}: two-term split off"


# tag, C0, C1, groups, FiLM (None / "ss" scale-shift / "add"), SiLU, output ("f16", "lo" with the split, "e4m3").
# Hoisted (256 % (C / 8) == 0): 256, 256+256.  Prologue fast path (power-of-two group width <= 32, C % 32 == 0, C <= 1024):
# cpg 8, 16, 2; the loop: cpg 24, 9, 3, 5 and C = 1792.
GN_CASES = [
    ("C256 hoisted", 256, 0, 32, "ss", True, "f16"),
    ("C256+256 hoisted", 256, 256, 32, "ss", True, "f16"),
    ("C256 hoisted split", 256, 0, 32, None, True, "lo"),
    ("C256 hoisted film_add fast", 256, 0, 32, "add", False, "f16"),
    ("C512+256 cpg24", 512, 256, 32, "ss", True, "f16"),
    ("C192+96 cpg9 film_add", 192, 96, 32, "add", True, "f16"),
    ("C96 cpg2 film_add fast", 96, 0, 48, "add", True, "f16"),
    ("C96 cpg3 split", 96, 0, 32, None, True, "lo"),
    ("C40 cpg5", 40, 0, 8, "ss", False, "f16"),
    ("C1024+768 cpg56", 1024, 768, 32, "ss", True, "f16"),
    ("C256 hoisted e4m3", 256, 0, 32, "ss", True, "e4m3"),
    ("C512+256 cpg24 film_add e4m3", 512, 256, 32, "add", True, "e4m3"),
]


@pytest.mark.parametrize("case", GN_CASES, ids=[c[0] for c in GN_CASES])
def test_group_norm_apply_fp16_sources(case):
    tag, C0, C1, groups, film_kind, silu, form = case
    N, H, W = 3, 16, 16
    C = C0 + C1
    g = _gen(tag)
    # per-channel scale and offset: the moments of x + e differ from those of x
    src = lambda c: (torch.randn(N, H, W, c, generator=g) * (torch.rand(c, generator=g) * 1.5 + 0.5)
                     + torch.randn(c, generator=g)).half().cuda()
    x0 = src(C0)
    x1 = src(C1) if C1 else None
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g) * 0.2
    film = (torch.randn(N, 6 * C, generator=g) * 0.3).cuda() if film_kind else None
    out = G.nan_like_buffer((N + 1, H, W, C), torch.uint8 if form == "e4m3" else torch.float16)
    lo = G.nan_like_buffer((N + 1, H, W, C), torch.float16) if form == "lo" else None
    st0 = _exact_stats(x0).cuda()
    st1 = _exact_stats(x1).cuda() if C1 else None
    _lib.check(G.gn_apply(x0, x1, out, groups=groups, gamma=gamma, beta=beta, stats0=st0, stats1=st1, film=film,
                          film_ld=6 * C, film_off=2 * C, film_add=film_kind == "add", silu=silu, out_e4m3=form == "e4m3",
                          out_lo=lo))
    x = torch.cat([x0, x1], -1) if C1 else x0
    y, A, Bm, _, _ = _gn_ref(x, groups, gamma, beta, film, 2 * C, film_kind == "add", silu)
    _check_apply(out, y, _slack(x, A, Bm, silu), N, f"gn_apply {tag}", e4m3=form == "e4m3", out_lo=lo)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_group_norm_raw_outputs_bit_exact(mode):
    """The fp32-source kernel's raw outputs: mode 0 the fp16 copy (operand of a skip conv), mode 1 the nearest-2x
    upsample, mode 2 the 2x2 average summed as (((0 + a00) + a01) + a10) + a11, times 0.25, in fp32."""
    N, H, W, C0, C1 = 2, 16, 16, 128, 64
    g = _gen(f"raw {mode}")
    x0 = torch.randn(N, H, W, C0, generator=g)
    x1 = torch.randn(N, H, W, C1, generator=g) * 3 + 1
    x = torch.cat([x0, x1], -1)
    C = C0 + C1
    Ho, Wo = (2 * H, 2 * W) if mode == 1 else ((H // 2, W // 2) if mode == 2 else (H, W))
    out = G.nan_like_buffer((N + 1, Ho, Wo, C), torch.float16)
    raw16 = G.nan_like_buffer((N + 1, Ho, Wo, C), torch.float16) if mode == 0 else None
    raw32 = G.nan_like_buffer((N + 1, Ho, Wo, C), torch.float32) if mode != 0 else None
    _lib.check(G.gn_apply(x0.cuda(), x1.cuda(), out, groups=32, gamma=torch.ones(C), beta=torch.zeros(C), mode=mode,
                          out_raw16=raw16, out_raw32=raw32))
    _check_guard(out, N, f"raw mode {mode} activation")
    if mode == 0:
        _check_guard(raw16, N, "raw16")
        assert torch.equal(raw16[:N].cpu().view(torch.int16), x.half().view(torch.int16))
    elif mode == 1:
        _check_guard(raw32, N, "raw32 up")
        want = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
        assert torch.equal(raw32[:N].cpu(), want)
    else:
        _check_guard(raw32, N, "raw32 pool")
        acc = torch.zeros(N, Ho, Wo, C)
        for dy in (0, 1):
            for dx in (0, 1):
                acc = acc + x[:, dy::2, dx::2, :]
        assert torch.equal(raw32[:N].cpu(), acc * 0.25)


# ----------------------------------------------------------------------------------------------------------------------
# d. conv1 -> GN2 at a DC offset: how far the fused statistics can be trusted
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [0, 10, 30, 100])
def test_in_block_chain_at_dc_offset(k):
    """A conv with fp16 output and fused statistics feeds the apply, as conv1 -> GN2 does, with every channel biased to a
    group mean of k sigma.  The epilogue sums v and v^2 in fp32 (relative error <= GAMMA12 each), so with sums over n
    values of a group, |dS| <= GAMMA12 sum|v| and |dQ| <= GAMMA12 Q, and var = Q/n - mean^2 is off by at most
        dvar = GAMMA12 (Q/n + 2 |mean| sum|v| / n)  ~  GAMMA12 (1 + 3 k^2) sigma^2,
    rstd by dvar / (2 var) relative, the mean by GAMMA12 sum|v| / n.  The test derives these bounds from the data, prints
    them beside the measured errors, requires the measured ones to stay inside, and widens the output bar of test c by
    what they allow."""
    N, H, W, Cin, C, groups = 2, 32, 32, 128, 256, 32
    tag = f"dc offset k={k}"
    g = _gen(tag)
    act = _act(g, N, H, W, Cin, False)
    w = torch.randn(C, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin)
    b = torch.full((C,), float(k)) + torch.randn(C, generator=g) * 0.01
    h = G.nan_like_buffer((N + 1, H, W, C), torch.float16)
    stats = _stats_buffer(N, C)
    rc, _ = G.conv_ex(act, w, b, 3, h, 1, stats=stats)
    _lib.check(rc)
    _check_guard(h, N, f"{tag} hidden tensor")
    _check_stats(stats, _f64(h[:N]), N, tag)
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g) * 0.2
    film = (torch.randn(N, 6 * C, generator=g) * 0.3).cuda()
    out = G.nan_like_buffer((N + 1, H, W, C), torch.float16)
    x = h[:N].contiguous()
    _lib.check(G.gn_apply(x, None, out, groups=groups, gamma=gamma, beta=beta, stats0=stats[:N].contiguous(), film=film,
                          film_ld=6 * C, film_off=2 * C, silu=True))
    y, A, Bm, mean, rstd = _gn_ref(x, groups, gamma, beta, film, 2 * C, False, True)
    _, _, _, mean_f, rstd_f = _gn_ref(x, groups, gamma, beta, film, 2 * C, False, True, stats=stats[:N])
    v = _f64(x).reshape(N, H * W, groups, -1)
    n = v.shape[1] * v.shape[3]
    abs_mean = v.abs().sum((1, 3)) / n
    sq_mean = (v * v).sum((1, 3)) / n
    var = sq_mean - mean * mean
    dmean = GAMMA12 * abs_mean
    drstd = GAMMA12 * (sq_mean + 2 * mean.abs() * abs_mean) / (2 * var)
    sigma = var.sqrt()
    m_err = float(((mean_f - mean).abs() / sigma).max())
    r_err = float(((rstd_f / rstd) - 1).abs().max())
    print(f"[fused] {tag}: group mean / sigma {float((mean / sigma).mean()):.1f}; measured mean error {m_err:.2e} sigma "
          f"(bound {float((dmean / sigma).max()):.2e}), rstd relative error {r_err:.2e} (bound {float(drstd.max()):.2e})")
    assert bool(((mean_f - mean).abs() <= dmean).all()), f"{tag}: fused mean outside the fp32 rounding bound"
    assert bool(((rstd_f / rstd - 1).abs() <= drstd).all()), f"{tag}: fused rstd outside the fp32 rounding bound"
    cpg = C // groups
    dm_c, dr_c = dmean.repeat_interleave(cpg, 1), drstd.repeat_interleave(cpg, 1)
    m_c = mean.repeat_interleave(cpg, 1)
    xv = _f64(x)
    widen = (dm_c[:, None, None, :] + (xv - m_c[:, None, None, :]).abs() * dr_c[:, None, None, :]) * A.abs()[:, None, None, :]
    _check_apply(out, y, _slack(x, A, Bm, True) + 1.1 * widen, N, tag)


# ----------------------------------------------------------------------------------------------------------------------
# e. determinism and batch invariance of the statistics
# ----------------------------------------------------------------------------------------------------------------------
def _hidden_conv(act, w, b, N):
    H, W, C = act.shape[1], act.shape[2], w.shape[0]
    out = G.nan_like_buffer((N + 1, H, W, C), torch.float16)
    stats = _stats_buffer(N, C)
    rc, _ = G.conv_ex(act, w, b, 3, out, 1, stats=stats)
    _lib.check(rc)
    return out, stats


def test_statistics_run_to_run_bit_identical():
    """The benchmark layer (N = 32, 128^2, 256 -> 256, fp16 output with statistics), 20 launches: the fp64 atomics add the
    tiles' fp32 partials in whatever order the tiles finish, and the results stay bit-identical."""
    N, H, W, C = 32, 128, 128, 256
    g = _gen("determinism")
    act = _act(g, N, H, W, C, False)
    w, b = _conv_weights(g, C, C, 3)
    out0, st0 = _hidden_conv(act, w, b, N)
    _check_stats(st0, out0[:N].double(), N, "benchmark layer")
    for i in range(19):
        out, st = _hidden_conv(act, w, b, N)
        assert torch.equal(st.view(torch.int64), st0.view(torch.int64)), f"launch {i + 2}: statistics differ"
        assert torch.equal(out.view(torch.int16), out0.view(torch.int16)), f"launch {i + 2}: output differs"


@pytest.mark.parametrize("H,W", [(32, 32), (8, 8), (8, 4)], ids=["16x8x1", "8x8x2", "4x8x4"])
def test_statistics_batch_invariant(H, W):
    """A sample's statistics alone are bit-identical to that sample's statistics inside a batch, wherever the sample sits
    in its tile."""
    N, Cin, C = 7, 64, 128
    g = _gen(f"batch invariance {H}x{W}")
    act = _act(g, N, H, W, Cin, False)
    w, b = _conv_weights(g, C, Cin, 3)
    out, st = _hidden_conv(act, w, b, N)
    for i in range(N):
        o1, s1 = _hidden_conv(act[i:i + 1].contiguous(), w, b, 1)
        assert torch.equal(s1[0].view(torch.int64), st[i].view(torch.int64)), f"sample {i}: statistics depend on the batch"
        assert torch.equal(o1[0].view(torch.int16), out[i].view(torch.int16)), f"sample {i}: output depends on the batch"

"""GPU: the layers that change resolution, and the GroupNorm passes over fp32 sources, against float64 references.

Each test runs one op entry point on crafted data and compares every element with float64 computed on the CPU from the
same rounded operands the kernels read:
  a. gn_stats_kernel (ivid_op_gn_stats): |S - S64| <= gamma(m) sum|x| and |Q - Q64| <= gamma(m + 1) sum x^2 per (sample,
     channel), plus the fp64 rest, with m = ceil(min(HW, 256) / rows) the longest fp32 run of one thread
     (tests/resample_model.py).  The rstd that follows from these sums is also held to 2^-11, the fp16 activation's
     rounding, for data at a DC offset of k <= 30 sigma, and printed at k = 100.
  b. gn_apply_kernel over fp32 sources (ivid_op_group_norm_apply), modes 0 / 1 / 2: fp16 ulp + the apply slack of
     tests/test_gpu_fused_epilogue.py.  Mode 2 adds the three fp32 additions of the four activations (the x0.25 is
     exact); statistics left NULL add the bound of a, carried through the group mean, rstd and affine.
  c. Downsample2d's stride-2 conv (ivid_op_resample, mode 2, conv 1): (K + 1) 2^-23 S with S = sum |a w| + |b| and
     K = conv_pad_k(9C), the bound of tests/test_gpu_conv_slab.py; its gathered operand bit for bit.
  d. Upsample2d's conv (mode 1, conv 1): the same bound with K = 9 conv_pad_k(C); its operand is nearest-2x bit for bit.
  e. AvgPool2d(2) / nearest 2x (conv 0): bit for bit against numpy float32, and the pool within its three roundings of
     float64, 2^-24 (|a00 + a01| + |a10 + a11| + |sum|) / 4: 2 fp32 ulp of the mean where the four inputs share a sign,
     more where they cancel.
  The statistics each resampling op emits are checked against float64 sums of its own fp32 output: the fused bound of
  tests/test_gpu_fused_epilogue.py (12 roundings) where the conv epilogue takes them, the bound of a otherwise.
  f. ivid_op_resample runs what the network runs: each down / up layer of the plainconv and plainpool configs, fed its
     input tap, gives that layer's output tap bit for bit.

Every output and statistics buffer is prefilled with NaN and holds one guard sample past N: every valid element must
come back finite and the guard must stay NaN.  Each case prints its worst |err| / bound."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
import resample_model as M
from ivid_b200 import _lib
from test_gpu_fused_epilogue import _check_apply, _check_guard, _exact_stats, _f64, _gen, _gn_ref, _slack

pytestmark = pytest.mark.gpu

U23 = 2.0 ** -23
FUSED_BAR = 1e-6            # the fused statistics: 12 fp32 roundings, 12 * 2^-24 = 7.2e-7 (test_gpu_fused_epilogue.py)


def _stats_buffer(N, C):
    st = G.nan_like_buffer((N + 1, C, 2), torch.float64)
    st[:N].zero_()
    return st


def _gn_stats(x, N, H, W, C, stats):
    return _lib.lib().ivid_op_gn_stats(x.data_ptr(), N, H, W, C, stats.data_ptr(), _lib.cur_stream())


def _resample(mode, conv, x, out, *, N, w=None, b=None, out16=None, stats=None, operand=None):
    _, H, W, C = x.shape
    p = lambda t: t.data_ptr() if t is not None else None
    wh = w.float().contiguous() if w is not None else None
    bh = b.float().contiguous() if b is not None else None
    a = _lib.OpResampleT(mode=mode, conv=conv, x_dev=x.data_ptr(), N=N, H=H, W=W, C=C, w_host=p(wh), b_host=p(bh),
                         out_dev=out.data_ptr(), out16_dev=p(out16), stats_dev=p(stats), operand_dev=p(operand))
    return _lib.lib().ivid_op_resample(ctypes.byref(a), _lib.cur_stream())


def _check_stats_bound(stats, vals, N, C, HW, tag):
    """stats [N+1, C, 2] from gn_stats against float64 sums of vals [N, HW, C] (the fp32 values it read)."""
    _check_guard(stats, N, f"{tag} statistics")
    v = vals.numpy()
    bS, bQ = M.gn_stats_bound(v, C, HW)
    st = stats[:N].cpu().numpy()
    rs = float((np.abs(st[..., 0] - v.sum(1)) / bS).max())
    rq = float((np.abs(st[..., 1] - (v * v).sum(1)) / bQ).max())
    print(f"[resample] {tag}: gn_stats |S - S64| / bound max {rs:.3e}, |Q - Q64| / bound max {rq:.3e} "
          f"(m = {M.gn_stats_run(C, HW)})")
    assert rs <= 1.0 and rq <= 1.0, f"{tag}: gn_stats outside its fp32 rounding bound"
    return bS, bQ


def _check_fused_stats(stats, vals, N, tag):
    _check_guard(stats, N, f"{tag} statistics")
    st = stats[:N].cpu()
    S64, A64, Q64 = vals.sum(1), vals.abs().sum(1), (vals * vals).sum(1)
    rs = float(((st[..., 0] - S64).abs() / A64).max())
    rq = float(((st[..., 1] - Q64).abs() / Q64).max())
    print(f"[resample] {tag}: fused statistics |S - S64| / sum|v| max {rs:.2e}, |Q - Q64| / Q64 max {rq:.2e} "
          f"(bar {FUSED_BAR:.0e})")
    assert rs <= FUSED_BAR and rq <= FUSED_BAR, f"{tag}: fused statistics off"


# ----------------------------------------------------------------------------------------------------------------------
# a. the separate statistics pass
# ----------------------------------------------------------------------------------------------------------------------
def _offset_data(g, N, HW, C, k):
    """[N, HW, C] fp32: per-channel sigma in [0.5, 2) and mean k sigma (+- 0.1 sigma)."""
    sigma = torch.rand(C, generator=g) * 1.5 + 0.5
    mu = (k + 0.1 * torch.randn(C, generator=g)) * sigma
    return torch.randn(N, HW, C, generator=g) * sigma + mu


@pytest.mark.parametrize("case", M.STATS_CASES, ids=[M.stats_case_id(c) for c in M.STATS_CASES])
def test_gn_stats(case):
    C, HW, N, k = case
    tag = M.stats_case_id(case)
    g = _gen(tag)
    x = _offset_data(g, N, HW, C, k)
    stats = _stats_buffer(N, C)
    _lib.check(_gn_stats(x.cuda(), N, HW, 1, C, stats))
    v = x.double()
    _check_stats_bound(stats, v, N, C, HW, tag)
    # the rstd the apply forms from these sums, per group, against the exact one
    groups = 32 if C % 32 == 0 else 8
    n = HW * (C // groups)
    st = stats[:N].cpu()

    def rstd(S, Q):
        mean = S.reshape(N, groups, -1).sum(-1) / n
        var = (Q.reshape(N, groups, -1).sum(-1) / n - mean * mean).clamp_min(0)
        return 1.0 / torch.sqrt(var + 1e-5)

    r_err = float((rstd(st[..., 0], st[..., 1]) / rstd(v.sum(1), (v * v).sum(1)) - 1).abs().max())
    print(f"[resample] {tag}: rstd relative error {r_err:.3e} = {r_err / 2.0 ** -11:.3f} x 2^-11 (DC offset {k} sigma)")
    if k <= 30:
        assert r_err <= 2.0 ** -11, f"{tag}: rstd error exceeds the fp16 activation's rounding"


def test_gn_stats_rejects_bad_arguments():
    x = torch.zeros(2, 4, 4, 8, device="cuda")
    st = G.nan_like_buffer((2, 8, 2), torch.float64)
    for args in [(2, 4, 4, 6), (0, 4, 4, 8), (2, 0, 4, 8), (2, 4, 4, 0)]:
        assert _gn_stats(x, *args, st) == _lib.IVID_ERR_INVALID_ARGUMENT, f"{args}: {_lib.last_error()}"
    assert _lib.lib().ivid_op_gn_stats(None, 2, 4, 4, 8, st.data_ptr(), _lib.cur_stream()) == _lib.IVID_ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert bool(torch.isnan(st).all()), "a kernel ran"


# ----------------------------------------------------------------------------------------------------------------------
# b. GroupNorm apply over fp32 sources
# ----------------------------------------------------------------------------------------------------------------------
def _stats_widen(x0, x1, N, groups, film, film_add, A, mean, rstd):
    """The bound of a on each source's gn_stats sums, carried to the output: |dy| <= (dmean + |x - mean| drstd) |A|."""
    parts = [x0] + ([x1] if x1 is not None else [])
    dS, dQ = [], []
    for t in parts:
        _, H, W, c = t.shape
        bS, bQ = M.gn_stats_bound(_f64(t[:N]).reshape(N, H * W, c).numpy(), c, H * W)
        dS.append(torch.from_numpy(bS))
        dQ.append(torch.from_numpy(bQ))
    dS, dQ = torch.cat(dS, -1), torch.cat(dQ, -1)
    x = torch.cat([_f64(t[:N]) for t in parts], -1)
    Nn, H, W, C = x.shape
    if film_add:
        e = _f64(film)[:, 2 * C:3 * C]
        dQ = dQ + 2 * e.abs() * dS
        x = x + e[:, None, None, :]
    n = H * W * (C // groups)
    dmean = dS.reshape(N, groups, -1).sum(-1) / n
    var = 1.0 / (rstd * rstd) - 1e-5
    dvar = dQ.reshape(N, groups, -1).sum(-1) / n + (2 * mean.abs() + dmean) * dmean
    drstd = dvar / (2 * (var + 1e-5)) * 1.01
    cpg = C // groups
    dm_c, dr_c, m_c = (t.repeat_interleave(cpg, 1)[:, None, None, :] for t in (dmean, drstd, mean))
    return (dm_c + (x - m_c).abs() * dr_c) * A.abs()[:, None, None, :]


def _apply_case_id(c):
    return c[0].replace(" ", "-")


@pytest.mark.parametrize("case", M.APPLY_CASES, ids=[_apply_case_id(c) for c in M.APPLY_CASES])
def test_group_norm_apply_fp32_sources(case):
    tag, C0, C1, groups, film_kind, with_stats, mode, H, W, N = case
    C = C0 + C1
    g = _gen(tag)
    src = lambda c: (torch.randn(N, H, W, c, generator=g) * (torch.rand(c, generator=g) * 1.5 + 0.5)
                     + torch.randn(c, generator=g)).cuda()
    x0 = src(C0)
    x1 = src(C1) if C1 else None
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g) * 0.2
    film = (torch.randn(N, 6 * C, generator=g) * 0.3).cuda() if film_kind else None
    Ho, Wo = (2 * H, 2 * W) if mode == 1 else ((H // 2, W // 2) if mode == 2 else (H, W))
    out = G.nan_like_buffer((N + 1, Ho, Wo, C), torch.float16)
    st0 = _exact_stats(x0).cuda() if with_stats else None
    st1 = _exact_stats(x1).cuda() if with_stats and C1 else None
    assert M.apply_path(case) == ("fast" if tag.startswith("fast") else "loop")
    _lib.check(G.gn_apply(x0, x1, out, groups=groups, gamma=gamma, beta=beta, stats0=st0, stats1=st1, film=film,
                          film_ld=6 * C, film_off=2 * C, film_add=film_kind == "add", silu=True, mode=mode))
    x = torch.cat([x0, x1], -1) if C1 else x0
    y, A, Bm, mean, rstd = _gn_ref(x, groups, gamma, beta, film, 2 * C, film_kind == "add", True)
    slack = _slack(x, A, Bm, True)
    if not with_stats:
        slack = slack + 1.1 * _stats_widen(x0, x1, N, groups, film, film_kind == "add", A, mean, rstd)
    if mode == 1:
        up = lambda t: t.repeat_interleave(2, 1).repeat_interleave(2, 2)
        y, slack = up(y), up(slack)
    elif mode == 2:
        q = lambda t, dy, dx: t[:, dy::2, dx::2]
        s1 = q(y, 0, 0) + q(y, 0, 1)
        s2 = s1 + q(y, 1, 0)
        s3 = s2 + q(y, 1, 1)
        add = 2.0 ** -24 * (s1.abs() + s2.abs() + s3.abs())
        slack = 0.25 * (q(slack, 0, 0) + q(slack, 0, 1) + q(slack, 1, 0) + q(slack, 1, 1) + add)
        y = 0.25 * s3
    _check_apply(out, y, slack, N, f"gn_apply fp32 {tag}")


# ----------------------------------------------------------------------------------------------------------------------
# c / d. the resampling convs
# ----------------------------------------------------------------------------------------------------------------------
def _im2col_s2(x):
    """col [N, Ho, Wo, 9C] = x[2yo + dy - 1, 2xo + dx - 1] at tap dy * 3 + dx, zero outside the image."""
    N, H, W, C = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    return torch.cat([xp[:, dy:dy + H:2, dx:dx + W:2] for dy in range(3) for dx in range(3)], -1)


@pytest.mark.parametrize("case", M.DOWN_CASES + M.UP_CASES, ids=[M.conv_case_id(c) for c in M.DOWN_CASES + M.UP_CASES])
def test_resample_conv(case):
    mode, C, N, Ho, Wo = case
    tag = M.conv_case_id(case)
    TW, TH, TN, fused = G.conv_tile(Ho, Wo)
    assert (TW, TH, TN) == M.conv_tile(Ho, Wo) and bool(fused) == M.conv_can_fuse_stats(Ho, Wo)
    H, W = (Ho // 2, Wo // 2) if mode == 1 else (2 * Ho, 2 * Wo)
    g = _gen(tag)
    x = torch.randn(N, H, W, C, generator=g).half()
    w = torch.randn(C, C, 3, 3, generator=g) / math.sqrt(9 * C)
    b = torch.randn(C, generator=g) * 0.5
    out = G.nan_like_buffer((N + 1, Ho, Wo, C), torch.float32)
    out16 = G.nan_like_buffer((N + 1, Ho, Wo, C), torch.float16)
    stats = _stats_buffer(N, C)
    operand = G.nan_like_buffer((N + 1, Ho, Wo, 9 * C if mode == 2 else C), torch.float16)
    _lib.check(_resample(mode, 1, x.cuda(), out, N=N, w=w, b=b, out16=out16, stats=stats, operand=operand))
    _check_guard(out, N, tag)
    _check_guard(out16, N, f"{tag} fp16 copy")
    _check_guard(operand, N, f"{tag} operand")
    x64, w64 = x.double().permute(0, 3, 1, 2), w.half().double()
    if mode == 1:
        x64 = x64.repeat_interleave(2, 2).repeat_interleave(2, 3)
    stride = 2 if mode == 2 else 1
    want = F.conv2d(x64, w64, b.double(), stride=stride, padding=1).permute(0, 2, 3, 1)
    S = F.conv2d(x64.abs(), w64.abs(), b.double().abs(), stride=stride, padding=1).permute(0, 2, 3, 1)
    K = M.conv_K(mode, C)
    got = _f64(out[:N])
    ratio = float(((got - want).abs() / ((K + 1) * U23 * S)).max())
    G.report(f"resample {tag}", got, want)
    print(f"[resample] {tag}: max |err| / bound {ratio:.3e} (K = {K})")
    want_op = _im2col_s2(x) if mode == 2 else x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert torch.equal(operand[:N].cpu().view(torch.int16), want_op.view(torch.int16)), f"{tag}: conv operand differs"
    assert ratio <= 1.0, f"{tag}: error {ratio:.3g}x the fp32-accumulation bound"
    assert torch.equal(out16[:N].view(torch.int16), out[:N].half().view(torch.int16)), f"{tag}: fp16 copy != out.half()"
    vals = got.reshape(N, Ho * Wo, C)
    if fused:
        _check_fused_stats(stats, vals, N, tag)
    else:
        _check_stats_bound(stats, vals, N, C, Ho * Wo, tag)


# ----------------------------------------------------------------------------------------------------------------------
# e. pooling / nearest without a conv
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", M.PLAIN_CASES, ids=[M.plain_case_id(c) for c in M.PLAIN_CASES])
def test_resample_plain(case):
    mode, C, N, H, W = case
    tag = M.plain_case_id(case)
    Ho, Wo = (2 * H, 2 * W) if mode == 1 else (H // 2, W // 2)
    g = _gen(tag)
    x = torch.randn(N, H, W, C, generator=g) * 2 + torch.randn(C, generator=g)
    out = G.nan_like_buffer((N + 1, Ho, Wo, C), torch.float32)
    out16 = G.nan_like_buffer((N + 1, Ho, Wo, C), torch.float16)
    stats = _stats_buffer(N, C)
    _lib.check(_resample(mode, 0, x.cuda(), out, N=N, out16=out16, stats=stats))
    _check_guard(out, N, tag)
    _check_guard(out16, N, f"{tag} fp16 copy")
    got = out[:N].cpu()
    if mode == 1:
        assert torch.equal(got, x.repeat_interleave(2, 1).repeat_interleave(2, 2)), f"{tag}: nearest 2x is not a copy"
    else:
        x64 = x.double().numpy()
        p64 = 0.25 * (x64[:, 0::2, 0::2] + x64[:, 0::2, 1::2] + x64[:, 1::2, 0::2] + x64[:, 1::2, 1::2])
        err = np.abs(got.double().numpy() - p64)
        ratio = float((err / M.pool_bound(x64)).max())
        # where the four inputs share a sign no partial sum exceeds the total: within 2 ulp of the float64 mean
        q = [x64[:, dy::2, dx::2] for dy in (0, 1) for dx in (0, 1)]
        same = np.all([np.sign(t) == np.sign(q[0]) for t in q[1:]], 0)
        ulps = float((err / M.ulp32(p64))[same].max())
        print(f"[resample] {tag}: pool |err| / bound max {ratio:.3f}; same-sign windows: max {ulps:.2f} fp32 ulp of the "
              f"float64 mean")
        assert np.array_equal(got.numpy().view(np.int32), M.pool_f32(x.numpy()).view(np.int32)), \
            f"{tag}: pool differs from ((a00 + a01) + (a10 + a11)) * 0.25 in fp32"
        assert ratio <= 1.0 and ulps <= 2.0
    assert torch.equal(out16[:N].view(torch.int16), out[:N].half().view(torch.int16)), f"{tag}: fp16 copy != out.half()"
    _check_stats_bound(stats, got.double().reshape(N, Ho * Wo, C), N, C, Ho * Wo, tag)


def test_resample_rejects_bad_arguments():
    """Shapes and forms the network never runs are refused with IVID_ERR_INVALID_ARGUMENT before anything is launched."""
    N, C = 2, 64
    x16 = torch.zeros(N, 8, 8, C, dtype=torch.float16, device="cuda")
    x32 = torch.zeros(N, 8, 8, C, device="cuda")
    w = torch.zeros(C, C, 3, 3)
    out = G.nan_like_buffer((N, 16, 16, C), torch.float32)
    op = G.nan_like_buffer((N, 16, 16, C), torch.float16)
    cases = {
        "mode 0": _resample(0, 1, x16, out, N=N, w=w),
        "conv 2": _resample(1, 2, x16, out, N=N, w=w),
        "conv without weights": _resample(1, 1, x16, out, N=N),
        "odd width to pool": _resample(2, 0, x32[:, :, :7].contiguous(), out, N=N),
        "C % 8": _resample(1, 0, x32[..., :60].contiguous(), out, N=N),
        "N = 0": _resample(1, 0, x32, out, N=0),
        "operand without a conv": _resample(1, 0, x32, out, N=N, operand=op),
    }
    torch.cuda.synchronize()
    for name, rc in cases.items():
        assert rc == _lib.IVID_ERR_INVALID_ARGUMENT, f"{name}: status {rc}, {_lib.last_error()}"
    assert bool(torch.isnan(out).all()) and bool(torch.isnan(op.float()).all()), "a kernel ran"


# ----------------------------------------------------------------------------------------------------------------------
# f. the op runs what the network runs
# ----------------------------------------------------------------------------------------------------------------------
def _tap(net, N, name):
    L = _lib.lib()
    C, H, W = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), None, 0, ctypes.byref(C), ctypes.byref(H), ctypes.byref(W)))
    out = torch.empty((N, C.value, H.value, W.value), dtype=torch.float32)
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), _lib.ptr(out), out.numel(), None, None, None))
    return out.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("tag", ["plainconv", "plainpool"])
def test_resample_op_matches_network(tag):
    import ivid_b200.backbones as backbones
    from oracle import unet_ref
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "options_golden.npz"))
    cfg = json.loads(bytes(gold[f"{tag}_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(sd)
    net = net.cuda()
    x = torch.from_numpy(gold[f"{tag}_x"])
    N = x.shape[0]
    net(x.cuda(), torch.from_numpy(gold[f"{tag}_t"]).cuda(), torch.from_numpy(gold[f"{tag}_c"]).cuda())
    torch.cuda.synchronize()
    blocks, _ = unet_ref._topology(cfg)
    layers = [l for blk in blocks for l in blk["layers"]]
    conv = 1 if cfg["conv_resample"] else 0
    checked = 0
    for i, l in enumerate(layers):
        if l[0] not in ("down", "up"):
            continue
        name, mode = l[1], 2 if l[0] == "down" else 1
        xin = _tap(net, N, layers[i - 1][1])
        want = _tap(net, N, name)
        C = xin.shape[-1]
        out = G.nan_like_buffer(tuple(want.shape), torch.float32)
        if conv:
            sub = ".op" if mode == 2 else ".conv"
            w, b = sd[name + sub + ".weight"], sd[name + sub + ".bias"]
            rc = _resample(mode, 1, xin.half().cuda(), out, N=N, w=w, b=b)
        else:
            rc = _resample(mode, 0, xin.cuda(), out, N=N)
        _lib.check(rc)
        same = torch.equal(out.cpu().view(torch.int32), want.view(torch.int32))
        print(f"[resample] {tag} {name} ({l[0]}, C{C}, {xin.shape[1]}x{xin.shape[2]}): op output "
              f"{'bit-identical to' if same else 'DIFFERS from'} the network's")
        assert same, f"{tag} {name}: ivid_op_resample differs from the network's layer"
        checked += 1
    assert checked >= 2, f"{tag}: no down / up layers found"

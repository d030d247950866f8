"""GPU: AdmUnet2d, the ops and the samplers at channel widths that are not multiples of 64 — the conv op with padded K
chunks and padded output columns, GroupNorm over concatenations whose seam and groups are not 64-aligned, the network and
InpaintCFG against the unmodified reference (widths_golden.npz), per-block taps, determinism and batch invariance, the
fused output-head step at final width 96 and a guided DDIM run.  Eps bars follow tests/test_gpu_geometry.py (_bar of the
TF32-class floor)."""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
import precision_model as PM
from ivid_b200 import _lib
from oracle import sampler_ref, unet_ref

pytestmark = pytest.mark.gpu
NORTH_STAR = 1e-3
HARD_CAP = 1.6e-3
STEP_TOL = 1e-3
UNET_TAGS = ["mc96", "mc32", "frac", "g8", "narrow8", "legacy96"]
STRENGTH = 0.5
WIDTHS = [8, 24, 32, 40, 96, 160, 288]


def _bar(floor):
    return min(max(NORTH_STAR, 1.15 * floor), HARD_CAP)


@pytest.fixture(scope="module")
def wid():
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "widths_golden.npz")))


def _cfg(g, tag):
    return json.loads(bytes(g[f"{tag}_cfg"]).decode())


def _T(g, tag, k):
    return torch.from_numpy(g[f"{tag}_{k}"])


def _load(cfg, sd):
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(sd)
    return net.cuda()


# ------------------------------------------------------------------------------------------------------------------
# ops
# ------------------------------------------------------------------------------------------------------------------
CONV_CASES = [(ci, co, 3) for ci in WIDTHS for co in WIDTHS] + [(c, c, 1) for c in WIDTHS]


@pytest.mark.parametrize("Cin,Cout,k", CONV_CASES)
def test_conv_any_width_matches_torch(Cin, Cout, k):
    """conv(a) + skip(x) as a second K segment + residual, fp32 and fp16 outputs; bars of test_conv_any_size_matches_torch.
    The skip segment takes the next width of the list, so both segments have partial 64-channel chunks in most cases."""
    Cx = WIDTHS[(WIDTHS.index(Cin) + 1) % len(WIDTHS)]
    H, W = (12, 20) if (Cin + Cout) % 16 else (16, 16)
    g = torch.Generator().manual_seed(Cin * 1000 + Cout * 10 + k)
    N = 3
    a = torch.randn(N, Cin, H, W, generator=g); x = torch.randn(N, Cx, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k); b = 0.1 * torch.randn(Cout, generator=g)
    w2 = torch.randn(Cout, Cx, 1, 1, generator=g) / math.sqrt(Cx); b2 = 0.1 * torch.randn(Cout, generator=g)
    res = torch.randn(N, Cout, H, W, generator=g)
    ah, xh = a.half(), x.half()
    ref16 = F.conv2d(ah.float(), w.half().float(), b, padding=k // 2) + F.conv2d(xh.float(), w2.half().float(), b2) + res
    ref32 = F.conv2d(a, w, b, padding=k // 2) + F.conv2d(x, w2, b2) + res
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().cuda()
    for out16 in (False, True):
        out = G.conv2d(nhwc(ah), w, b, k, act2=nhwc(xh), w2=w2.reshape(Cout, Cx), b2=b2, residual=nhwc(res), out_fp16=out16)
        got = out.float().permute(0, 3, 1, 2).cpu()
        r16 = G.report(f"conv {Cin}+{Cx}->{Cout} k{k} {H}x{W} fp16-out={out16} (vs fp16-rounded operands)", got, ref16)
        r32 = G.report(f"conv {Cin}+{Cx}->{Cout} k{k} {H}x{W} fp16-out={out16} (vs fp32)", got, ref32)
        assert r32 < 2e-3
        if not out16:
            assert r16 < 2e-5


def test_conv_width_not_multiple_of_8_raises():
    a = torch.zeros(1, 4, 4, 20, dtype=torch.float16, device="cuda")
    with pytest.raises(AssertionError):
        G.conv2d(a, torch.zeros(32, 20, 3, 3), torch.zeros(32), 3)


GN_CASES = [
    # N, H, W, C0, C1, groups, silu, mode, film
    (2, 16, 16, 192, 96, 32, True, 0, False),    # 288 = 192 (+) 96: groups of 9 channels straddle the seam
    (2, 16, 16, 192, 96, 32, True, 0, True),
    (2, 16, 16, 96, 96, 32, True, 0, False),     # seam at 96, groups of 6
    (2, 16, 16, 32, 0, 32, True, 0, True),       # groups of one channel
    (2, 16, 16, 40, 0, 8, True, 0, True),        # groups of 5 (C % 32 != 0)
    (2, 16, 16, 80, 40, 8, True, 0, False),      # 120 = 80 (+) 40: groups of 15 straddle the seam
    (2, 16, 16, 160, 0, 32, True, 2, False),     # 2x2 average pool
    (2, 8, 8, 96, 0, 32, True, 1, False),        # nearest 2x upsample
]


@pytest.mark.parametrize("N,H,W,C0,C1,groups,silu,mode,film", GN_CASES)
def test_group_norm_any_width_matches_torch(N, H, W, C0, C1, groups, silu, mode, film):
    g = torch.Generator().manual_seed(C0 * 1000 + C1 * 10 + mode)
    C = C0 + C1
    x0 = torch.randn(N, C0, H, W, generator=g) * 1.7 + 0.3
    x1 = (torch.randn(N, C1, H, W, generator=g) * 0.6 - 0.2) if C1 else None
    gamma = 1 + 0.1 * torch.randn(C, generator=g); beta = 0.1 * torch.randn(C, generator=g)
    x = torch.cat([x0, x1], 1) if C1 else x0
    y = F.group_norm(x, groups, gamma, beta, 1e-5)
    fl = None
    if film:
        fl = 0.3 * torch.randn(N, 2 * C, generator=g)
        y = y * (1 + fl[:, :C, None, None]) + fl[:, C:, None, None]
    if silu:
        y = F.silu(y)
    if mode == 1:
        y = F.interpolate(y, scale_factor=2, mode="nearest")
    elif mode == 2:
        y = F.avg_pool2d(y, 2)
    out = G.group_norm(x0.permute(0, 2, 3, 1).contiguous().cuda(), x1.permute(0, 2, 3, 1).contiguous().cuda() if C1 else None,
                       groups, gamma, beta, fl.cuda() if film else None, silu, mode)
    r = G.report(f"group_norm C{C0}+{C1} groups {groups} mode{mode} film{film}", out.float().permute(0, 3, 1, 2), y)
    assert r < 6e-4     # output is rounded to fp16 (2^-11 relative)


# ------------------------------------------------------------------------------------------------------------------
# network and framework against the reference
# ------------------------------------------------------------------------------------------------------------------
def _tap(net, N, name):
    import ctypes
    L = _lib.lib()
    C, H, W = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), None, 0, ctypes.byref(C), ctypes.byref(H), ctypes.byref(W)))
    out = torch.empty((N, C.value, H.value, W.value), dtype=torch.float32)
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), _lib.ptr(out), out.numel(), None, None, None))
    return out


def _check(name, got, ref, floor):
    err = G.report(name, got, ref)
    print(f"[parity] {name}: eps rel {err:.3e}  TF32-class floor {floor:.3e}  bar {_bar(floor):.3e}")
    assert err <= _bar(floor), f"{name}: eps rel {err:.3e} > bar {_bar(floor):.3e} (floor {floor:.3e})"


@pytest.mark.parametrize("tag", UNET_TAGS)
def test_unet_any_width_vs_reference_golden(wid, tag):
    cfg = _cfg(wid, tag)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    net = _load(cfg, sd)
    x, t, c = _T(wid, tag, "x"), _T(wid, tag, "t"), _T(wid, tag, "c")
    ref = _T(wid, tag, "eps")
    got = net(x.cuda(), t.cuda(), c.cuda())
    assert got.shape == ref.shape
    if tag == "legacy96":
        # plain resampling layers and use_scale_shift_norm=False are outside the precision model: the bar of
        # test_backbone_options
        r = G.report(f"{tag} eps", got, ref)
        assert r < HARD_CAP
    else:
        _check(f"{tag} eps", got, ref, PM.rel(PM.forward(cfg, sd, x, t, c, PM.TF32_CLASS), ref))
    taps = {}
    unet_ref.unet_forward(cfg, sd, x, t, c, taps=taps)
    blocks, _ = unet_ref._topology(cfg)
    worst = 0.0
    for name in [l[1] for b in blocks for l in b["layers"] if l[0] != "conv"]:
        got_t = _tap(net, x.shape[0], name)
        assert got_t.shape == taps[name].shape, name
        r = G.rel(got_t, taps[name])
        print(f"[tap] {tag} {name} C{got_t.shape[1]} rel {r:.3e}")
        worst = max(worst, r)
    assert worst < HARD_CAP


def test_inpaint_model_inference_vs_reference_golden(wid):
    cfg = _cfg(wid, "inpaint96")
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    fw = frameworks.InpaintCFG(_load(cfg, sd), timesteps=1000, beta_schedule="linear")
    g = lambda k: _T(wid, "inpaint96", k)
    ref = g("eps")
    got = fw.model_inference(g("x").cuda(), g("t").cuda(), g("y").cuda(), g("mask").cuda(), g("c").cuda(), strength=STRENGTH,
                             noise=g("noise").cuda(), mask_rgb=g("mask_rgb").cuda())
    noise = g("noise")
    ci = sampler_ref.make_inpaint_inputs(g("x"), g("y"), g("mask"), g("mask_rgb"), noise[:, :3], noise[:, 3:])
    pm = lambda xx, tt, cc: PM.forward(cfg, sd, xx, tt, cc, PM.TF32_CLASS)
    _check("inpaint96 eps", got, ref, PM.rel(sampler_ref.cond_eps(pm, ci, g("t"), g("c"), STRENGTH), ref))


@pytest.mark.parametrize("tag", UNET_TAGS)
def test_any_width_deterministic_and_batch_invariant(wid, tag):
    cfg = _cfg(wid, tag)
    net = _load(cfg, unet_ref.make_synthetic_state_dict(cfg, seed=77))
    N = 8
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, 4, 32, 32, generator=g).cuda()
    t = torch.arange(N, device="cuda") * 120 + 3; c = torch.arange(N, device="cuda") % 10
    first = net(x, t, c).clone()
    assert torch.isfinite(first).all()
    bad = sum(0 if torch.equal(net(x, t, c), first) else 1 for _ in range(5))
    assert bad == 0, f"{bad} of 5 forwards differ from the first"
    for i in (0, 5):
        one = net(x[i:i + 1].contiguous(), t[i:i + 1], c[i:i + 1])
        assert torch.equal(one, first[i:i + 1]), f"sample {i}: eps depends on the batch"


# ------------------------------------------------------------------------------------------------------------------
# samplers
# ------------------------------------------------------------------------------------------------------------------
def _kernel_names(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {e.name for e in prof.events()}


def test_fused_head_step_at_final_width_96(wid):
    """Final width 96 keeps the tap-column output head, so the production loop ends every forward in
    step_kernel<HeadTaps, Update<kind>>; with return_trajectory=True it takes eps_gather_kernel + step_kernel<EpsRows, ...>
    instead.  Same Philox draws -> the same bits."""
    cfg = _cfg(wid, "mc96")
    fw = frameworks.ClassifierFreeGuidance(_load(cfg, unet_ref.make_synthetic_state_dict(cfg, seed=77)), timesteps=1000,
                                           beta_schedule="linear")
    rng = np.random.default_rng(2)
    x = torch.from_numpy(rng.standard_normal((2, 4, 32, 32)).astype(np.float32)).cuda()
    classes = torch.tensor([1, 2]).cuda()
    for s, kw in ((samplers.DdimSampler(fw), dict(steps=8, eta=1.0)), (samplers.DdpmSampler(fw), dict())):
        torch.manual_seed(5)
        # the first forward of a plan runs eagerly, so its kernels are visible to the profiler by name
        a, fused = _kernel_names(lambda: s.sample(2, noise=x, classes=classes, strength=0.5, verbose=False, **kw).samples)
        torch.manual_seed(5)
        b, separate = _kernel_names(lambda: s.sample(2, noise=x, classes=classes, strength=0.5, verbose=False,
                                                     return_trajectory=True, **kw))
        assert any("step_kernel<ivid::HeadTaps" in n for n in fused), "the fused head step is not active at final width 96"
        assert not any("step_kernel<ivid::HeadTaps" in n for n in separate)
        assert any("eps_gather_kernel" in n for n in separate)
        G.report(f"{type(s).__name__}: fused head+step vs separate kernels at width 96", a, b.samples)
        assert torch.isfinite(a).all()
        assert torch.equal(a, b.samples)


def test_inpaint_ddim_guided_steps_mc96(wid):
    """A short DDIM run of InpaintCFG at model_channels=96 with injected hole noise and the multiview guidance terms,
    teacher-forced against the oracle at every step."""
    cfg = _cfg(wid, "inpaint96")
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    fw = frameworks.InpaintCFG(_load(cfg, sd), timesteps=1000, beta_schedule="linear")
    s = samplers.DdimSampler(fw)
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", 1000))
    model = lambda xx, tt, cc: unet_ref.unet_forward(cfg, sd, xx, tt, cc)
    g = lambda k: _T(wid, "inpaint96", k)
    y, mask, mask_rgb, classes = g("y"), g("mask"), g("mask_rgb"), g("c")
    convex = torch.from_numpy(np.random.default_rng(3).uniform(-1, 1, (2, 1, 32, 32)).astype(np.float32))
    rng = np.random.default_rng(4)
    xo = g("x")
    worst = 0.0
    for (tt, tp) in sampler_ref.ddim_schedule(1000, 4):
        t = torch.tensor([tt] * 2); tpv = torch.tensor([tp] * 2)
        cn = torch.from_numpy(rng.standard_normal((2, 4, 32, 32)).astype(np.float32))
        ci = sampler_ref.make_inpaint_inputs(xo, y, mask, mask_rgb, cn[:, :3], cn[:, 3:])
        eps = sampler_ref.cond_eps(model, ci, t - 1, classes, STRENGTH)
        ref, _ = sampler_ref.ddim_step(tb, xo, t, tpv, eps, torch.zeros_like(xo), replace_rgb=(0.1, y[:, :3], mask_rgb),
                                       replace_depth=(0.2, y[:, 3:], mask), constrain_depth=(0.5, convex))
        yc, mc, mrc = y.cuda(), mask.cuda(), mask_rgb.cuda()
        out = s.sample_once(xo.cuda(), t.cuda(), tpv.cuda(), classes.cuda(), strength=STRENGTH, y=yc, mask=mc, mask_rgb=mrc,
                            replace_rgb=(0.1, yc[:, :3], mrc), replace_depth=(0.2, yc[:, 3:], mc),
                            constrain_depth=(0.5, convex.cuda()), noise=torch.zeros_like(xo).cuda(), cond_noise=cn.cuda())
        worst = max(worst, G.report(f"inpaint96 ddim-4 {tt}->{tp}", out.pred_x_prev, ref))
        xo = ref
    assert worst < STEP_TOL

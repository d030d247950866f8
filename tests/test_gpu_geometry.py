"""GPU: AdmUnet2d, the ops and the samplers at input sizes other than a square power of two — the conv op at layer sizes whose
tiles are smaller than before, both attention ops at sequence lengths that are not multiples of 64, the network and the
super-resolution framework against the unmodified reference (geometry_golden.npz), per-block taps, determinism, the plan
cache, the error contract and the samplers.  Eps bars follow tests/test_gpu_unet.py (_bar of the TF32-class floor)."""
import ctypes
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
UNET_TAGS = ["np2", "np2_single", "short", "rect", "big"]
SR_TAGS = ["sr4", "sr3"]
SR_STRENGTH = 0.5


def _bar(floor):
    return min(max(NORTH_STAR, 1.15 * floor), HARD_CAP)


@pytest.fixture(scope="module")
def geo():
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "geometry_golden.npz")))


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
@pytest.mark.parametrize("H,W", [(12, 20), (24, 24), (6, 10), (48, 80), (3, 5)])
@pytest.mark.parametrize("k", [3, 1])
def test_conv_any_size_matches_torch(H, W, k):
    """conv(a) + skip(x) as a second K segment + residual, fp32 and fp16 outputs; bars of test_conv_matches_torch."""
    g = torch.Generator().manual_seed(H * 100 + W + k)
    N, C, Cx, Co = 3, 64, 64, 128
    a = torch.randn(N, C, H, W, generator=g); x = torch.randn(N, Cx, H, W, generator=g)
    w = torch.randn(Co, C, k, k, generator=g) / math.sqrt(C * k * k); b = 0.1 * torch.randn(Co, generator=g)
    w2 = torch.randn(Co, Cx, 1, 1, generator=g) / math.sqrt(Cx); b2 = 0.1 * torch.randn(Co, generator=g)
    res = torch.randn(N, Co, H, W, generator=g)
    ah, xh = a.half(), x.half()
    ref16 = F.conv2d(ah.float(), w.half().float(), b, padding=k // 2) + F.conv2d(xh.float(), w2.half().float(), b2) + res
    ref32 = F.conv2d(a, w, b, padding=k // 2) + F.conv2d(x, w2, b2) + res
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().cuda()
    for out16 in (False, True):
        out = G.conv2d(nhwc(ah), w, b, k, act2=nhwc(xh), w2=w2.reshape(Co, Cx), b2=b2, residual=nhwc(res), out_fp16=out16)
        got = out.float().permute(0, 3, 1, 2).cpu()
        r16 = G.report(f"conv N{N} {H}x{W} k{k} fp16-out={out16} (vs fp16-rounded operands)", got, ref16)
        r32 = G.report(f"conv N{N} {H}x{W} k{k} fp16-out={out16} (vs fp32)", got, ref32)
        assert r32 < 2e-3
        if not out16:
            assert r16 < 2e-5


def _torch_attention(qh, C, d):
    """QKVAttention (adm.py:233-253) in fp32 on the fp16 inputs, qh [N, 3C, T]."""
    N, _, T = qh.shape
    q, k, v = qh.float().reshape(N * (C // d), 3 * d, T).split(d, dim=1)
    s = 1 / math.sqrt(math.sqrt(d))
    w = torch.softmax(torch.einsum("bct,bcs->bts", q * s, k * s), dim=-1)
    return torch.einsum("bts,bcs->bct", w, v).reshape(N, C, T)


@pytest.mark.parametrize("d", [64, 128, 192, 512])
@pytest.mark.parametrize("T", [1, 15, 16, 36, 60, 100, 144, 240, 576, 1000])
def test_attention_any_length_matches_torch(T, d):
    C = 2 * d if d < 512 else d
    N = 2
    qh = torch.randn(N, 3 * C, T, generator=torch.Generator().manual_seed(T * 7 + d)).half()
    ref = _torch_attention(qh, C, d)
    qkv = qh.permute(0, 2, 1).contiguous().cuda()
    outs = {}
    out = torch.empty((N, T, C), dtype=torch.float16, device="cuda")
    _lib.check(_lib.lib().ivid_op_attention_heads(_lib.ptr(qkv), N, T, C, d, _lib.ptr(out), _lib.cur_stream()))
    outs["heads"] = out
    if d == 64:
        outs["attention"] = G.attention(qkv, C)
        assert torch.equal(outs["attention"], outs["heads"])
    for name, o in outs.items():
        assert torch.isfinite(o.float()).all()
        assert G.report(f"{name} N{N} T{T} C{C} d{d}", o.float().permute(0, 2, 1), ref) < 2e-3


# ------------------------------------------------------------------------------------------------------------------
# network and framework against the reference
# ------------------------------------------------------------------------------------------------------------------
def _tap(net, N, name):
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
def test_unet_any_size_vs_reference_golden(geo, tag):
    cfg = _cfg(geo, tag)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    net = _load(cfg, sd)
    x, t, c = _T(geo, tag, "x"), _T(geo, tag, "t"), _T(geo, tag, "c")
    ref = _T(geo, tag, "eps")
    got = net(x.cuda(), t.cuda(), c.cuda())
    assert got.shape == ref.shape
    _check(f"{tag} eps", got, ref, PM.rel(PM.forward(cfg, sd, x, t, c, PM.TF32_CLASS), ref))
    if tag not in ("rect", "np2"):
        return
    # every block output: covers the up-ResBlocks' upsampled residual at the 24- and 12-wide levels
    taps = {}
    unet_ref.unet_forward(cfg, sd, x, t, c, taps=taps)
    blocks, _ = unet_ref._topology(cfg)
    worst = 0.0
    for name in [l[1] for b in blocks for l in b["layers"]]:
        got_t = _tap(net, x.shape[0], name)
        assert got_t.shape == taps[name].shape, name
        r = G.rel(got_t, taps[name])
        print(f"[tap] {tag} {name} {tuple(got_t.shape[2:])} rel {r:.3e}")
        worst = max(worst, r)
    assert worst < HARD_CAP


@pytest.mark.parametrize("tag", SR_TAGS)
def test_superres_any_scale_vs_reference_golden(geo, tag):
    cfg = _cfg(geo, tag)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    fw = frameworks.SuperResCFG(_load(cfg, sd), timesteps=1000, beta_schedule="linear")
    x, y, t, c = _T(geo, tag, "x"), _T(geo, tag, "y"), _T(geo, tag, "t"), _T(geo, tag, "c")
    ref = _T(geo, tag, "eps")
    got = fw.model_inference(x.cuda(), t.cuda(), y.cuda(), c.cuda(), strength=SR_STRENGTH)
    pm = lambda xx, tt, cc: PM.forward(cfg, sd, xx, tt, cc, PM.TF32_CLASS)
    floor = PM.rel(sampler_ref.cond_eps(pm, sampler_ref.make_sr_inputs(x, y), t, c, SR_STRENGTH), ref)
    _check(f"{tag} eps", got, ref, floor)


# ------------------------------------------------------------------------------------------------------------------
# determinism, plan cache, error contract
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag,H,W", [("rect", 40, 24), ("np2", 48, 48)])
def test_any_size_deterministic_and_batch_invariant(geo, tag, H, W):
    cfg = _cfg(geo, tag)
    net = _load(cfg, unet_ref.make_synthetic_state_dict(cfg, seed=77))
    N = 8
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, 4, H, W, generator=g).cuda()
    t = torch.arange(N, device="cuda") * 120 + 3; c = torch.arange(N, device="cuda") % 10
    first = net(x, t, c).clone()
    bad = sum(0 if torch.equal(net(x, t, c), first) else 1 for _ in range(10))
    assert bad == 0, f"{bad} of 10 forwards differ from the first"
    for i in (0, 5):
        one = net(x[i:i + 1].contiguous(), t[i:i + 1], c[i:i + 1])
        assert torch.equal(one, first[i:i + 1]), f"sample {i}: eps depends on the batch"


def test_plan_cache_alternating_sizes(geo):
    cfg = _cfg(geo, "rect")
    net = _load(cfg, unet_ref.make_synthetic_state_dict(cfg, seed=77))
    g = torch.Generator().manual_seed(9)
    xa = torch.randn(2, 4, 32, 32, generator=g).cuda(); xb = torch.randn(2, 4, 40, 24, generator=g).cuda()
    t = torch.tensor([500, 20], device="cuda"); c = torch.tensor([1, -1], device="cuda")
    a0 = net(xa, t, c).clone()
    b0 = net(xb, t, c).clone()
    assert b0.shape == (2, 4, 40, 24)
    a1 = net(xa, t, c)
    assert torch.equal(a0, a1)
    assert _tap(net, 2, "input_blocks.0.0").shape == (2, 64, 32, 32)       # the tap follows the latest forward of batch 2
    net(xb, t, c)
    assert _tap(net, 2, "input_blocks.0.0").shape == (2, 64, 40, 24)


def test_geometry_error_contract(geo):
    """The reference fails in torch.cat (RuntimeError) when a size is not divisible by 2^(levels-1)."""
    cfg = _cfg(geo, "short")                       # three downsamples
    net = _load(cfg, unet_ref.make_synthetic_state_dict(cfg, seed=77))
    t = torch.tensor([5], device="cuda")
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 4, 36, 36, device="cuda"), t)
    cfg2 = _cfg(geo, "rect")                       # two downsamples
    net2 = _load(cfg2, unet_ref.make_synthetic_state_dict(cfg2, seed=77))
    with pytest.raises(RuntimeError):
        net2(torch.zeros(1, 4, 30, 30, device="cuda"), t)
    with pytest.raises(AssertionError):
        net2(torch.zeros(1, 3, 32, 32, device="cuda"), t)
    assert net2(torch.zeros(1, 4, 32, 32, device="cuda"), t).shape == (1, 4, 32, 32)    # still usable afterwards


# ------------------------------------------------------------------------------------------------------------------
# samplers
# ------------------------------------------------------------------------------------------------------------------
SAMPLER_CASES = [("rect", (40, 24)), ("np2", (48, 48))]


def _sampler_setup(geo, tag):
    cfg = _cfg(geo, tag)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    fw = frameworks.ClassifierFreeGuidance(_load(cfg, sd), timesteps=1000, beta_schedule="linear")
    model = lambda xx, tt, cc: unet_ref.unet_forward(cfg, sd, xx, tt, cc)
    return fw, model, sampler_ref.Tables(sampler_ref.get_betas("linear", 1000))


@pytest.mark.parametrize("tag,hw", SAMPLER_CASES)
def test_ddpm_sample_once_any_size(geo, tag, hw):
    fw, model, tb = _sampler_setup(geo, tag)
    s = samplers.DdpmSampler(fw)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, *hw, generator=g); z = torch.randn(2, 4, *hw, generator=g)
    classes = torch.tensor([2, 9])
    for ti in (999, 400, 0):
        t = torch.tensor([ti, ti])
        eps = sampler_ref.cfg_eps(model, x, t, classes, 0.5)
        ref, _ = sampler_ref.ddpm_step(tb, x, t, eps, z)
        out = s.sample_once(x.cuda(), t.cuda(), classes.cuda(), strength=0.5, noise=z.cuda())
        assert out.pred_x_prev.shape == (2, 4) + hw
        assert G.report(f"ddpm {tag} {hw} t={ti}", out.pred_x_prev, ref) < STEP_TOL


@pytest.mark.parametrize("tag,hw", SAMPLER_CASES)
def test_ddim_sample_torch_rng_teacher_forced(geo, tag, hw):
    """DdimSampler.sample(rng="torch", return_trajectory=True) for 5 steps; every step against the oracle's step from the
    sampler's own previous x_t (eta = 0: the step noise has no effect).  The 48 model is sampled through image_size=48."""
    fw, model, tb = _sampler_setup(geo, tag)
    s = samplers.DdimSampler(fw)
    classes = torch.tensor([2, 9])
    torch.manual_seed(21)
    if hw[0] == hw[1]:
        res = s.sample(2, image_size=hw[0], classes=classes.cuda(), steps=5, strength=0.5, verbose=False, rng="torch",
                       return_trajectory=True)
        torch.manual_seed(21)
        x = torch.randn((2, 4) + hw, device="cuda").cpu()
    else:
        x = torch.randn((2, 4) + hw)
        res = s.sample(2, noise=x.cuda(), classes=classes.cuda(), steps=5, strength=0.5, verbose=False, rng="torch",
                       return_trajectory=True)
    assert res.samples.shape == (2, 4) + hw and len(res.pred_x_t) == 5
    worst = 0.0
    xo = x
    for i, (tt, tp) in enumerate(sampler_ref.ddim_schedule(1000, 5)):
        t = torch.tensor([tt] * 2); tpv = torch.tensor([tp] * 2)
        eps = sampler_ref.cfg_eps(model, xo, t - 1, classes, 0.5)
        ref, _ = sampler_ref.ddim_step(tb, xo, t, tpv, eps, torch.zeros_like(xo))
        worst = max(worst, G.report(f"ddim-5 {tag} {hw} {tt}->{tp}", res.pred_x_t[i], ref))
        xo = res.pred_x_t[i].cpu()
    assert worst < STEP_TOL
    assert torch.equal(res.samples, res.pred_x_t[-1])


def test_philox_sample_non_square_noise(geo):
    fw, _, _ = _sampler_setup(geo, "rect")
    s = samplers.DdimSampler(fw)
    noise = torch.randn(2, 4, 40, 24, generator=torch.Generator().manual_seed(4)).cuda()
    classes = torch.tensor([3, 5], device="cuda")
    torch.manual_seed(8)
    a = s.sample(2, noise=noise, classes=classes, steps=4, strength=0.5, verbose=False).samples
    torch.manual_seed(8)
    b = s.sample(2, noise=noise, classes=classes, steps=4, strength=0.5, verbose=False).samples
    assert a.shape == (2, 4, 40, 24)
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)

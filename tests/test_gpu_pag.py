"""GPU: perturbed-attention guidance (PAG).  Bitwise unless a tolerance is stated.

- the attention op's perturbed rows are the V channels, and its other rows the op over those rows alone;
- forward_perturbed against the float64 model (tests/pag_ref.py) within the eps bar of tests/test_gpu_unet.py, per layer
  within HARD_CAP;
- a 3N forward: rows [0, 2N) are today's 2N CFG forward and rows [2N, 3N) forward_perturbed, deterministic and
  batch-invariant; with InpaintCFG the perturbed rows take the conditional rows' assembly and hole noise; a PAG plan's reuse
  forward reads its own feature cache;
- steps of every kind against the float64 mix plus update (5e-6), with the host and device routes equal;
- the separate route (EpsRows), the fused route (HeadTaps) and, with dynamic thresholding, the thresholded routes agree, with
  and without classes;
- runs: sample(rng="torch") equals chained sample_once, also with InpaintCFG and the multiview guidance, SuperResCFG, fp8
  and feature reuse; pag_scale=0 and an interval that excludes every step give the run without PAG; the profiled conv FLOPs
  of a PAG step are 1.5x / 2x those of a step without."""
import ctypes
import json

import numpy as np
import pytest
import torch

import gpu_util as G
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
import pag_ref
from ivid_b200 import _lib
from ivid_b200.inference import build_modelviews, sample_all
from oracle import unet_ref

import precision_model as PM

pytestmark = pytest.mark.gpu
NORTH_STAR = 1e-3
HARD_CAP = 1.6e-3


def _bar(floor):
    # the eps bar of tests/test_gpu_unet.py
    return min(max(NORTH_STAR, 1.15 * floor), HARD_CAP)
T = 1000
S = 0.5
W = 1.5


def _randn(seed, shape):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal(shape).astype(np.float32)).cuda()


def _cfg(golden, tag):
    key = f"{tag}_cfg" if f"{tag}_cfg" in golden else f"schemacfg_{tag}"
    return json.loads(bytes(golden[key]).decode())


def _net(cfg, seed=1234):
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    return net.cuda()


def _fw(golden, tag, cls, seed=1234):
    return cls(_net(_cfg(golden, tag), seed), timesteps=T, beta_schedule="linear")


# ---------------------------------------------------------------------------------------------------------------- op
@pytest.mark.parametrize("d", [64, 128, 192, 512])
@pytest.mark.parametrize("Tq", [64, 256, 1024, 100])
def test_attention_op_rows(d, Tq):
    N, C = 3, 2 * d if d < 512 else 512
    L = _lib.lib()
    qkv = (torch.randn(N, Tq, 3 * C, device="cuda") * 0.5).half().contiguous()
    ref = torch.empty(N, Tq, C, dtype=torch.float16, device="cuda")
    _lib.check(L.ivid_op_attention_heads(_lib.ptr(qkv), N, Tq, C, d, _lib.ptr(ref), _lib.cur_stream()))
    v = torch.cat([qkv[..., 3 * d * h + 2 * d: 3 * d * h + 3 * d] for h in range(C // d)], dim=-1)
    for row0 in (0, 1, 2, N):
        out = torch.full((N, Tq, C), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(L.ivid_op_attention_perturbed(_lib.ptr(qkv), N, Tq, C, d, row0, _lib.ptr(out), _lib.cur_stream()))
        assert torch.equal(out[row0:], v[row0:]), f"identity rows differ from V (row0={row0})"
        if row0 > 0:
            alone = torch.empty(row0, Tq, C, dtype=torch.float16, device="cuda")
            q0 = qkv[:row0].contiguous()
            _lib.check(L.ivid_op_attention_heads(_lib.ptr(q0), row0, Tq, C, d, _lib.ptr(alone), _lib.cur_stream()))
            assert torch.equal(out[:row0], alone)
            assert torch.equal(out[:row0], ref[:row0])


# ----------------------------------------------------------------------------------------------------------- forward
def _tap(net, N, name):
    L = _lib.lib()
    C, H, W_ = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), None, 0, ctypes.byref(C), ctypes.byref(H), ctypes.byref(W_)))
    out = torch.empty((N, C.value, H.value, W_.value), dtype=torch.float32)
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), _lib.ptr(out), out.numel(), None, None, None))
    return out


def _layer_sets(cfg):
    names = pag_ref.attention_layers(cfg)
    ins = [n for n in names if n.startswith("input")]
    outs = [n for n in names if n.startswith("output")]
    return [("middle", ("middle_block.1",)), ("span", tuple(ins[-1:] + ["middle_block.1"] + outs[:1]))]


@pytest.mark.parametrize("tag", ["tiny", "rgbd_imagenet_adm_128_large_cfg"])
def test_forward_perturbed_vs_model(golden, tag):
    cfg = _cfg(golden, tag)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    net = _net(cfg)
    S_ = cfg["image_size"]
    x = torch.from_numpy(np.random.default_rng(5).standard_normal((2, cfg["in_channels"], S_, S_)).astype(np.float32))
    t = torch.tensor([700, 120]); c = torch.tensor([3, -1]) if cfg.get("num_classes") else None
    plain = unet_ref.unet_forward(cfg, sd, x, t, c)
    # the TF32-class floor of the network (precision_model has no perturbed form; an identity layer drops the softmax
    # roundings, so the unperturbed floor does not understate the perturbed one)
    bar = _bar(PM.rel(PM.forward(cfg, sd, x, t, c, PM.TF32_CLASS), plain))
    for label, layers in _layer_sets(cfg):
        taps = {}
        ref = pag_ref.perturbed_forward(cfg, sd, x, t, c, layers, taps=taps)
        got = net.forward_perturbed(x.cuda(), t.cuda(), c.cuda() if c is not None else None, layers=layers)
        err = G.report(f"{tag} {label} perturbed eps", got, ref)
        print(f"[parity] {tag} {label}: bar {bar:.3e}")
        assert err <= bar, f"{tag} {label}: {err:.3e} > bar {bar:.3e}"
        assert G.rel(ref, plain) > 2 * err, "the perturbation must move eps by more than the kernels' error"
        worst = max(G.rel(_tap(net, 2, n), w) for n, w in taps.items() if n != "emb")
        assert worst <= HARD_CAP, f"{tag} {label}: worst tap {worst:.3e}"


def test_row_isolation_3n(golden):
    cfg = _cfg(golden, "rgbd_imagenet_adm_128_large_cfg")
    net = _net(cfg)
    L = _lib.lib()
    N, S_ = 2, cfg["image_size"]
    x = _randn(7, (N, 4, S_, S_))
    t = torch.tensor([500, 500], device="cuda")
    c = torch.tensor([1, 7], device="cuda")
    layers = ("middle_block.1",)
    net._ensure_packed()
    idx = net.pag_layer_indices(layers)
    arr = (ctypes.c_int * 1)(*idx)
    t3 = t.repeat(3).contiguous(); c3 = torch.cat([c, torch.full_like(c, -1), c]).contiguous()

    def f3():
        out = torch.empty(3 * N, 4, S_, S_, device="cuda")
        _lib.check(L.ivid_unet_forward_perturbed(net._handle, _lib.ptr(x), N, S_, S_, None, _lib.ptr(t3), _lib.ptr(c3), _lib.ptr(out),
                                                 3 * N, 2 * N, arr, 1, -1, _lib.cur_stream()))
        return out
    a = f3()
    two = torch.empty(2 * N, 4, S_, S_, device="cuda")
    _lib.check(L.ivid_unet_forward_hw(net._handle, _lib.ptr(x), N, S_, S_, None, _lib.ptr(t3[:2 * N].contiguous()),
                                      _lib.ptr(c3[:2 * N].contiguous()), _lib.ptr(two), 2 * N, _lib.cur_stream()))
    assert torch.equal(a[:2 * N], two)
    assert torch.equal(a[2 * N:], net.forward_perturbed(x, t, c, layers=layers))
    for _ in range(9):
        assert torch.equal(f3(), a)
    # batch invariance: the perturbed rows of one sample alone
    one = net.forward_perturbed(x[1:], t[1:], c[1:], layers=layers)
    assert torch.equal(a[2 * N + 1:], one)


# ------------------------------------------------------------------------------------------------------------- mix
@pytest.mark.parametrize("cfg,s", [(0, 0.0), (1, S), (2, -0.3)])
def test_guidance_mix_matches_fp32_model(cfg, s):
    n = 4 * 32 * 32 * 3
    blocks = 3 if cfg == 1 else 2
    eps = _randn(11, (blocks * n,))
    out = torch.empty(n, device="cuda")
    _lib.check(_lib.lib().ivid_guidance_mix(_lib.ptr(eps), n, cfg, s, 1, W, _lib.ptr(out), _lib.cur_stream()))
    e = eps.cpu().numpy()
    ec, ep = e[:n], e[(blocks - 1) * n:]
    eu = e[n:2 * n] if cfg == 1 else None
    assert np.array_equal(out.cpu().numpy(), pag_ref.mix32(ec, ep, W, cfg, s, eu))


# ----------------------------------------------------------------------------------------------------------- steps
KINDS = {
    "ddpm": (samplers.DdpmSampler, {}),
    "ddim": (samplers.DdimSampler, dict(eta=1.0)),
    "dpm_ode": (samplers.DpmSolverSampler, {}),
    "dpm_sde": (samplers.DpmSolverSampler, dict(sde=True)),
    "unipc": (samplers.UniPcSampler, {}),
}


def _once(s, x, t, tp, classes, **kw):
    N = x.shape[0]
    tt = torch.full((N,), t, device="cuda")
    if s.KIND == 0:
        return s.sample_once(x, tt, classes, **kw)
    return s.sample_once(x, tt, torch.full((N,), tp, device="cuda"), classes, **kw)


def _tables(fw):
    acp = np.cumprod(1.0 - np.asarray(fw.betas, np.float64))
    return acp


def _eps64(net, x, tm, classes, cfg, s=S, w=W):
    """The float64 mix of the fp32 rows the step's forward computes (the forward is row-isolated and batch-invariant)."""
    N = x.shape[0]
    tt = torch.full((N,), tm, device="cuda")
    ec = net(x, tt, classes)
    ep = net.forward_perturbed(x, tt, classes)
    eu = net(x, tt, torch.full((N,), -1, device="cuda")) if cfg == 1 else None
    return pag_ref.torch_mix64(ec, ep, w, cfg, s, eu).numpy()


STEP_TOL = 5e-6


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("classes_on", [True, False])
def test_step_matches_float64_and_host_route(golden, kind, classes_on):
    """One PAG step of every kind (second order / with history where the kind has one) against the float64 mix of the
    forward's eps rows plus the kind's float64 update (oracle/dpm_ref.py, tests/dpm_sde_ref.py, tests/unipc_ref.py), within
    5e-6 of the sample's scale (fp32 coefficients and fp32 arithmetic of the mix and the update).  The device-timestep route
    (sample_once) and the host-int route (ivid_sampler_step) give the same bits."""
    import dpm_sde_ref
    import unipc_ref
    from oracle import dpm_ref
    cls, kw = KINDS[kind]
    fw = _fw(golden, "tiny", frameworks.ClassifierFreeGuidance)
    s = cls(fw)
    net = fw.backbone
    N = 2
    x = _randn(3, (N, 4, 32, 32))
    z = _randn(4, (N, 4, 32, 32))
    d_prev = _randn(6, (N, 4, 32, 32)) * 0.5
    base = _randn(7, (N, 4, 32, 32))
    classes = torch.tensor([1, 2], device="cuda") if classes_on else None
    cfg = 1 if classes_on else 0
    acp = _tables(fw)
    t, tp, t_last = (400, 0, None) if kind == "ddpm" else (600, 580, 620)
    tm = t if kind == "ddpm" else t - 1
    eps = _eps64(net, x, tm, classes, cfg)
    x64, z64 = x.double().cpu().numpy(), z.double().cpu().numpy()
    dp64, b64 = d_prev.double().cpu().numpy(), base.double().cpu().numpy()
    k = dict(strength=S, pag_scale=W, noise=z)
    host_kw = {}
    if kind == "ddpm":
        x0 = s.sqrt_recip_alphas_cumprod[t] * x64 - s.sqrt_recipm1_alphas_cumprod[t] * eps
        want = s.posterior_mean_coef1[t] * x0 + s.posterior_mean_coef2[t] * x64 + \
            (1.0 if t != 0 else 0.0) * np.exp(0.5 * s.posterior_log_variance_clipped[t]) * z64
    elif kind == "ddim":
        eta = kw["eta"]
        k["eta"] = eta
        ab, abp = acp[t - 1], acp[tp - 1]
        x0 = np.sqrt(1 / ab) * x64 - np.sqrt(1 / ab - 1) * eps
        sigma = eta * np.sqrt((1 - abp) / (1 - ab)) * np.sqrt(1 - ab / abp)
        want = np.sqrt(abp) * x0 + np.sqrt(1 - abp - sigma ** 2) * eps + sigma * z64
        host_kw = dict(eta=eta)
    elif kind == "dpm_ode":
        want = dpm_ref.step(acp, x64, t, tp, eps, dp64, t_last)[0]
        k.update(prev=(t_last, d_prev))
        host_kw = dict(order=2, prev=(t_last, d_prev))
    elif kind == "dpm_sde":
        want = dpm_sde_ref.sde_step(acp, x64, t, tp, eps, z64, dp64, t_last)[0]
        k.update(prev=(t_last, d_prev), sde=True)
        host_kw = dict(order=2, prev=(t_last, d_prev), sde=True)
    else:
        d0 = dpm_ref.guided_x0(acp, x64, t, tp, eps)
        want = unipc_ref.step(acp, x64, d0, t, tp, 2, 1, hist=[(t_last, dp64)], base=b64)[0]
        k.update(prev=[(t_last, d_prev)], prev_x=base, order=2)
        k.pop("noise")
        host_kw = dict(order=2, prev=[(t_last, d_prev)], prev_x=base)
    out = _once(s, x, t, tp, classes, **k)
    err = float(np.abs(out.pred_x_prev.double().cpu().numpy() - want).max() / np.abs(want).max())
    print(f"[pag] {kind} classes={classes_on} step vs float64: {err:.3e}")
    assert err < STEP_TOL
    pag = (W, net.pag_layer_indices(["middle_block.1"]))
    eta = host_kw.pop("eta", 0.0)
    noise = None if kind in ("dpm_ode", "unipc") else z
    host = s._native_step(x, t, tp, classes, False, eta, dict(strength=S), noise, None, pag=pag, **host_kw)
    assert torch.equal(out.pred_x_prev, host.pred_x_prev) and torch.equal(out.pred_x_0, host.pred_x_0)


def _grid(s, steps, start):
    """(t, t_prev) of the executed steps of ivid_sampler_run, in order."""
    if s.KIND == 0:
        return [(T - 1 - i, 0) for i in range(start, T)]
    jump = T // steps
    return [(jump * (steps - i), jump * (steps - 1 - i)) for i in range(start, steps)]


def _run_injected(s, x, classes, steps, noise_all, start=0, threshold=None, cond_noise_all=None, eta=0.0, sde=False,
                  cache_interval=0, **kw):
    """ivid_sampler_run with the per-step draws injected: the host-int route with the separate step kernel
    (step_kernel<EpsRows, ...>), since per-step noise pointers rule out the fused head step."""
    net = s._net()
    img = x.clone().contiguous()
    pag = (kw.pop("pag_scale"), net.pag_layer_indices(kw.pop("pag_layers", ["middle_block.1"])))
    a, keep = s._step_args(img.device, classes, False, eta, kw, seed=0, hw=img.shape[-2:], order=2, sde=sde,
                           threshold=threshold, pag=pag, cache=(cache_interval, 0, 0))
    a.start_step = start
    ca = cond_noise_all.contiguous() if cond_noise_all is not None else None
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().ivid_sampler_run(s._handle, net._handle, _lib.ptr(img), img.shape[0], steps, ctypes.byref(a),
                                               _lib.ptr(noise_all.contiguous()), _lib.ptr(ca), None, None,
                                               _lib.cur_stream(img.device)))
    torch.cuda.synchronize()
    del keep
    return img


def _chain(s, x, classes, grid, noise_all=None, cond_noise_all=None, eta=0.0, sde=False, reuse=None, **kw):
    """Chained sample_once calls (device-timestep route, fused head step) over `grid`, with the history a run keeps; noise
    injected per step, or drawn by sample_once as sample(rng="torch") draws it when noise_all is None."""
    xa, prev, prev_x = x.clone(), None, None
    for i, (t, tp) in enumerate(grid):
        k = dict(kw)
        if noise_all is not None:
            k["noise"] = noise_all[i]
        if cond_noise_all is not None:
            k["cond_noise"] = cond_noise_all[i]
        if reuse is not None:
            k["reuse_features"] = reuse[i]
        if s.KIND == 1:
            k["eta"] = eta
        if s.KIND == 2 and not s.UNIPC:
            k.update(prev=prev, sde=sde)
        if s.UNIPC:
            k.update(prev=prev, prev_x=prev_x)
        out = _once(s, xa, t, tp, classes, **k)
        if s.KIND == 2 and not s.UNIPC:
            prev = (t, out.pred_x_0)
        if s.UNIPC:
            prev, prev_x = ([(t, out.pred_x_0)] + (prev or []))[:2], out.corrected_x_t
        xa = out.pred_x_prev
    return xa


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("threshold", [None, 0.9])
@pytest.mark.parametrize("model", ["cfg", "single_category"])
def test_routes_agree(golden, kind, threshold, model):
    """The separate route (ivid_sampler_run with injected noise: step_kernel<EpsRows, ...>) equals chained sample_once
    calls (the fused head step, step_kernel<HeadTaps, ...>) with PAG, bit for bit; with dynamic thresholding both run the
    thresholded route (StoreX0 from either source, then ThresholdedX0).  `single_category`: a GaussianDiffusion without
    classes, whose only guidance is PAG.  DDPM runs the last 8 of its 1000 steps (start_step)."""
    cls, kw = KINDS[kind]
    fw_cls = frameworks.ClassifierFreeGuidance if model == "cfg" else frameworks.GaussianDiffusion
    s = cls(_fw(golden, "tiny", fw_cls))
    N = 2
    x = _randn(1, (N, 4, 32, 32))
    classes = torch.tensor([1, 2], device="cuda") if model == "cfg" else None
    steps, start = (T, T - 8) if kind == "ddpm" else (6, 0)
    grid = _grid(s, steps, start)
    noise_all = _randn(2, (len(grid), N, 4, 32, 32))
    guid = dict(strength=S) if model == "cfg" else {}
    thr = None if threshold is None else (threshold, float("inf"))
    sde, eta = kw.get("sde", False), kw.get("eta", 0.0)
    a = _run_injected(s, x, classes, steps, noise_all, start=start, threshold=thr, eta=eta, sde=sde, pag_scale=W, **guid)
    b = _chain(s, x, classes, grid, noise_all=noise_all, eta=eta, sde=sde, pag_scale=W, dynamic_threshold=threshold, **guid)
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)


@pytest.mark.parametrize("kind", [k for k in KINDS if k != "ddpm"])
def test_run_equals_chained_steps(golden, kind):
    """sample(rng="torch") runs the host-int route step by step (fused head step); sample_once reads t on the device.  Both
    with PAG and CFG on the class-conditional tiny network: the same bits."""
    cls, kw = KINDS[kind]
    s = cls(_fw(golden, "tiny", frameworks.ClassifierFreeGuidance))
    x = _randn(1, (2, 4, 32, 32))
    classes = torch.tensor([1, 2], device="cuda")
    extra = dict(strength=S, pag_scale=W, pag_layers=("middle_block.1",))
    torch.manual_seed(5)
    run = s.sample(2, noise=x, classes=classes, steps=6, rng="torch", verbose=False, **kw, **extra).samples
    torch.manual_seed(5)
    chained = _chain(s, x, classes, _grid(s, 6, 0), eta=kw.get("eta", 0.0), sde=kw.get("sde", False), **extra)
    assert torch.isfinite(run).all()
    assert torch.equal(run, chained)


def _inpaint_args(golden):
    g = golden
    y = torch.from_numpy(g["ddim_y"]).cuda(); mask = torch.from_numpy(g["ddim_mask"]).cuda()
    mask_rgb = torch.from_numpy(g["ddim_mask_rgb"]).cuda(); convex = torch.from_numpy(g["ddim_convex"]).cuda()
    return dict(y=y, mask=mask, mask_rgb=mask_rgb, replace_rgb=(0.1, y[:, :3], mask_rgb), replace_depth=(0.2, y[:, 3:], mask),
                constrain_depth=(0.5, convex))


COMPOSE = ["inpaint_ddim", "inpaint_dpm_sde", "superres", "fp8", "cache", "inpaint_cache"]


@pytest.mark.parametrize("case", COMPOSE)
def test_run_equals_chained_steps_composed(golden, case):
    """sample(rng="torch") against chained sample_once with PAG, bit for bit, for InpaintCFG with the multiview replace /
    constrain guidance (its hole noise drawn with torch once per step and shared by the perturbed rows), SuperResCFG, fp8
    and feature reuse (reuse forwards of the PAG plan read that plan's cache, on both routes)."""
    N = 2
    x = _randn(1, (N, 4, 32, 32))
    classes = torch.tensor([1, 2], device="cuda")
    args, cache, reuse, sde = {}, {}, None, False
    if case.startswith("inpaint"):
        s = (samplers.DpmSolverSampler if case == "inpaint_dpm_sde" else samplers.DdimSampler)(
            _fw(golden, "tiny_cond", frameworks.InpaintCFG))
        args = _inpaint_args(golden)
        sde = case == "inpaint_dpm_sde"
    elif case == "superres":
        s = samplers.DdimSampler(_fw(golden, "tiny_sr", frameworks.SuperResCFG))
        args = dict(y=_randn(9, (N, 4, 16, 16)))
    else:
        s = samplers.DdimSampler(_fw(golden, "tiny", frameworks.ClassifierFreeGuidance))
    if case.endswith("cache"):
        cache = dict(cache_interval=2)
        reuse = [i % 2 == 1 for i in range(6)]
    if case == "fp8":
        s.framework.backbone.set_precision("fp8")
    extra = dict(strength=S, pag_scale=W, **args)
    torch.manual_seed(5)
    run = s.sample(N, noise=x, classes=classes, steps=6, rng="torch", verbose=False, **({"sde": True} if sde else {}), **cache,
                   **extra).samples
    torch.manual_seed(5)
    chained = _chain(s, x, classes, _grid(s, 6, 0), sde=sde, reuse=reuse, **extra)
    torch.manual_seed(5)
    plain = s.sample(N, noise=x, classes=classes, steps=6, rng="torch", verbose=False, **({"sde": True} if sde else {}), **cache,
                     strength=S, **args).samples
    assert torch.isfinite(run).all()
    assert torch.equal(run, chained)
    assert not torch.equal(run, plain)


def _cond_forward(net, x, cond, N, nf, row0, classes):
    L = _lib.lib()
    S_ = x.shape[-1]
    t = torch.full((nf,), 300, device="cuda")
    out = torch.empty(nf, 4, S_, S_, device="cuda")
    idx = net.pag_layer_indices(["middle_block.1"])
    arr = (ctypes.c_int * 1)(*idx)
    _lib.check(L.ivid_unet_forward_perturbed(net._handle, _lib.ptr(x), N, S_, S_, ctypes.byref(cond), _lib.ptr(t), _lib.ptr(classes),
                                             _lib.ptr(out), nf, row0, arr, 1, -1, _lib.cur_stream()))
    return out


@pytest.mark.parametrize("noise", ["injected", "philox"])
def test_perturbed_rows_share_the_conditional_inputs(golden, noise):
    """InpaintCFG: rows [2N, 3N) of a PAG forward equal an N-row forward in which every row is perturbed, with the same
    conditional inputs and hole noise (injected, or Philox indexed by the conditional row): the perturbed rows see exactly
    the assembly the conditional rows see.  model_inference's PAG eps is the fp32 mix of those rows."""
    fw = _fw(golden, "tiny_cond", frameworks.InpaintCFG)
    net = fw.backbone
    net._ensure_packed()
    a = _inpaint_args(golden)
    N = a["y"].shape[0]
    x = _randn(3, (N, 4, 32, 32))
    z = _randn(4, (N, 4, 32, 32))
    cond = _lib.CondT()
    cond.kind = 1
    cond.y_dev, cond.mask_dev, cond.mask_rgb_dev = a["y"].data_ptr(), a["mask"].data_ptr(), a["mask_rgb"].data_ptr()
    if noise == "injected":
        cond.noise_dev = z.data_ptr()
    else:
        cond.seed, cond.stream_id = 1234, 7
    c = torch.tensor([1, 2], device="cuda")[:N]
    c3 = torch.cat([c, torch.full_like(c, -1), c]).contiguous()
    full = _cond_forward(net, x, cond, N, 3 * N, 2 * N, c3)
    alone = _cond_forward(net, x, cond, N, N, 0, c.contiguous())
    plain = _cond_forward(net, x, cond, N, N, N, c.contiguous())
    assert torch.equal(full[2 * N:], alone)
    assert torch.equal(full[:N], plain)
    if noise == "injected":
        got = fw.model_inference(x, torch.full((N,), 300, device="cuda"), a["y"], a["mask"], classes=c, strength=S,
                                 noise=z, mask_rgb=a["mask_rgb"], pag_scale=W)
        e = full.cpu().numpy()
        assert np.array_equal(got.cpu().numpy(), pag_ref.mix32(e[:N], e[2 * N:], W, 1, S, e[N:2 * N]))


def test_pag_plan_keeps_its_own_feature_cache(golden):
    """A reuse forward of the PAG plan reads the deep features of that plan's last full forward: after a full 3N PAG forward,
    a 2N forward of other inputs and then a reuse forward of the PAG plan with the first inputs, the reuse forward equals the
    full one bit for bit (the same inputs give the same shallow features, and the cached deep ones are its own)."""
    cfg = _cfg(golden, "tiny")
    net = _net(cfg)
    net._ensure_packed()
    L = _lib.lib()
    N = 2
    x, x2 = _randn(1, (N, 4, 32, 32)), _randn(2, (N, 4, 32, 32))
    t3 = torch.full((3 * N,), 400, device="cuda")
    c3 = torch.tensor([1, 2, -1, -1, 1, 2], device="cuda")
    arr = (ctypes.c_int * 1)(*net.pag_layer_indices(["middle_block.1"]))

    def pag(xx, branch):
        out = torch.empty(3 * N, 4, 32, 32, device="cuda")
        _lib.check(L.ivid_unet_forward_perturbed(net._handle, _lib.ptr(xx), N, 32, 32, None, _lib.ptr(t3), _lib.ptr(c3), _lib.ptr(out),
                                                 3 * N, 2 * N, arr, 1, branch, _lib.cur_stream()))
        return out
    full = pag(x, -1)
    other = torch.empty(2 * N, 4, 32, 32, device="cuda")
    t2, c2 = t3[:2 * N].contiguous(), c3[:2 * N].contiguous()
    _lib.check(L.ivid_unet_forward_hw(net._handle, _lib.ptr(x2), N, 32, 32, None, _lib.ptr(t2), _lib.ptr(c2), _lib.ptr(other), 2 * N,
                                      _lib.cur_stream()))
    _lib.check(L.ivid_unet_forward_reuse(net._handle, _lib.ptr(x2), N, 32, 32, None, _lib.ptr(t2), _lib.ptr(c2), _lib.ptr(other), 2 * N,
                                         0, _lib.cur_stream()))
    reused = pag(x, 0)
    assert torch.equal(reused, full)
    assert not torch.equal(pag(x2, 0), pag(x2, -1)), "a reuse forward with other inputs must differ from the full one"


@pytest.mark.parametrize("kind", ["ddim", "dpm_ode", "unipc"])
def test_zero_scale_and_excluded_interval_are_the_plain_run(golden, kind):
    cls, kw = KINDS[kind]
    s = cls(_fw(golden, "tiny", frameworks.ClassifierFreeGuidance))
    x = _randn(1, (2, 4, 32, 32))
    classes = torch.tensor([1, 2], device="cuda")
    run = lambda **k: s.sample(2, noise=x, classes=classes, steps=8, verbose=False, **kw, **k).samples
    torch.manual_seed(2); plain = run(strength=S)
    torch.manual_seed(2); zero = run(strength=S, pag_scale=0.0)
    assert torch.equal(plain, zero)
    torch.manual_seed(2); plain0 = run(strength=0.0)
    torch.manual_seed(2); excl = run(strength=S, pag_scale=W, guidance_interval=(0, 0))   # the grid's model times are 124 .. 999
    torch.manual_seed(2); on = run(strength=S, pag_scale=W)
    assert torch.equal(plain0, excl)
    assert not torch.equal(on, plain)


def _profile_conv_flops(net, fn):
    L = _lib.lib()
    _lib.check(L.ivid_unet_profile_begin(net._handle))
    fn()
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 20)
    _lib.check(L.ivid_unet_profile_end(net._handle, buf, len(buf)))
    prof = json.loads(buf.value.decode())
    return sum(v["flops"] for k, v in prof.items() if k.startswith("conv_gemm")), prof


def test_profiled_flops(golden):
    fw = _fw(golden, "tiny", frameworks.ClassifierFreeGuidance)
    s = samplers.DdimSampler(fw)
    net = fw.backbone
    x = _randn(2, (2, 4, 32, 32)); c = torch.tensor([1, 2], device="cuda")
    step = lambda **k: _once(s, x, 500, 480, c, noise=torch.zeros_like(x), **k)
    step(strength=S); step(strength=S, pag_scale=W); step(strength=S, pag_scale=0.0)
    cfg_f, _ = _profile_conv_flops(net, lambda: step(strength=S))
    pag_f, prof = _profile_conv_flops(net, lambda: step(strength=S, pag_scale=W))
    zero_f, prof0 = _profile_conv_flops(net, lambda: step(strength=S, pag_scale=0.0))
    # the profile prints 7 significant digits
    assert abs(pag_f / cfg_f - 1.5) < 1e-5 and zero_f == cfg_f
    assert "attention_identity" in prof and "attention_identity" not in prof0
    gd = _fw(golden, "tiny", frameworks.GaussianDiffusion)
    sg = samplers.DdimSampler(gd)
    one = lambda **k: _once(sg, x, 500, 480, None, noise=torch.zeros_like(x), **k)
    one(); one(pag_scale=W)
    base_f, _ = _profile_conv_flops(gd.backbone, one)
    pag1_f, _ = _profile_conv_flops(gd.backbone, lambda: one(pag_scale=W))
    assert abs(pag1_f / base_f - 2.0) < 1e-5


def test_pipeline_sample_all(golden):
    fw_u = _fw(golden, "tiny", frameworks.GaussianDiffusion)
    fw_c = _fw(golden, "tiny_cond", frameworks.InpaintCFG)
    mv = build_modelviews("3x9", 1)[:2]
    run = lambda **k: [r[2] for r in sample_all(fw_u, fw_c, [0], 4, 4, mv, batchsize=1, **k)]
    torch.manual_seed(0); plain = run()
    torch.manual_seed(0); default = run(pag_scale=None)
    torch.manual_seed(0); pag = run(pag_scale=W)
    assert all(torch.equal(a, b) for a, b in zip(plain, default))
    assert all(torch.isfinite(p).all() for p in pag) and not torch.equal(pag[0], plain[0])

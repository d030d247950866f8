"""GPU: adaptive projected guidance (`apg=eta`, `(eta, r)` or `(eta, r, beta)`).

ivid_op_apg against the float64 model on crafted data, within the bound of its fp32 operations, and batch invariant; every
step kind on the cfg, inpaint and super-resolution frameworks against the float64 step built from the GPU's own D_c and D_u;
the bitwise properties of the native loop (fused == separate route, ivid_sampler_run == chained sample_once with apg_state,
host == device route, run to run, also with a guidance interval, feature reuse, dynamic thresholding, PAG, SDEdit and fp8);
apg=None is the plain run; no allocation inside a run; one sample_all pipeline run."""
import ctypes
import json

import numpy as np
import pytest
import torch

import apg_ref
import dynamic_threshold_ref as R
import gpu_util as G
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
import unipc_ref
from ivid_b200 import _lib
from ivid_b200.inference.sample import build_modelviews, sample_all
from oracle import sampler_ref, unet_ref

pytestmark = pytest.mark.gpu
T = 1000
S = 3.0
APG = (0.0, 4.0, -0.5)           # the paper's eta and beta, with a norm bound that acts on random weights
STEP_BAR = 1e-5                  # relative L2 of the step against the float64 step from the GPU's D_c, D_u; worst case printed


def _fw(golden, tag, seed, cls):
    cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    return cls(net.cuda(), timesteps=T, beta_schedule="linear")


def _randn(seed, shape, scale=1.0):
    return torch.from_numpy((np.random.default_rng(seed).standard_normal(shape) * scale).astype(np.float32)).cuda()


# ------------------------------------------------------------------------------------------------------------------------
# the op
# ------------------------------------------------------------------------------------------------------------------------
def _op(dc, du, state, s, eta, r, beta):
    """ivid_op_apg over [N, M]: (D, m); state is not modified."""
    dc, du = dc.contiguous().cuda(), du.contiguous().cuda()
    m = state.clone().contiguous().cuda()
    out = torch.empty_like(dc)
    N, M = dc.shape
    _lib.check(_lib.lib().ivid_op_apg(_lib.ptr(dc), _lib.ptr(du), _lib.ptr(m), N, M, float(s), float(eta), float(r), float(beta),
                                      _lib.ptr(out), _lib.cur_stream()))
    return out, m


def _crafted(M, rng):
    """Samples (D_c, D_u) that stress the op: gaussian, D_c = 0, m = 0 (D_c == D_u), one outlier, ties, subnormals."""
    g = lambda: rng.standard_normal(M).astype(np.float32)
    sub = np.float32(1e-40)
    base = g()
    sets = [
        (g() * 2, g() * 2),
        (np.zeros(M, np.float32), g()),
        (base, base.copy()),
        (np.concatenate([g()[:-1], np.float32([1e6])]), g()),
        (np.round(g() * 2).astype(np.float32), np.round(g() * 2).astype(np.float32)),
        ((g() * sub).astype(np.float32), (g() * sub).astype(np.float32)),
    ]
    return np.stack([a for a, _ in sets]), np.stack([b for _, b in sets])


@pytest.mark.parametrize("M", [4 * 128 * 128, 4 * 256 * 256, 4 * 24 * 40])
def test_op_vs_model(M):
    rng = np.random.default_rng(M)
    dc, du = _crafted(M, rng)
    worst = 0.0
    for eta, r, beta in ((1.0, 0.0, 0.0), (0.0, 0.0, 0.0), (0.0, 1.0, -0.5), (0.5, 1e3, 0.9)):
        state = torch.zeros(dc.shape)
        for step in range(3):              # a chain: the momentum state carries from step to step
            d_in, u_in = dc * (1 + 0.1 * step), du
            out, m = _op(torch.from_numpy(d_in), torch.from_numpy(u_in), state, S, eta, r, beta)
            ref, mref = apg_ref.apg64(d_in, u_in, S, eta, r, beta, state.numpy())
            bound = apg_ref.bound32(d_in, u_in, S, eta, r, beta, state.numpy())
            err = np.abs(out.cpu().numpy().astype(np.float64) - ref)
            merr = np.abs(m.cpu().numpy().astype(np.float64) - mref)
            tiny = np.finfo(np.float32).smallest_subnormal
            ratio = float((err / (bound + tiny)).max())
            worst = max(worst, ratio)
            assert np.all(err <= bound + tiny), (eta, r, beta, step, float(err.max()))
            assert np.all(merr <= 4 * apg_ref.EPS32 * (np.abs(d_in) + np.abs(u_in) + abs(beta) * np.abs(state.numpy())) + tiny)
            assert torch.isfinite(out).all()
            state = m.cpu()
    # D_c = 0: D = s c m, the update is the plain one (k = 0); m = 0: D = D_c
    out, _ = _op(torch.from_numpy(dc), torch.from_numpy(du), torch.zeros(dc.shape), S, 0.0, 0.0, 0.0)
    assert torch.equal(out[2].cpu(), torch.from_numpy(dc[2]))
    print(f"[apg op] M={M}: worst error / fp32 bound = {worst:.3e}")


def test_op_batch_invariance():
    rng = np.random.default_rng(7)
    M = 4 * 32 * 48
    dc = torch.from_numpy(rng.standard_normal((32, M)).astype(np.float32))
    du = dc + torch.from_numpy(rng.standard_normal((32, M)).astype(np.float32))
    st = torch.from_numpy(rng.standard_normal((32, M)).astype(np.float32))
    full, mfull = _op(dc, du, st, S, *APG)
    for N in range(1, 33):
        out, m = _op(dc[:N], du[:N], st[:N], S, *APG)
        assert torch.equal(out, full[:N]) and torch.equal(m, mfull[:N]), N
    for n in (0, 5, 31):
        out, m = _op(dc[n:n + 1], du[n:n + 1], st[n:n + 1], S, *APG)
        assert torch.equal(out[0], full[n]) and torch.equal(m[0], mfull[n]), n


# ------------------------------------------------------------------------------------------------------------------------
# steps against the float64 step
# ------------------------------------------------------------------------------------------------------------------------
KINDS = {  # name: (class, sample_once kwargs, order)
    "ddpm": (samplers.DdpmSampler, {}, 1),
    "ddim_eta0": (samplers.DdimSampler, dict(eta=0.0), 1),
    "ddim_eta1": (samplers.DdimSampler, dict(eta=1.0), 1),
    "dpm_ode_o1": (samplers.DpmSolverSampler, {}, 1),
    "dpm_ode_o2": (samplers.DpmSolverSampler, {}, 2),
    "dpm_sde_o1": (samplers.DpmSolverSampler, dict(sde=True), 1),
    "dpm_sde_o2": (samplers.DpmSolverSampler, dict(sde=True), 2),
    "unipc_o1": (samplers.UniPcSampler, {}, 1),
    "unipc_o2": (samplers.UniPcSampler, {}, 2),
    "unipc_o3": (samplers.UniPcSampler, {}, 3),
}


def _setup(golden, fwname):
    """(framework, x_t, classes, model kwargs, replace / constrain guidance kwargs)."""
    if fwname == "cfg":
        fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
        x = _randn(1, (2, 4, 32, 32), 2.0)
        return fw, x, torch.tensor([1, 2]).cuda(), {}, {}
    if fwname == "inpaint":
        fw = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
        x = torch.from_numpy(golden["step_x_t"]).cuda()
        y = torch.from_numpy(golden["ddim_y"]).cuda(); mask = torch.from_numpy(golden["ddim_mask"]).cuda()
        mask_rgb = torch.from_numpy(golden["ddim_mask_rgb"]).cuda(); convex = torch.from_numpy(golden["ddim_convex"]).cuda()
        kw = dict(y=y, mask=mask, mask_rgb=mask_rgb, cond_noise=_randn(3, tuple(x.shape)))
        guide = dict(replace_rgb=(0.1, y[:, :3], mask_rgb), replace_depth=(0.2, y[:, 3:], mask), constrain_depth=(0.5, convex))
        return fw, x, torch.arange(1, x.shape[0] + 1).cuda(), kw, guide
    fw = _fw(golden, "tiny_sr", 1234, frameworks.SuperResCFG)
    x = torch.from_numpy(golden["sr_x"]).cuda()
    return fw, x, torch.arange(1, x.shape[0] + 1).cuda(), dict(y=torch.from_numpy(golden["sr_y"]).cuda()), {}


def _once(s, kind, x, t, tp, classes, z, hist, base, **kw):
    cls, extra, order = KINDS[kind]
    N = x.shape[0]
    tt = torch.full((N,), t, device="cuda")
    if s.KIND == 0:
        return s.sample_once(x, tt, classes, noise=z, **kw)
    tpt = torch.full((N,), tp, device="cuda")
    if s.KIND == 1:
        return s.sample_once(x, tt, tpt, classes, noise=z, **extra, **kw)
    if s.UNIPC:
        return s.sample_once(x, tt, tpt, classes, noise=z, prev=hist[:order - 1] or None, prev_x=base if order > 1 else None,
                             order=order, **kw)
    return s.sample_once(x, tt, tpt, classes, noise=z, prev=hist[0] if order == 2 and hist else None, **extra, **kw)


@pytest.mark.parametrize("fwname", ["cfg", "inpaint", "superres"])
def test_step_vs_float64(golden, fwname, monkeypatch):
    """Each kind with APG against the float64 step from the GPU's own D_c and D_u: the pred_x_0 of the same step at strength 0
    with the classes and with the null class, without replace guidance.  A second step from the first step's apg_state
    checks the momentum."""
    monkeypatch.setattr(R, "_threshold_t", lambda x0, p, s_max: x0)          # the reference's steps without thresholding
    monkeypatch.setattr(R, "threshold", lambda x0, p, s_max=None: (None, np.asarray(x0)))
    fw, x, classes, kw, guide = _setup(golden, fwname)
    acp = sampler_ref.Tables(sampler_ref.get_betas("linear", T)).alphas_cumprod
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", T))
    N = x.shape[0]
    z = _randn(4, tuple(x.shape))
    hist_x = [_randn(5 + j, tuple(x.shape)).clamp(-1, 1) for j in range(2)]
    base = _randn(7, tuple(x.shape), 2.0)
    g64 = {k: tuple(v.double().cpu() if torch.is_tensor(v) else v for v in val) for k, val in guide.items()}
    null = torch.full_like(classes, -1)
    worst = 0.0
    for kind, (cls, extra, order) in KINDS.items():
        s = cls(fw)
        steps = [(999, 0), (10, 0)] if s.KIND == 0 else [(1000, 980), (500, 480), (20, 0)]
        for (t, tp) in steps:
            hist = [(t + 20 * (j + 1), hist_x[j]) for j in range(2) if t + 20 * (j + 1) <= T]
            if s.UNIPC and len(hist) < order - 1:
                continue
            gk = guide if s.KIND != 0 else {}
            d_c = _once(s, kind, x, t, tp, classes, z, hist, base, strength=0.0, **kw).pred_x_0.double().cpu()
            d_u = _once(s, kind, x, t, tp, null, z, hist, base, strength=0.0, **kw).pred_x_0.double().cpu()
            state = None
            for rep in range(2):
                out = _once(s, kind, x, t, tp, classes, z, hist, base, strength=S, apg=APG, apg_state=state, **gk, **kw)
                d, m = apg_ref.apg64(d_c.numpy(), d_u.numpy(), S, *APG, m_prev=None if state is None else state.double().cpu().numpy())
                d = torch.from_numpy(d)
                x64, z64 = x.double().cpu(), z.double().cpu()
                tn, tpn = torch.tensor([t] * N), torch.tensor([tp] * N)
                if s.KIND == 0:
                    ref, ref0 = R.ddpm_step(tb, x64, tn, None, z64, 1.0, x0=d)
                elif s.KIND == 1:
                    ref, ref0 = R.ddim_step(tb, x64, tn, tpn, None, z64, 1.0, eta=extra["eta"], x0=d, **g64)
                else:
                    gn = {k: tuple(v.numpy() if torch.is_tensor(v) else v for v in val) for k, val in g64.items()}
                    d0 = R.dpm_d0(acp, x64.numpy(), t, tp, None, 1.0, x0=d.numpy(), **gn)
                    h64 = [(tl, hx.double().cpu().numpy()) for tl, hx in hist]
                    if s.UNIPC:
                        n = min(order - 1, len(h64))
                        q = 1 if tp == 0 else min(order, n + 1)
                        ref = torch.from_numpy(unipc_ref.step(acp, x64.numpy(), d0, t, tp, q, min(order, n), h64[:n],
                                                              base.double().cpu().numpy())[0])
                    else:
                        o2 = order == 2 and h64 and tp != 0
                        ref = torch.from_numpy(R.dpm_update(acp, x64.numpy(), d0, t, tp, h64[0][1] if o2 else None,
                                                            h64[0][0] if o2 else None, z64.numpy() if extra.get("sde") else None))
                    ref0 = torch.from_numpy(d0)
                name = f"{fwname} {kind} t={t}->{tp} step {rep}"
                worst = max(worst, G.report(name, out.pred_x_prev, ref), G.report(name + " x_0", out.pred_x_0, ref0))
                # m from the GPU's D_c, D_u: their own roundings bound the difference, one unit of the terms of
                # sqrt(1/acp) x_t - sqrt(1/acp - 1) eps each, which cancel to D: |D| + 2 sqrt(1/acp) |x_t|
                mp = np.zeros_like(m) if state is None else state.double().cpu().numpy()
                srac = np.sqrt(1.0 / acp[t if s.KIND == 0 else t - 1])
                mbound = 4 * apg_ref.EPS32 * (apg_ref.m_bound_mag(d_c.numpy(), d_u.numpy(), APG[2], mp)
                                              + 4 * srac * np.abs(x.double().cpu().numpy()))
                assert np.all(np.abs(out.apg_state.double().cpu().numpy() - m) <= mbound), name
                state = out.apg_state
    print(f"[apg] worst relative L2 against the float64 step: {worst:.3e}")
    assert worst <= STEP_BAR


# ------------------------------------------------------------------------------------------------------------------------
# bitwise properties of the native loop
# ------------------------------------------------------------------------------------------------------------------------
def _grid(s, steps, start):
    if s.KIND == 0:
        return [(T - 1 - i, 0) for i in range(start, T)]
    jump = T // steps
    return [(jump * (steps - i), jump * (steps - 1 - i)) for i in range(start, steps)]


def _run_injected(s, x, classes, steps, noise_all, apg, start=0, order=2, eta=0.0, sde=False, interval=None, cache=0,
                  threshold=None, pag_scale=None, **kw):
    """ivid_sampler_run with the step noise injected: the host-int route with the separate step kernels."""
    net = s._net()
    img = x.clone().contiguous()
    pag = (pag_scale, net.pag_layer_indices(["middle_block.1"])) if pag_scale else None
    a, keep = s._step_args(img.device, classes, False, eta, kw, seed=0, hw=img.shape[-2:], order=order, sde=sde,
                           interval=interval, cache=(cache, 0, 0), threshold=samplers.samplers._check_threshold(threshold, False),
                           pag=pag, apg=samplers.samplers._check_apg(apg, s.framework, classes, kw.get("strength", 3.0)))
    a.start_step = start
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().ivid_sampler_run(s._handle, net._handle, _lib.ptr(img), img.shape[0], steps, ctypes.byref(a),
                                               _lib.ptr(noise_all.contiguous()), None, None, None, _lib.cur_stream(img.device)))
    torch.cuda.synchronize()
    del keep
    return img


def _chain(s, x, classes, grid, noise_all, apg, order=2, eta=0.0, sde=False, interval=None, cache=0, threshold=None, **kw):
    """Chained sample_once (device-timestep route, fused head step) with the history and the APG state a run keeps."""
    reuse = s._reuse_schedule([t if s.KIND == 0 else t - 1 for (t, _) in grid], classes, kw, interval, cache,
                              (1,) if kw.get("pag_scale") else None)
    xa, prev, prev_x, state = x.clone(), None, None, None
    N = x.shape[0]
    for i, (t, tp) in enumerate(grid):
        k = dict(kw, noise=noise_all[i], guidance_interval=interval, reuse_features=reuse[i], dynamic_threshold=threshold,
                 apg=apg, apg_state=state)
        tt, tpt = torch.full((N,), t, device="cuda"), torch.full((N,), tp, device="cuda")
        if s.KIND == 0:
            out = s.sample_once(xa, tt, classes, **k)
        elif s.KIND == 1:
            out = s.sample_once(xa, tt, tpt, classes, eta=eta, **k)
        elif s.UNIPC:
            out = s.sample_once(xa, tt, tpt, classes, prev=prev, prev_x=prev_x, order=order, **k)
            prev, prev_x = ([(t, out.pred_x_0)] + (prev or []))[:order], out.corrected_x_t
        else:
            out = s.sample_once(xa, tt, tpt, classes, prev=prev if order == 2 else None, sde=sde, **k)
            prev = (t, out.pred_x_0)
        state = out.apg_state
        xa = out.pred_x_prev
    return xa


LOOP_CASES = {   # name: (class, run options)
    "ddpm": (samplers.DdpmSampler, {}),
    "ddim": (samplers.DdimSampler, dict(eta=1.0)),
    "dpm_ode": (samplers.DpmSolverSampler, {}),
    "dpm_sde": (samplers.DpmSolverSampler, dict(sde=True)),
    "unipc": (samplers.UniPcSampler, dict(order=3)),
    "ddim_interval": (samplers.DdimSampler, dict(eta=1.0, interval=(300, 700))),
    "dpm_cache": (samplers.DpmSolverSampler, dict(cache=2)),
    "unipc_threshold": (samplers.UniPcSampler, dict(order=2, threshold=0.995)),
    "ddim_pag": (samplers.DdimSampler, dict(eta=1.0, pag_scale=1.5)),
    "dpm_sdedit": (samplers.DpmSolverSampler, dict(start=4)),
    "ddim_fp8": (samplers.DdimSampler, dict(eta=1.0, fp8=True)),
}


@pytest.mark.parametrize("case", list(LOOP_CASES))
def test_loop_equalities(golden, case):
    """ivid_sampler_run with injected noise == chained sample_once with apg_state (host-int separate route == device-timestep
    fused route); with Philox noise fused == separate route and run to run."""
    cls, opt = LOOP_CASES[case]
    opt = dict(opt)
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    if opt.pop("fp8", False):
        fw.backbone.set_precision("fp8")
    s = cls(fw)
    steps = T if s.KIND == 0 else 10
    start = opt.pop("start", 0)
    grid = _grid(s, steps, start)
    x = _randn(7, (3, 4, 32, 32), 2.0)
    noise_all = _randn(8, (len(grid), 3, 4, 32, 32))
    classes = torch.tensor([1, 2, 3]).cuda()
    a = _run_injected(s, x, classes, steps, noise_all, APG, start=start, strength=S, **opt)
    b = _chain(s, x, classes, grid, noise_all, APG, strength=S, **opt)
    assert torch.isfinite(a).all()
    assert torch.equal(a, b), "ivid_sampler_run == chained sample_once"
    plain = _run_injected(s, x, classes, steps, noise_all, None, start=start, strength=S, **opt)
    assert not torch.equal(a, plain), "APG changes the samples"
    kw = {}
    if s.KIND == 1:
        kw["eta"] = opt["eta"]
    if s.KIND == 2:
        kw.update(order=opt.get("order", 2), **({"sde": True} if opt.get("sde") else {}))
    init = dict(init=_randn(9, (3, 4, 32, 32)).clamp(-1, 1), init_strength=0.6) if start else dict(noise=x)
    run = lambda traj: s.sample(3, classes=classes, steps=steps, strength=S, verbose=False, return_trajectory=traj, apg=APG,
                                guidance_interval=opt.get("interval"), cache_interval=opt.get("cache") or None,
                                dynamic_threshold=opt.get("threshold"), pag_scale=opt.get("pag_scale"), **init, **kw).samples
    torch.manual_seed(2)
    f1 = run(False)
    torch.manual_seed(2)
    sep = run(True)
    torch.manual_seed(2)
    f2 = run(False)
    assert torch.equal(f1, sep), "fused == separate route"
    assert torch.equal(f1, f2), "run to run"


@pytest.mark.parametrize("fwname", ["cfg", "inpaint"])
def test_host_route_equals_device_route(golden, fwname):
    fw, x, classes, kw, guide = _setup(golden, fwname)
    z = _randn(9, tuple(x.shape))
    state = _randn(10, tuple(x.shape))
    apg = samplers.samplers._check_apg(APG, fw, classes, S)
    bad = []
    for kind, (cls, extra, order) in KINDS.items():
        if order != 1:
            continue
        s = cls(fw)
        t, tp = (500, 0) if s.KIND == 0 else (500, 480)
        gk = guide if s.KIND != 0 else {}
        k = dict(kw, strength=S)
        cond_noise = k.pop("cond_noise", None)
        dev = _once(s, kind, x, t, tp, classes, z, [], None, apg=APG, apg_state=state, cond_noise=cond_noise, **gk, **k)
        host = s._native_step(x, t, tp, classes, False, extra.get("eta", 0.0), dict(k, **gk),
                              z if s.KIND != 2 or extra.get("sde") else None, cond_noise, order=1, sde=bool(extra.get("sde")),
                              apg=apg, apg_state=state)
        for f in ("pred_x_prev", "pred_x_0", "apg_state"):
            if not torch.equal(dev[f], host[f]):
                bad.append((kind, f))
    assert bad == []


def test_unguided_device_step_leaves_the_state(golden):
    """Outside the guidance interval the device-timestep step is the unguided step bit for bit and returns m_prev as given."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    x = _randn(11, (2, 4, 32, 32))
    classes = torch.tensor([1, 2]).cuda()
    state = _randn(12, (2, 4, 32, 32))
    s = samplers.DdimSampler(fw)
    tt, tpt = torch.full((2,), 500, device="cuda"), torch.full((2,), 480, device="cuda")
    z = torch.zeros_like(x)
    out = s.sample_once(x, tt, tpt, classes, noise=z, strength=S, guidance_interval=(0, 100), apg=APG, apg_state=state)
    plain = s.sample_once(x, tt, tpt, classes, noise=z, strength=S, guidance_interval=(0, 100))
    assert torch.equal(out.pred_x_prev, plain.pred_x_prev) and torch.equal(out.apg_state, state)


def test_apg_none_is_the_plain_run(golden):
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    x = _randn(13, (2, 4, 32, 32))
    classes = torch.tensor([1, 2]).cuda()
    for cls in (samplers.DdimSampler, samplers.UniPcSampler):
        s = cls(fw)
        torch.manual_seed(4)
        a = s.sample(2, noise=x, classes=classes, steps=10, strength=S, verbose=False).samples
        torch.manual_seed(4)
        b = s.sample(2, noise=x, classes=classes, steps=10, strength=S, verbose=False, apg=None).samples
        assert torch.equal(a, b), cls


def test_no_allocation_inside_a_run(golden):
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    x = _randn(14, (2, 4, 32, 32))
    classes = torch.tensor([1, 2]).cuda()
    s = samplers.DpmSolverSampler(fw)
    run = lambda: s.sample(2, noise=x, classes=classes, steps=10, strength=S, verbose=False, apg=APG).samples
    run()
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info()[0]
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == before


def test_pipeline_sample_all(golden):
    fw_u = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fw_c = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    mv = build_modelviews("random", 1, rng=np.random.default_rng(0))
    run = lambda **k: [r[2] for r in sample_all(fw_u, fw_c, [0], 4, 4, mv, classes=[3], batchsize=1, **k)]
    torch.manual_seed(0); plain = run()
    torch.manual_seed(0); apg = run(apg=APG)
    assert all(torch.isfinite(p).all() for p in apg) and not torch.equal(apg[0], plain[0])

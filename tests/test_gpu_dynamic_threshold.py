"""GPU: dynamic thresholding of x_0 (`dynamic_threshold=p` or `(p, s_max)`).

The selection and the clamp / scale (ivid_op_dynamic_threshold) against the oracle's fp32 arithmetic bit for bit on crafted
data; every step kind against the float64 step computed from the GPU's own x_t, x_0 and z; the bitwise properties of the
native loop (s_max = 1 is clip_denoised, fused == separate route, loop == chained sample_once, host == device route, run to run,
also with a guidance interval, feature reuse and fp8); the [-1, 1] bound of the final samples; no allocation inside a run."""
import ctypes
import json

import numpy as np
import pytest
import torch

import dynamic_threshold_ref as R
import gpu_util as G
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from oracle import sampler_ref, unet_ref

pytestmark = pytest.mark.gpu
T = 1000
P = 0.995
STEP_BAR = 1e-6          # float64 step from the GPU's own x_t, x_0 and z; measured worst case printed by the test


def _fw(golden, tag, seed, cls):
    cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    return cls(net.cuda(), timesteps=T, beta_schedule="linear")


def _randn(seed, shape, scale=1.0):
    return torch.from_numpy((np.random.default_rng(seed).standard_normal(shape) * scale).astype(np.float32)).cuda()


def _op(x, p, s_max=0.0):
    """ivid_op_dynamic_threshold of x [N, M]: (s [N], x')."""
    x = x.contiguous().cuda()
    N, M = x.shape
    s = torch.empty(N, device="cuda")
    y = torch.empty_like(x)
    _lib.check(_lib.lib().ivid_op_dynamic_threshold(_lib.ptr(x), N, M, float(p), float(s_max), _lib.ptr(s), _lib.ptr(y),
                                                    _lib.cur_stream()))
    return s, y


def _crafted(M, rng):
    """Sets that stress the selection: ties across v_k / v_{k+1}, all equal, all zero, all below 1, one outlier, +-0, subnormals."""
    g = lambda: rng.standard_normal(M).astype(np.float32)
    sets = {
        "gauss": g() * 3,
        "ties": np.round(g() * 4).astype(np.float32),
        "equal": np.full(M, -2.5, np.float32),
        "zeros": np.zeros(M, np.float32),
        "below_one": (g() * 0.2).clip(-0.99, 0.99),
        "outlier": np.concatenate([g()[:-1] * 0.5, np.float32([1e30])]),
        "signed_zero": np.where(rng.random(M) < 0.5, np.float32(-0.0), np.float32(0.0)) + np.where(rng.random(M) < 0.1, g(), 0).astype(np.float32),
        "subnormal": (rng.integers(1, 1 << 23, M).astype(np.uint32).view(np.float32) * np.where(rng.random(M) < 0.5, -1, 1)).astype(np.float32),
        "mixed_exp": (g() * np.float32(2.0) ** rng.integers(-40, 40, M)).astype(np.float32),
    }
    sets["ties_k"] = np.repeat(np.float32([0.5, 1.5, 3.0, 7.0]), M // 4 + 1)[:M] * np.where(rng.random(M) < 0.5, -1, 1).astype(np.float32)
    for v in sets.values():
        rng.shuffle(v)
    return sets


@pytest.mark.parametrize("M", [4 * 128 * 128, 4 * 256 * 256, 4 * 32 * 48])
def test_op_matches_oracle_bitwise(M):
    rng = np.random.default_rng(M)
    sets = _crafted(M, rng)
    bad = []
    for p in (1e-6, 0.5, P, 1.0):
        for s_max in (0.0, 2.0):
            x = np.stack(list(sets.values()))
            s, y = _op(torch.from_numpy(x), p, s_max)
            s_ref, y_ref = R.threshold(x, p, s_max if s_max > 0 else None)
            for i, name in enumerate(sets):
                if s[i].item() != s_ref[i] or not np.array_equal(y[i].cpu().numpy().view(np.uint32), y_ref[i].view(np.uint32)):
                    bad.append((name, p, s_max, s[i].item(), float(s_ref[i])))
    assert bad == []


def test_op_batch_sizes_and_invariance():
    """N from 1 to 32: a sample's s and x' are those of the sample alone."""
    M = 4 * 32 * 48
    rng = np.random.default_rng(5)
    x = torch.from_numpy((rng.standard_normal((32, M)) * rng.uniform(0.5, 5, (32, 1))).astype(np.float32))
    s_all, y_all = _op(x, P)
    s_ref, y_ref = R.threshold(x.numpy(), P)
    assert np.array_equal(s_all.cpu().numpy(), s_ref) and np.array_equal(y_all.cpu().numpy(), y_ref)
    for N in (1, 2, 3, 7, 16, 32):
        s, y = _op(x[:N], P)
        assert torch.equal(s, s_all[:N]) and torch.equal(y, y_all[:N]), N
    for i in (0, 13, 31):
        s, y = _op(x[i:i + 1], P)
        assert torch.equal(s, s_all[i:i + 1]) and torch.equal(y, y_all[i:i + 1]), i


# ------------------------------------------------------------------------------------------------------------------------
# steps
# ------------------------------------------------------------------------------------------------------------------------
KINDS = {  # name: (class, sample_once kwargs, order)
    "ddpm": (samplers.DdpmSampler, {}, 1),
    "ddim_eta0": (samplers.DdimSampler, dict(eta=0.0), 1),
    "ddim_eta1": (samplers.DdimSampler, dict(eta=1.0), 1),
    "dpm_ode_o1": (samplers.DpmSolverSampler, {}, 1),
    "dpm_ode_o2": (samplers.DpmSolverSampler, {}, 2),
    "dpm_sde_o1": (samplers.DpmSolverSampler, dict(sde=True), 1),
    "dpm_sde_o2": (samplers.DpmSolverSampler, dict(sde=True), 2),
}


def _setup(golden, fwname):
    """(framework, x_t, classes, model kwargs, replace / constrain guidance kwargs) of a framework of the step tests."""
    if fwname in ("uncond", "cfg"):
        fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
        x = _randn(1, (2, 4, 32, 32), 2.0)
        return fw, x, (torch.tensor([1, 2]).cuda() if fwname == "cfg" else None), dict(strength=3.0), {}
    if fwname == "inpaint":
        fw = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
        x = torch.from_numpy(golden["step_x_t"]).cuda()
        y = torch.from_numpy(golden["ddim_y"]).cuda(); mask = torch.from_numpy(golden["ddim_mask"]).cuda()
        mask_rgb = torch.from_numpy(golden["ddim_mask_rgb"]).cuda(); convex = torch.from_numpy(golden["ddim_convex"]).cuda()
        kw = dict(strength=3.0, y=y, mask=mask, mask_rgb=mask_rgb, cond_noise=_randn(3, tuple(x.shape)))
        guide = dict(replace_rgb=(0.1, y[:, :3], mask_rgb), replace_depth=(0.2, y[:, 3:], mask), constrain_depth=(0.5, convex))
        return fw, x, torch.arange(1, x.shape[0] + 1).cuda(), kw, guide
    fw = _fw(golden, "tiny_sr", 1234, frameworks.SuperResCFG)
    x = torch.from_numpy(golden["sr_x"]).cuda()
    return fw, x, torch.arange(1, x.shape[0] + 1).cuda(), dict(strength=3.0, y=torch.from_numpy(golden["sr_y"]).cuda()), {}


def _once(s, kind, x, t, tp, classes, z, prev, **kw):
    cls, extra, order = KINDS[kind]
    N = x.shape[0]
    tt = torch.full((N,), t, device="cuda")
    if s.KIND == 0:
        return s.sample_once(x, tt, classes, noise=z, **kw)
    tpt = torch.full((N,), tp, device="cuda")
    if s.KIND == 1:
        return s.sample_once(x, tt, tpt, classes, noise=z, **extra, **kw)
    return s.sample_once(x, tt, tpt, classes, noise=z, prev=prev if order == 2 else None, **extra, **kw)


@pytest.mark.parametrize("fwname", ["uncond", "cfg", "inpaint", "superres"])
def test_step_vs_float64(golden, fwname):
    """Each kind, thresholded at p = 0.995 with and without s_max, against the float64 step from the GPU's own x_t, z and x_0
    (the pred_x_0 of the same step run without thresholding and without replace guidance)."""
    fw, x, classes, kw, guide = _setup(golden, fwname)
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", T))
    acp = tb.alphas_cumprod
    N = x.shape[0]
    z = _randn(4, tuple(x.shape))
    d_prev = _randn(5, tuple(x.shape)).clamp(-1, 1)
    g64 = {k: tuple(v.double().cpu() if torch.is_tensor(v) else v for v in val) for k, val in guide.items()}
    worst = 0.0
    for kind, (cls, extra, order) in KINDS.items():
        s = cls(fw)
        steps = [(999, 0), (10, 0), (0, 0)] if s.KIND == 0 else [(1000, 980), (500, 480), (20, 0)]
        for (t, tp) in steps:
            prev = (t + 20, d_prev) if t + 20 <= T else None
            gk = guide if s.KIND != 0 else {}
            raw = _once(s, kind, x, t, tp, classes, z, prev, **kw)
            for s_max in (None, 2.0):
                dt = P if s_max is None else (P, s_max)
                out = _once(s, kind, x, t, tp, classes, z, prev, dynamic_threshold=dt, **gk, **kw)
                x64, z64, x0 = x.double().cpu(), z.double().cpu(), raw.pred_x_0.double().cpu()
                if s.KIND == 0:
                    ref, ref0 = R.ddpm_step(tb, x64, torch.tensor([t] * N), None, z64, P, s_max, x0=x0)
                elif s.KIND == 1:
                    ref, ref0 = R.ddim_step(tb, x64, torch.tensor([t] * N), torch.tensor([tp] * N), None, z64, P, s_max,
                                            eta=extra["eta"], x0=x0, **g64)
                else:
                    gn = {k: tuple(v.numpy() if torch.is_tensor(v) else v for v in val) for k, val in g64.items()}
                    d0 = R.dpm_d0(acp, x64.numpy(), t, tp, None, P, s_max, x0=x0.numpy(), **gn)
                    o2 = order == 2 and prev is not None and tp != 0
                    ref = torch.from_numpy(R.dpm_update(acp, x64.numpy(), d0, t, tp, d_prev.double().cpu().numpy() if o2 else None,
                                                        t + 20 if o2 else None, z64.numpy() if extra.get("sde") else None))
                    ref0 = torch.from_numpy(d0)
                name = f"{fwname} {kind} t={t}->{tp} s_max={s_max}"
                worst = max(worst, G.report(name, out.pred_x_prev, ref), G.report(name + " x_0", out.pred_x_0, ref0))
                assert gk or out.pred_x_0.abs().max() <= 1.0, name
    print(f"[threshold] worst relative L2 against the float64 step: {worst:.3e}")
    assert worst <= STEP_BAR


def test_smax_one_equals_clip_every_kind_both_routes(golden):
    """s_max = 1 gives s = 1: clip_denoised=True bit for bit, on the fused route (no trajectory) and the separate one."""
    fu = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    x = _randn(6, (2, 4, 32, 32), 2.0)
    classes = torch.tensor([3, 4]).cuda()
    for kind, (cls, extra, order) in KINDS.items():
        s = cls(fu)
        kw = dict(extra, order=order) if s.KIND == 2 else dict(extra)
        steps = None if s.KIND == 0 else 10
        for traj in (False, True):
            run = lambda **o: s.sample(2, noise=x, classes=classes, steps=steps, strength=3.0, verbose=False,
                                       return_trajectory=traj, **kw, **o).samples
            torch.manual_seed(1)
            a = run(clip_denoised=True)
            torch.manual_seed(1)
            b = run(dynamic_threshold=(0.5, 1.0))
            assert torch.isfinite(a).all()
            assert torch.equal(a, b), (kind, traj)


def _run_injected(s, x, classes, steps, noise_all, threshold, interval=None, cache=None, order=2, sde=False, eta=0.0, **kw):
    """ivid_sampler_run with the per-step draws injected (separate route)."""
    net = s._net()
    img = x.clone().contiguous()
    a, keep = s._step_args(img.device, classes, False, eta, kw, seed=0, hw=img.shape[-2:], order=order, sde=sde,
                           interval=interval, cache=cache, threshold=samplers.samplers._check_threshold(threshold, False))
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().ivid_sampler_run(s._handle, net._handle, _lib.ptr(img), img.shape[0], steps, ctypes.byref(a),
                                               _lib.ptr(noise_all.contiguous()), None, None, None, _lib.cur_stream(img.device)))
    torch.cuda.synchronize()
    del keep
    return img


LOOP_CASES = {   # name: (kind, extra run options)
    "ddpm": ("ddpm", {}),
    "ddim": ("ddim_eta1", {}),
    "dpm_ode": ("dpm_ode_o2", {}),
    "dpm_sde": ("dpm_sde_o2", {}),
    "ddim_interval": ("ddim_eta1", dict(interval=(300, 700))),
    "dpm_cache": ("dpm_ode_o2", dict(cache=2)),
    "ddim_fp8": ("ddim_eta1", dict(fp8=True)),
}


@pytest.mark.parametrize("case", list(LOOP_CASES))
def test_loop_equalities(golden, case):
    """ivid_sampler_run with injected noise == chained sample_once; fused == separate route with Philox noise; run to run."""
    kind, opt = LOOP_CASES[case]
    cls, extra, order = KINDS[kind]
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    if opt.get("fp8"):
        fw.backbone.set_precision("fp8")
    s = cls(fw)
    steps = T if s.KIND == 0 else 10
    x = _randn(7, (3, 4, 32, 32), 2.0)
    noise_all = _randn(8, (steps, 3, 4, 32, 32))
    classes = torch.tensor([1, 2, 3]).cuda()
    interval = opt.get("interval")
    cache_interval = opt.get("cache")
    strength = 3.0
    dt = (P, 4.0)
    # the loop on the host-int route with injected noise
    a = _run_injected(s, x, classes, steps, noise_all, dt, interval=interval,
                      cache=(cache_interval, 0, 0) if cache_interval else None, order=order, sde=bool(extra.get("sde")),
                      eta=extra.get("eta", 0.0), strength=strength)
    # chained sample_once on the device route
    xa, prev = x.clone(), None
    sched = [(t, 0) for t in reversed(range(T))] if s.KIND == 0 else sampler_ref.ddim_schedule(T, steps)
    reuse = s._reuse_schedule([t if s.KIND == 0 else t - 1 for (t, _) in sched], classes, dict(strength=strength), interval,
                              cache_interval or 0)
    for i, (t, tp) in enumerate(sched):
        out = _once(s, kind, xa, t, tp, classes, noise_all[i], prev, strength=strength, dynamic_threshold=dt,
                    guidance_interval=interval, reuse_features=reuse[i])
        prev, xa = (t, out.pred_x_0), out.pred_x_prev
    assert torch.isfinite(a).all()
    assert torch.equal(a, xa), "ivid_sampler_run == chained sample_once"
    # Philox noise: fused (no trajectory) == separate (trajectory), and run to run
    kw = dict(extra, order=order) if s.KIND == 2 else dict(extra)
    run = lambda traj: s.sample(3, noise=x, classes=classes, steps=steps, strength=strength, verbose=False, return_trajectory=traj,
                                dynamic_threshold=dt, guidance_interval=interval, cache_interval=cache_interval, **kw).samples
    torch.manual_seed(2)
    f1 = run(False)
    torch.manual_seed(2)
    sep = run(True)
    torch.manual_seed(2)
    f2 = run(False)
    assert torch.equal(f1, sep), "fused == separate route"
    assert torch.equal(f1, f2), "run to run"


def test_host_route_equals_device_route(golden):
    fw, x, classes, kw, guide = _setup(golden, "inpaint")
    z = _randn(9, tuple(x.shape))
    bad = []
    for kind, (cls, extra, order) in KINDS.items():
        s = cls(fw)
        t, tp = (500, 0) if s.KIND == 0 else (500, 480)
        gk = guide if s.KIND != 0 else {}
        k = dict(kw); cond_noise = k.pop("cond_noise")
        dev = _once(s, kind, x, t, tp, classes, z, None, dynamic_threshold=P, cond_noise=cond_noise, **gk, **k)
        host = s._native_step(x, t, tp, classes, False, extra.get("eta", 0.0), dict(k, **gk), z if s.KIND != 2 or extra.get("sde") else None,
                              cond_noise, order=1, sde=bool(extra.get("sde")), threshold=(P, float("inf")))
        for f in ("pred_x_prev", "pred_x_0"):
            if not torch.equal(dev[f], host[f]):
                bad.append((kind, f))
    assert bad == []


def test_final_samples_bounded(golden):
    """Random weights at strength 3 drive x_0 far outside [-1, 1]: thresholded, every final DDPM / DDIM / DPM-Solver++ sample
    lies in [-1, 1]; unthresholded, it does not."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    x = _randn(10, (2, 4, 32, 32))
    classes = torch.tensor([5, 6]).cuda()
    for cls, kw in ((samplers.DdpmSampler, {}), (samplers.DdimSampler, dict(eta=0.0)), (samplers.DpmSolverSampler, {}),
                    (samplers.DpmSolverSampler, dict(sde=True))):
        s = cls(fw)
        run = lambda **o: s.sample(2, noise=x, classes=classes, steps=20, strength=3.0, verbose=False, **kw, **o).samples
        torch.manual_seed(3)
        a = run(dynamic_threshold=P)
        torch.manual_seed(3)
        b = run()
        print(f"[bound] {cls.__name__} {kw}: max |x| thresholded {a.abs().max().item():.4f}, plain {b.abs().max().item():.4f}")
        assert a.abs().max() <= 1.0
        assert b.abs().max() > 1.0


def test_no_allocation_inside_a_run(golden):
    """After a warm-up run the same thresholded run changes the device's free memory by nothing."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    x = _randn(11, (2, 4, 32, 32))
    classes = torch.tensor([1, 2]).cuda()
    s = samplers.DpmSolverSampler(fw)
    run = lambda: s.sample(2, noise=x, classes=classes, steps=10, strength=3.0, verbose=False, dynamic_threshold=P).samples
    run()
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info()[0]
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == before

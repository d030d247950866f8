"""GPU: classifier-free guidance restricted to an interval of model times (`guidance_interval=(t_lo, t_hi)`).

A step whose model time lies outside the interval is the same step at strength 0.  So the oracle of a whole run is the
sampler with a per-step strength of s inside the interval and 0 outside, and every check below is bitwise except the one
against the float64-free reference step, which uses the existing sampler parity bars.  The host-int route runs an unguided
step as a batch-N forward; the device-timestep route (sample_once) keeps the batch-2N forward and drops the null-class half
in the step kernel; the forward is batch-invariant, so both give the same bits."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import gpu_util as G
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from ivid_b200.inference import build_modelviews, sample_all
from oracle import sampler_ref, unet_ref

pytestmark = pytest.mark.gpu
STEP_TOL = 1e-3
T = 1000
S = 0.5
HERE = os.path.dirname(os.path.abspath(__file__))


def _cfg(golden, tag):
    return json.loads(bytes(golden[f"{tag}_cfg"]).decode())


def _fw(golden, tag, seed, cls):
    cfg = _cfg(golden, tag)
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    return cls(net.cuda(), timesteps=T, beta_schedule="linear")


def _randn(seed, shape):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal(shape).astype(np.float32)).cuda()


def _guidance(golden):
    y = torch.from_numpy(golden["ddim_y"]).cuda(); mask = torch.from_numpy(golden["ddim_mask"]).cuda()
    mask_rgb = torch.from_numpy(golden["ddim_mask_rgb"]).cuda(); convex = torch.from_numpy(golden["ddim_convex"]).cuda()
    return dict(y=y, mask=mask, mask_rgb=mask_rgb, replace_rgb=(0.1, y[:, :3], mask_rgb), replace_depth=(0.2, y[:, 3:], mask),
                constrain_depth=(0.5, convex))


# sampler kinds: (name, class, sample() kwargs)
KINDS = {
    "ddpm": (samplers.DdpmSampler, {}),
    "ddim": (samplers.DdimSampler, dict(eta=1.0)),
    "dpm_ode": (samplers.DpmSolverSampler, {}),
    "dpm_sde": (samplers.DpmSolverSampler, dict(sde=True)),
}


def _schedule(s, steps):
    """(t, t_prev, model time) of every step of a run, as ivid_sampler_run walks them."""
    if s.KIND == 0:
        return [(t, 0, t) for t in reversed(range(T))]
    return [(t, tp, t - 1) for (t, tp) in sampler_ref.ddim_schedule(T, steps)]


def _run_injected(s, x, classes, steps, noise_all, interval=None, cond_noise_all=None, eta=0.0, sde=False, **kw):
    """ivid_sampler_run (host-int route, separate step kernel) with the per-step draws injected."""
    net = s._net()
    img = x.clone().contiguous()
    a, keep = s._step_args(img.device, classes, False, eta, kw, seed=0, hw=img.shape[-2:], order=2, sde=sde, interval=interval)
    ca = cond_noise_all.contiguous() if cond_noise_all is not None else None
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().ivid_sampler_run(s._handle, net._handle, _lib.ptr(img), img.shape[0], steps, ctypes.byref(a),
                                               _lib.ptr(noise_all.contiguous()), _lib.ptr(ca), None, None,
                                               _lib.cur_stream(img.device)))
    torch.cuda.synchronize()
    del keep
    return img


def _chained(s, x, classes, steps, noise_all, interval, cond_noise_all=None, eta=0.0, sde=False, **kw):
    """The per-step-strength oracle on the native steps: chained sample_once with strength s inside the interval, 0 outside."""
    xa, prev = x.clone(), None
    N = x.shape[0]
    lo, hi = interval
    for i, (t, tp, tm) in enumerate(_schedule(s, steps)):
        k = dict(kw, strength=S if lo <= tm <= hi else 0.0, noise=noise_all[i])
        if cond_noise_all is not None:
            k["cond_noise"] = cond_noise_all[i]
        tt = torch.full((N,), t, device="cuda")
        if s.KIND == 0:
            out = s.sample_once(xa, tt, classes, **k)
        elif s.KIND == 1:
            out = s.sample_once(xa, tt, torch.full((N,), tp, device="cuda"), classes, eta=eta, **k)
        else:
            out = s.sample_once(xa, tt, torch.full((N,), tp, device="cuda"), classes, prev=prev, sde=sde, **k)
            prev = (t, out.pred_x_0)
        xa = out.pred_x_prev
    return xa


@pytest.mark.parametrize("kind", list(KINDS))
def test_full_interval_equals_no_interval(golden, kind):
    """An interval covering every model time guides every step: the same bits as no interval (Philox noise, fused route)."""
    cls, kw = KINDS[kind]
    s = cls(_fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance))
    x = _randn(1, (2, 4, 32, 32))
    classes = torch.tensor([1, 2]).cuda()
    run = lambda **gi: s.sample(2, noise=x, classes=classes, steps=10, strength=S, verbose=False, **kw, **gi).samples
    torch.manual_seed(3)
    a = run()
    torch.manual_seed(3)
    b = run(guidance_interval=(0, T - 1))
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)


@pytest.mark.parametrize("kind", ["ddim", "dpm_ode", "dpm_sde"])
def test_empty_interval_equals_strength_zero(golden, kind):
    """The 10-step grid's model times are 99, 199, ..., 999: (0, 50) excludes all of them, so the run is the strength-0 run."""
    cls, kw = KINDS[kind]
    s = cls(_fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance))
    x = _randn(2, (2, 4, 32, 32))
    classes = torch.tensor([3, 4]).cuda()
    torch.manual_seed(4)
    a = s.sample(2, noise=x, classes=classes, steps=10, strength=S, verbose=False, guidance_interval=(0, 50), **kw).samples
    torch.manual_seed(4)
    b = s.sample(2, noise=x, classes=classes, steps=10, strength=0.0, verbose=False, **kw).samples
    torch.manual_seed(4)
    c = s.sample(2, noise=x, classes=classes, steps=10, strength=S, verbose=False, **kw).samples
    assert torch.equal(a, b)
    assert not torch.equal(a, c), "guidance changes the samples"


@pytest.mark.parametrize("kind", list(KINDS))
def test_mixed_interval_run_equals_per_step_strength(golden, kind):
    """ivid_sampler_run with injected noise == chained sample_once with the host switching strength between s and 0."""
    cls, kw = KINDS[kind]
    s = cls(_fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance))
    steps = T if kind == "ddpm" else 10
    interval = (300, 700)
    x = _randn(5, (2, 4, 32, 32))
    noise_all = _randn(6, (steps, 2, 4, 32, 32))
    classes = torch.tensor([5, 6]).cuda()
    a = _run_injected(s, x, classes, steps, noise_all, interval, strength=S, **kw)
    b = _chained(s, x, classes, steps, noise_all, interval, **kw)
    c = _run_injected(s, x, classes, steps, noise_all, None, strength=S, **kw)
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)
    assert not torch.equal(a, c), "the interval leaves some steps unguided"


@pytest.mark.parametrize("kind", ["ddim", "dpm_ode"])
@pytest.mark.parametrize("tag", ["tiny_cond", "tiny_sr"])
def test_mixed_interval_conditional_frameworks(golden, tag, kind):
    """The same on InpaintCFG (hole noise injected, multiview replace / constrain guidance) and SuperResCFG."""
    cls, kw = KINDS[kind]
    if tag == "tiny_cond":
        fw = _fw(golden, tag, 4321, frameworks.InpaintCFG)
        x = torch.from_numpy(golden["step_x_t"]).cuda()
        extra = _guidance(golden)
        cond_noise_all = _randn(7, (6,) + tuple(x.shape))
    else:
        fw = _fw(golden, tag, 1234, frameworks.SuperResCFG)
        x = torch.from_numpy(golden["sr_x"]).cuda()
        extra = dict(y=torch.from_numpy(golden["sr_y"]).cuda())
        cond_noise_all = None
    s = cls(fw)
    N = x.shape[0]
    classes = torch.arange(1, N + 1).cuda()
    noise_all = _randn(8, (6,) + tuple(x.shape))
    interval = (300, 700)             # the 6-step grid: model times 165, 331, 497, 663, 829, 995
    a = _run_injected(s, x, classes, 6, noise_all, interval, cond_noise_all=cond_noise_all, strength=S, **kw, **extra)
    b = _chained(s, x, classes, 6, noise_all, interval, cond_noise_all=cond_noise_all, **kw, **extra)
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)


def _device_vs_host(golden):
    """sample_once (device timestep, batch-2N forward, in-kernel gating) == _native_step (host int, batch-N forward when
    unguided), for one step inside and one outside the interval, DDPM / DDIM / DPM-Solver++; returns the failures."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    x = _randn(9, (2, 4, 32, 32)); z = _randn(10, (2, 4, 32, 32))
    classes = torch.tensor([7, 8]).cuda()
    interval = (300, 700)
    bad = []
    for kind in ("ddpm", "ddim", "dpm_sde"):
        cls, kw = KINDS[kind]
        s = cls(fw)
        for (t, tp) in ((501, 401), (901, 801)):                      # model times 500 / 501 inside, 900 / 901 outside
            tt = torch.full((2,), t, device="cuda"); tpt = torch.full((2,), tp, device="cuda")
            if s.KIND == 0:
                dev = s.sample_once(x, tt, classes, noise=z, strength=S, guidance_interval=interval)
                host = s._native_step(x, t, 0, classes, False, 0.0, dict(strength=S), z, None, interval=interval)
                plain = s.sample_once(x, tt, classes, noise=z, strength=S if 300 <= t <= 700 else 0.0)
            else:
                sde = kw.get("sde", False)
                once = lambda st, gi: s.sample_once(x, tt, tpt, classes, noise=z, strength=st, guidance_interval=gi,
                                                    **({"sde": sde} if s.KIND == 2 else {"eta": kw["eta"]}))
                dev = once(S, interval)
                host = s._native_step(x, t, tp, classes, False, kw.get("eta", 0.0), dict(strength=S), z, None, order=1,
                                      sde=sde, interval=interval)
                plain = once(S if 300 <= t - 1 <= 700 else 0.0, None)
            for name, other in (("host route", host), ("per-step strength", plain)):
                for f in ("pred_x_prev", "pred_x_0"):
                    if not torch.equal(dev[f], other[f]):
                        bad.append(f"{kind} t={t}: device route != {name} ({f})")
    return bad


def test_device_route_equals_host_route(golden):
    """Fused route: the step is the output head's last kernel."""
    assert _device_vs_host(golden) == []


def test_device_route_equals_host_route_separate_kernel():
    """The separate eps_gather_kernel + step_kernel<EpsRows, ...> pair (IVID_NO_FUSED_STEP=1 is read once per process: a fresh one)."""
    code = ("import sys, json, os; sys.path[:0] = [sys.argv[1], sys.argv[2]]\n"
            "import numpy as np, test_gpu_guidance_interval as m\n"
            "golden = {k: v for i in (0, 1) for k, v in\n"
            "          np.load(os.path.join(sys.argv[2], 'golden', f'unet_sampler_golden_part{i}.npz')).items()}\n"
            "print(json.dumps(m._device_vs_host(golden)))\n")
    env = dict(os.environ, IVID_NO_FUSED_STEP="1")
    r = subprocess.run([sys.executable, "-s", "-c", code, os.path.dirname(HERE), HERE], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    assert json.loads(r.stdout.strip().splitlines()[-1]) == []


def test_unguided_step_vs_oracle(golden):
    """A step outside the interval against the reference's step on eps from ONE conditional forward (model_inference at
    strength 0), at the bars of tests/test_gpu_sampler.py."""
    cfg = _cfg(golden, "tiny")
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", T))
    model = lambda xx, tt, c: unet_ref.unet_forward(cfg, sd, xx, tt, c)
    x_t = torch.from_numpy(golden["step_x_t"]); classes = torch.from_numpy(golden["step_classes"])
    N = x_t.shape[0]
    z = torch.from_numpy(golden["ddpm_t999_noise"])
    ddpm = samplers.DdpmSampler(fw)
    for ti in (999, 1):
        t = torch.tensor([ti] * N)
        ref, _ = sampler_ref.ddpm_step(tb, x_t, t, sampler_ref.cfg_eps(model, x_t, t, classes, 0.0), z)
        out = ddpm.sample_once(x_t.cuda(), t.cuda(), classes.cuda(), strength=S, noise=z.cuda(), guidance_interval=(300, 700))
        r = G.report(f"unguided ddpm step t={ti}", out.pred_x_prev, ref)
        assert r < STEP_TOL and r < 4e-5
    ddim = samplers.DdimSampler(fw)
    for (tt, tp) in ((1000, 900), (200, 100)):
        t = torch.tensor([tt] * N); tpv = torch.tensor([tp] * N)
        ref, _ = sampler_ref.ddim_step(tb, x_t, t, tpv, sampler_ref.cfg_eps(model, x_t, t - 1, classes, 0.0), torch.zeros_like(x_t))
        out = ddim.sample_once(x_t.cuda(), t.cuda(), tpv.cuda(), classes.cuda(), strength=S, noise=torch.zeros_like(x_t).cuda(),
                               guidance_interval=(300, 700))
        r = G.report(f"unguided ddim step {tt}->{tp}", out.pred_x_prev, ref)
        assert r < STEP_TOL and r < 7.8e-4


def _conv_flops(s, x, t, classes, interval):
    net = s._net()
    step = lambda: s._native_step(x, t, 0, classes, False, 0.0, dict(strength=S), torch.zeros_like(x), None, interval=interval)
    step()
    torch.cuda.synchronize()
    L = _lib.lib()
    _lib.check(L.ivid_unet_profile_begin(net._handle))
    step()
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(L.ivid_unet_profile_end(net._handle, buf, len(buf)))
    fam = json.loads(buf.value.decode())
    return sum(v["flops"] for k, v in fam.items() if k.startswith("conv"))


def test_unguided_step_runs_batch_n_forward(golden):
    """The profiled conv FLOPs (algorithmic, proportional to the forward's batch) of an unguided step are half a guided one's."""
    s = samplers.DdpmSampler(_fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance))
    x = _randn(11, (2, 4, 32, 32)); classes = torch.tensor([1, 2]).cuda()
    guided = _conv_flops(s, x, 500, classes, (300, 700))
    unguided = _conv_flops(s, x, 900, classes, (300, 700))
    print(f"[flops] conv guided {guided:.4e} unguided {unguided:.4e}")
    assert guided > 0 and unguided * 2 == pytest.approx(guided, rel=1e-6)     # the profile JSON prints 7 significant digits


def test_fp8_mixed_interval(golden):
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fw.backbone.set_precision("fp8")
    s = samplers.DdimSampler(fw)
    x = _randn(12, (2, 4, 32, 32)); noise_all = _randn(13, (10, 2, 4, 32, 32)); classes = torch.tensor([1, 2]).cuda()
    a = _run_injected(s, x, classes, 10, noise_all, (300, 700), eta=1.0, strength=S)
    b = _chained(s, x, classes, 10, noise_all, (300, 700), eta=1.0)
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)


def test_torch_rng_stream_unchanged(golden):
    """rng='torch' with an interval draws exactly what it draws without one, and runs the per-step-strength steps."""
    s = samplers.DdimSampler(_fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance))
    x = _randn(14, (2, 4, 32, 32)); classes = torch.tensor([1, 2]).cuda()
    torch.manual_seed(21)
    a = s.sample(2, noise=x, classes=classes, steps=10, strength=S, eta=1.0, verbose=False, rng="torch", guidance_interval=(300, 700))
    after = torch.randn(4, device="cuda")
    torch.manual_seed(21)
    noise_all = torch.stack([torch.randn_like(x) for _ in range(10)])
    assert torch.equal(after, torch.randn(4, device="cuda")), "the torch RNG is consumed as without an interval"
    assert torch.equal(a.samples, _run_injected(s, x, classes, 10, noise_all, (300, 700), eta=1.0, strength=S))


def test_sample_all_full_interval_equals_default(golden):
    fu = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    mvs = build_modelviews("random", 3, rng=np.random.default_rng(1))
    kw = dict(fov=45, near=0.6, far=5, atol=0.03, rtol=0.03, erode_rgb=3, classes=[1, 2, 3], guidance=S, batchsize=2)
    a = list(sample_all(fu, fc, [5, 6, 7], 10, 4, mvs, **kw))
    b = list(sample_all(fu, fc, [5, 6, 7], 10, 4, mvs, guidance_interval=(0, T - 1), **kw))
    c = list(sample_all(fu, fc, [5, 6, 7], 10, 4, mvs, guidance_interval=(300, 700), **kw))
    assert len(a) == len(b) == 3
    for (_, _, sa, _), (_, _, sb, _) in zip(a, b):
        assert torch.equal(sa, sb)
    assert not all(torch.equal(sa, sc) for (_, _, sa, _), (_, _, sc, _) in zip(a, c))

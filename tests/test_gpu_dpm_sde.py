"""GPU: the stochastic DPM-Solver++(2M) update (DpmSolverSampler with sde=True).  Order 1 against the reference's DDIM step at
eta = 1 from the same x_t, eps and z; every 2M step of a guided run against the float64 update from the GPU's own x_t, D0,
D_{-1} and z; the bitwise properties of the native loop (fused == separate route with Philox noise, loop with injected noise
== chained sample_once, run to run, batch independence); the pipeline with solver='dpmpp_sde'; and the torch RNG stream."""
import ctypes
import json

import numpy as np
import pytest
import torch

import dpm_sde_ref as R
import gpu_util as G
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from ivid_b200.inference import build_modelviews, sample_all
from oracle import dpm_ref, sampler_ref, unet_ref

pytestmark = pytest.mark.gpu
STEP_TOL = 1e-3


def _fw(golden, tag, seed, cls):
    cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    return cls(net.cuda(), timesteps=1000, beta_schedule="linear")


def _guidance(golden):
    y = torch.from_numpy(golden["ddim_y"]).cuda(); mask = torch.from_numpy(golden["ddim_mask"]).cuda()
    mask_rgb = torch.from_numpy(golden["ddim_mask_rgb"]).cuda(); convex = torch.from_numpy(golden["ddim_convex"]).cuda()
    return dict(replace_rgb=(0.1, y[:, :3], mask_rgb), replace_depth=(0.2, y[:, 3:], mask), constrain_depth=(0.5, convex))


def _cond_kwargs(golden):
    y = torch.from_numpy(golden["ddim_y"]).cuda(); mask = torch.from_numpy(golden["ddim_mask"]).cuda()
    mask_rgb = torch.from_numpy(golden["ddim_mask_rgb"]).cuda()
    return dict(y=y, mask=mask, mask_rgb=mask_rgb, **_guidance(golden))


def _randn(seed, shape):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal(shape).astype(np.float32)).cuda()


def _run_injected(s, x, classes, steps, noise_all, **kw):
    """ivid_sampler_run with the per-step draws injected ([steps][N,C,H,W]); returns the samples."""
    net = s._net()
    img = x.clone().contiguous()
    noise_all = noise_all.contiguous()
    a, keep = s._step_args(img.device, classes, False, 0.0, kw, seed=0, hw=img.shape[-2:], order=2, sde=True)
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().ivid_sampler_run(s._handle, net._handle, _lib.ptr(img), img.shape[0], steps, ctypes.byref(a),
                                               _lib.ptr(noise_all), None, None, None, _lib.cur_stream(img.device)))
    torch.cuda.synchronize()
    del keep
    return img


def test_order1_steps_vs_ddim_eta1(golden):
    """First order is DDIM with eta = 1: each step against the reference's DDIM step (sampler_ref.ddim_step, fp32 tables as
    the reference reads them) at eta = 1, from the same x_t, the same guidance-mixed eps and the same injected z, with and
    without the replace / constrain guidance, at the bar of the ODE solver's order-1 check against DDIM at eta = 0."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = samplers.DpmSolverSampler(fw)
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", 1000))
    x_t = _randn(7, (2, 4, 32, 32)); z = _randn(8, (2, 4, 32, 32))
    classes = torch.tensor([1, 2]).cuda()
    N = x_t.shape[0]
    for (tt, tp) in [(1000, 980), (500, 480), (41, 21), (20, 0)]:
        eps = fw.model_inference(x_t, torch.tensor([tt - 1] * N, device="cuda"), classes, strength=0.5)
        for guided in (False, True):
            g = _guidance(golden) if guided else {}
            out = s.sample_once(x_t, torch.tensor([tt] * N, device="cuda"), torch.tensor([tp] * N, device="cuda"), classes,
                                prev=None, strength=0.5, noise=z, sde=True, **g)
            g_cpu = {k: tuple(v.cpu() if torch.is_tensor(v) else v for v in val) for k, val in g.items()}
            ref, x0 = sampler_ref.ddim_step(tb, x_t.cpu(), torch.tensor([tt] * N), torch.tensor([tp] * N), eps.cpu(), z.cpu(),
                                            eta=1.0, **g_cpu)
            r = G.report(f"dpm++ sde order-1 step {tt}->{tp} guided={guided} vs ddim eta=1", out.pred_x_prev, ref)
            assert r < STEP_TOL
            assert G.report(f"  x_0 of that step", out.pred_x_0, x0) < STEP_TOL
            if tp == 0:
                assert torch.equal(out.pred_x_prev, out.pred_x_0), "the final step returns x_0 and draws no noise"


def test_2m_step_arithmetic_teacher_forced(golden):
    """10-step guided 2M SDE run with rng='torch': every step's x_{t_prev} recomputed in float64 from the GPU's own x_t, D0,
    D_{-1} and the replayed torch draw z.  Free of the UNet's error, this isolates the update."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = samplers.DpmSolverSampler(fw)
    acp = s.alphas_cumprod
    x = _randn(0, (2, 4, 32, 32))
    classes = torch.tensor([1, 2]).cuda()
    torch.manual_seed(11)
    res = s.sample(2, noise=x, classes=classes, steps=10, strength=0.5, verbose=False, rng="torch", return_trajectory=True,
                   sde=True, **_guidance(golden))
    torch.manual_seed(11)
    zs = [torch.randn_like(x) for _ in range(10)]
    xt = [x] + res.pred_x_t[:-1]
    d0 = [d.double().cpu().numpy() for d in res.pred_x_0]
    worst = 0.0
    for i, (t, tp, t_last, o) in enumerate(dpm_ref.schedule(1000, 10, 2)):
        ref = R.sde_update(acp, xt[i].double().cpu().numpy(), d0[i], zs[i].double().cpu().numpy(), t, tp,
                           d0[i - 1] if o == 2 else None, t_last if o == 2 else None)
        worst = max(worst, G.report(f"dpm++ sde(2M) step {t}->{tp} (order {o}) vs float64 update", res.pred_x_t[i],
                                    torch.from_numpy(ref)))
    assert worst <= 1e-5
    assert torch.equal(res.pred_x_t[-1], res.pred_x_0[-1]) and torch.equal(res.samples, res.pred_x_t[-1])


def test_fused_equals_separate_route(golden):
    """Philox noise: without trajectories the update runs inside the output head's kernel, with them in the separate step
    kernel.  Both draw the same numbers and round the same way: same bits, on both models."""
    fu = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    x = _randn(2, (2, 4, 32, 32))
    classes = torch.tensor([1, 2]).cuda()
    for fw, kw in ((fu, {}), (fc, _cond_kwargs(golden))):
        s = samplers.DpmSolverSampler(fw)
        torch.manual_seed(5)
        a = s.sample(2, noise=x, classes=classes, steps=8, strength=0.5, verbose=False, sde=True, **kw).samples
        torch.manual_seed(5)
        b = s.sample(2, noise=x, classes=classes, steps=8, strength=0.5, verbose=False, return_trajectory=True, sde=True, **kw)
        G.report(f"{type(fw).__name__}: dpm++ sde fused vs separate", a, b.samples)
        assert torch.isfinite(a).all()
        assert torch.equal(a, b.samples)
        torch.manual_seed(5)
        ode = s.sample(2, noise=x, classes=classes, steps=8, strength=0.5, verbose=False, **kw).samples
        assert not torch.equal(ode, a), "the SDE update draws noise"


def test_loop_equals_chained_sample_once_and_is_deterministic(golden):
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = samplers.DpmSolverSampler(fw)
    x = _randn(3, (3, 4, 32, 32))
    noise_all = _randn(4, (10, 3, 4, 32, 32))
    classes = torch.tensor([1, 2, 3]).cuda()
    xa, prev = x.clone(), None
    for i, (tt, tp) in enumerate(sampler_ref.ddim_schedule(1000, 10)):
        out = s.sample_once(xa, torch.tensor([tt] * 3, device="cuda"), torch.tensor([tp] * 3, device="cuda"), classes, prev=prev,
                            strength=0.5, noise=noise_all[i], sde=True)
        prev, xa = (tt, out.pred_x_0), out.pred_x_prev
    a = _run_injected(s, x, classes, 10, noise_all, strength=0.5)
    assert torch.isfinite(a).all()
    assert torch.equal(a, xa), "ivid_sampler_run with injected noise equals chaining sample_once"
    for i in (0, 2):
        b = _run_injected(s, x[i:i + 1], classes[i:i + 1], 10, noise_all[:, i:i + 1], strength=0.5)
        assert torch.equal(b, a[i:i + 1]), f"sample {i} depends on its batch"
    run = lambda: s.sample(3, noise=x, classes=classes, steps=10, strength=0.5, verbose=False, sde=True).samples
    torch.manual_seed(9)
    p = run()
    torch.manual_seed(9)
    assert torch.equal(run(), p), "two runs with the same seed give the same bits"


def test_torch_rng_consumed_as_ddim(golden):
    """rng='torch' draws z with the torch generator where DdimSampler draws it (InpaintCFG hole noise, then randn_like(x_t)):
    the generator ends in the same state, and order 1 then equals DDIM at eta = 1 run for run."""
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    xc = torch.from_numpy(golden["step_x_t"]).cuda(); cc = torch.from_numpy(golden["step_classes"]).cuda()
    kw = dict(noise=xc, classes=cc, steps=5, strength=0.5, verbose=False, rng="torch", **_cond_kwargs(golden))
    for order in (1, 2):
        torch.manual_seed(7)
        a = samplers.DpmSolverSampler(fc).sample(2, order=order, sde=True, **kw)
        ra = torch.randn(4, device="cuda")
        torch.manual_seed(7)
        b = samplers.DdimSampler(fc).sample(2, eta=1.0, **kw)
        assert torch.equal(ra, torch.randn(4, device="cuda")), "the torch RNG is consumed exactly as DdimSampler consumes it"
        if order == 1:
            assert G.report("dpm++ sde order 1 vs ddim eta=1, InpaintCFG + guidance, rng=torch", a.samples, b.samples) < STEP_TOL


def test_sample_all_dpmpp_sde(golden):
    """The multiview pipeline with solver='dpmpp_sde' on the tiny models, viewset 'random'."""
    fu = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    mvs = build_modelviews("random", 3, rng=np.random.default_rng(1))
    kw = dict(fov=45, near=0.6, far=5, atol=0.03, rtol=0.03, erode_rgb=3)
    outs = list(sample_all(fu, fc, [5, 6, 7], 10, 4, mvs, classes=[1, 2, 3], guidance=0.5, batchsize=2, solver="dpmpp_sde", **kw))
    assert len(outs) == 3
    for meshes, colors, samples, conds in outs:
        assert samples.shape == (2, 4, 32, 32) and torch.isfinite(samples).all()
        assert conds["color"].shape == (1, 3, 32, 32) and conds["depth"].shape == (1, 1, 32, 32)

"""GPU: the DPM-Solver++(2M) sampler (DpmSolverSampler, sampler kind 2).  Its first order against the reference's own DDIM
step (golden fixture), the 2M step arithmetic against the float64 oracle (teacher-forced from the GPU's own x_t, D0 and
D_{-1}), whole runs against DdimSampler(eta=0), and the bitwise properties of the native loop: fused == separate route,
loop == chained sample_once, run-to-run and batch independence."""
import json

import numpy as np
import pytest
import torch

import gpu_util as G
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200.inference import build_modelviews, sample_all
from oracle import dpm_ref, sampler_ref, unet_ref

pytestmark = pytest.mark.gpu
STEP_TOL = 1e-3


def _fw(golden, tag, seed, cls):
    cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    return cls(net.cuda(), timesteps=1000, beta_schedule="linear")


def _cond_kwargs(golden):
    y = torch.from_numpy(golden["ddim_y"]).cuda(); mask = torch.from_numpy(golden["ddim_mask"]).cuda()
    mask_rgb = torch.from_numpy(golden["ddim_mask_rgb"]).cuda(); convex = torch.from_numpy(golden["ddim_convex"]).cuda()
    return dict(y=y, mask=mask, mask_rgb=mask_rgb, replace_rgb=(0.1, y[:, :3], mask_rgb), replace_depth=(0.2, y[:, 3:], mask),
                constrain_depth=(0.5, convex))


def test_order1_guided_steps_vs_reference_golden(golden):
    """First order is DDIM with eta = 0: the reference's own DdimSampler outputs (InpaintCFG, guidance 0.5, injected hole
    noise, replace / constrain at the pipeline's weights) at the bar of the DDIM step itself."""
    fw = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    s = samplers.DpmSolverSampler(fw)
    x_t = torch.from_numpy(golden["step_x_t"]).cuda(); classes = torch.from_numpy(golden["step_classes"]).cuda()
    N = x_t.shape[0]
    for (tt, tp) in [(1000, 980), (20, 0)]:
        cn = torch.cat([torch.from_numpy(golden[f"ddim_t{tt}_noise_rgb"]), torch.from_numpy(golden[f"ddim_t{tt}_noise_d"])], 1).cuda()
        out = s.sample_once(x_t, torch.tensor([tt] * N, device="cuda"), torch.tensor([tp] * N, device="cuda"), classes,
                            prev=None, strength=0.5, noise=torch.zeros_like(x_t), cond_noise=cn, **_cond_kwargs(golden))
        r = G.report(f"dpm++ order-1 guided step {tt}->{tp} x_prev", out.pred_x_prev, torch.from_numpy(golden[f"ddim_t{tt}_xprev"]))
        assert r < STEP_TOL and r < 2.6e-4          # the DDIM step's bar (test_ddim_guided_steps_vs_reference_golden)
        if tp == 0:
            assert torch.equal(out.pred_x_prev, out.pred_x_0), "the final step returns x_0"


def test_2m_step_arithmetic_teacher_forced(golden):
    """10-step 2M run: every step's x_{t_prev} recomputed in float64 from the GPU's own x_t, D0 and D_{-1}.  Free of the
    UNet's error, this isolates the update (fp32 coefficients and explicit-rounding arithmetic)."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = samplers.DpmSolverSampler(fw)
    acp = s.alphas_cumprod
    x = torch.from_numpy(np.random.default_rng(0).standard_normal((2, 4, 32, 32)).astype(np.float32)).cuda()
    classes = torch.tensor([1, 2]).cuda()
    res = s.sample(2, noise=x, classes=classes, steps=10, strength=0.5, verbose=False, return_trajectory=True)
    xt = [x] + res.pred_x_t[:-1]
    d0 = [d.double().cpu().numpy() for d in res.pred_x_0]
    worst = 0.0
    for i, (t, tp, t_last, o) in enumerate(dpm_ref.schedule(1000, 10, 2)):
        ref = dpm_ref.update(acp, xt[i].double().cpu().numpy(), d0[i], t, tp, d0[i - 1] if o == 2 else None, t_last if o == 2 else None)
        worst = max(worst, G.report(f"dpm++(2M) step {t}->{tp} (order {o}) vs float64 update", res.pred_x_t[i], torch.from_numpy(ref)))
    assert worst <= 1e-5
    assert torch.equal(res.pred_x_t[-1], res.pred_x_0[-1]) and torch.equal(res.samples, res.pred_x_t[-1])


def test_order1_runs_vs_ddim_eta0(golden):
    """Whole first-order runs against DdimSampler(eta=0) from the same x_T: the unconditional CFG model (Philox), and the
    InpaintCFG model with guidance, seeded with rng='torch' so that both draw the same hole noise."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    x = torch.from_numpy(np.random.default_rng(1).standard_normal((2, 4, 32, 32)).astype(np.float32)).cuda()
    classes = torch.tensor([1, 2]).cuda()
    a = samplers.DpmSolverSampler(fw).sample(2, noise=x, classes=classes, steps=10, order=1, strength=0.5, verbose=False).samples
    b = samplers.DdimSampler(fw).sample(2, noise=x, classes=classes, steps=10, eta=0.0, strength=0.5, verbose=False).samples
    assert G.report("dpm++ order 1 vs ddim eta=0, 10 steps", a, b) < STEP_TOL
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    xc = torch.from_numpy(golden["step_x_t"]).cuda(); cc = torch.from_numpy(golden["step_classes"]).cuda()
    kw = dict(noise=xc, classes=cc, steps=5, strength=0.5, verbose=False, rng="torch", **_cond_kwargs(golden))
    torch.manual_seed(7)
    a = samplers.DpmSolverSampler(fc).sample(2, order=1, **kw)
    ra = torch.randn(4)
    torch.manual_seed(7)
    b = samplers.DdimSampler(fc).sample(2, eta=0.0, **kw)
    assert torch.equal(ra, torch.randn(4)), "the torch RNG is consumed exactly as DdimSampler consumes it"
    assert G.report("dpm++ order 1 vs ddim eta=0, InpaintCFG + guidance, rng=torch", a.samples, b.samples) < STEP_TOL


def test_fused_equals_separate_route(golden):
    """Without trajectories the update runs inside the output head's kernel; with them, in the separate step kernel.  The
    arithmetic is pinned by explicit rounding: same bits, on both models (the InpaintCFG one with Philox hole noise)."""
    fu = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    x = torch.from_numpy(np.random.default_rng(2).standard_normal((2, 4, 32, 32)).astype(np.float32)).cuda()
    classes = torch.tensor([1, 2]).cuda()
    for fw, kw in ((fu, {}), (fc, _cond_kwargs(golden))):
        s = samplers.DpmSolverSampler(fw)
        torch.manual_seed(5)
        a = s.sample(2, noise=x, classes=classes, steps=8, strength=0.5, verbose=False, **kw).samples
        torch.manual_seed(5)
        b = s.sample(2, noise=x, classes=classes, steps=8, strength=0.5, verbose=False, return_trajectory=True, **kw)
        G.report(f"{type(fw).__name__}: dpm++ fused vs separate", a, b.samples)
        assert torch.isfinite(a).all()
        assert torch.equal(a, b.samples)


def test_loop_equals_chained_sample_once_and_is_deterministic(golden):
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = samplers.DpmSolverSampler(fw)
    x = torch.from_numpy(np.random.default_rng(3).standard_normal((3, 4, 32, 32)).astype(np.float32)).cuda()
    classes = torch.tensor([1, 2, 3]).cuda()
    xa, prev = x.clone(), None
    for (tt, tp) in sampler_ref.ddim_schedule(1000, 10):
        out = s.sample_once(xa, torch.tensor([tt] * 3, device="cuda"), torch.tensor([tp] * 3, device="cuda"), classes, prev=prev,
                            strength=0.5, noise=torch.zeros_like(xa))
        prev, xa = (tt, out.pred_x_0), out.pred_x_prev
    run = lambda xx, cc: s.sample(xx.shape[0], noise=xx, classes=cc, steps=10, strength=0.5, verbose=False).samples
    a = run(x, classes)
    assert torch.isfinite(a).all()
    assert torch.equal(a, xa), "the whole loop equals chaining sample_once"
    assert torch.equal(run(x, classes), a), "two runs give the same bits"
    for i in (0, 2):
        assert torch.equal(run(x[i:i + 1].contiguous(), classes[i:i + 1]), a[i:i + 1]), f"sample {i} depends on its batch"


def test_sample_all_dpmpp(golden):
    """The multiview pipeline with solver='dpmpp' on the tiny models, viewset 'random': unconditional view below 1000 steps
    and the guided conditional view both run DpmSolverSampler."""
    fu = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    mvs = build_modelviews("random", 3, rng=np.random.default_rng(1))
    kw = dict(fov=45, near=0.6, far=5, atol=0.03, rtol=0.03, erode_rgb=3)
    outs = list(sample_all(fu, fc, [5, 6, 7], 10, 4, mvs, classes=[1, 2, 3], guidance=0.5, batchsize=2, solver="dpmpp", **kw))
    assert len(outs) == 3
    for meshes, colors, samples, conds in outs:
        assert samples.shape == (2, 4, 32, 32) and torch.isfinite(samples).all()
        assert conds["color"].shape == (1, 3, 32, 32) and conds["depth"].shape == (1, 1, 32, 32)

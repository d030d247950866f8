"""GPU: the UniPC sampler (UniPcSampler, sampler kind 2 with unipc = 1).  Every step of guided runs at orders 2 and 3 against the
float64 UniPC step computed from the GPU's own x_t, D0, history and base; the bitwise properties of the native loop (fused ==
separate route, loop == chained sample_once, run to run, batch independence, cache_interval=1 == no caching, a full guidance
interval == none), the loop == chain equality with every option the step composes with, no allocation in a warm run, and the
multiview pipeline with solver='unipc'."""
import ctypes
import json

import numpy as np
import pytest
import torch

import gpu_util as G
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
import unipc_ref
from ivid_b200 import _lib
from ivid_b200.inference import build_modelviews, sample_all
from oracle import sampler_ref, unet_ref

pytestmark = pytest.mark.gpu
T = 1000
STEP_BAR = 1e-6          # float64 step from the GPU's own inputs; the measured worst case is printed by the test


def _fw(golden, tag, seed, cls):
    cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    return cls(net.cuda(), timesteps=T, beta_schedule="linear")


def _randn(seed, shape, scale=1.0):
    return torch.from_numpy((np.random.default_rng(seed).standard_normal(shape) * scale).astype(np.float32)).cuda()


def _cond_kwargs(golden):
    y = torch.from_numpy(golden["ddim_y"]).cuda(); mask = torch.from_numpy(golden["ddim_mask"]).cuda()
    mask_rgb = torch.from_numpy(golden["ddim_mask_rgb"]).cuda(); convex = torch.from_numpy(golden["ddim_convex"]).cuda()
    return dict(y=y, mask=mask, mask_rgb=mask_rgb, replace_rgb=(0.1, y[:, :3], mask_rgb), replace_depth=(0.2, y[:, 3:], mask),
                constrain_depth=(0.5, convex))


def _chain(s, x, classes, steps, order, cond_noise=None, reuse=None, **kw):
    """sample_once chained as the docstring says; returns the outputs of every step."""
    N = x.shape[0]
    xa, prev, px, outs = x.clone(), [], None, []
    for i, (t, tp) in enumerate(sampler_ref.ddim_schedule(T, steps)):
        extra = dict(cond_noise=cond_noise[i]) if cond_noise is not None else {}
        out = s.sample_once(xa, torch.full((N,), t, device="cuda"), torch.full((N,), tp, device="cuda"), classes, prev=prev,
                            prev_x=px, order=order, noise=torch.zeros_like(xa), reuse_features=bool(reuse and reuse[i]),
                            **extra, **kw)
        prev, px, xa = ([(t, out.pred_x_0)] + prev)[:3], out.corrected_x_t, out.pred_x_prev
        outs.append(out)
    return outs


def _run_native(s, x, classes, steps, order, cond_noise_all=None, interval=None, cache_interval=None, threshold=None, **kw):
    """ivid_sampler_run with the conditional hole noise injected (the separate route)."""
    net = s._net()
    img = x.clone().contiguous()
    a, keep = s._step_args(img.device, classes, False, 0.0, kw, seed=0, hw=img.shape[-2:], order=order, interval=interval,
                           cache=(cache_interval or 0, 0, 0), threshold=samplers.samplers._check_threshold(threshold, False))
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().ivid_sampler_run(s._handle, net._handle, _lib.ptr(img), img.shape[0], steps, ctypes.byref(a), None,
                                               _lib.ptr(cond_noise_all), None, None, _lib.cur_stream(img.device)))
    torch.cuda.synchronize()
    del keep
    return img


@pytest.mark.parametrize("order", [2, 3])
def test_step_arithmetic_teacher_forced(golden, order):
    """Guided 10-step runs (classifier-free guidance 0.5; InpaintCFG with the multiview replace / constrain guidance): every
    step's prediction and corrected x_t against the float64 UniPC step from the GPU's own x_t, D0, history and base."""
    acp = sampler_ref.Tables(sampler_ref.get_betas("linear", T)).alphas_cumprod
    worst = 0.0
    for tag, cls in (("tiny", frameworks.ClassifierFreeGuidance), ("tiny_cond", frameworks.InpaintCFG)):
        fw = _fw(golden, tag, 1234 if tag == "tiny" else 4321, cls)
        s = samplers.UniPcSampler(fw)
        if tag == "tiny":
            x, classes, kw = _randn(0, (2, 4, 32, 32)), torch.tensor([1, 2]).cuda(), {}
        else:
            x, kw = torch.from_numpy(golden["step_x_t"]).cuda(), _cond_kwargs(golden)
            classes = torch.from_numpy(golden["step_classes"]).cuda()
        cn = _randn(1, (10,) + tuple(x.shape)) if tag == "tiny_cond" else None
        outs = _chain(s, x, classes, 10, order, cond_noise=cn, strength=0.5, **kw)
        f64 = lambda v: v.double().cpu().numpy()
        xt, hist, base = f64(x), [], None
        for i, (t, tp, q, q_c) in enumerate(unipc_ref.schedule(T, 10, order)):
            d0 = f64(outs[i].pred_x_0)
            ref_p, ref_c = unipc_ref.step(acp, xt, d0, t, tp, q, q_c, hist, base)
            name = f"{tag} UniPC-{order} step {t}->{tp} (predictor {q}, corrector {q_c})"
            worst = max(worst, G.report(name + " x_prev", outs[i].pred_x_prev, torch.from_numpy(ref_p)),
                        G.report(name + " corrected x_t", outs[i].corrected_x_t, torch.from_numpy(ref_c)))
            if q_c == 0:
                assert torch.equal(outs[i].corrected_x_t, outs[i - 1].pred_x_prev if i else x)
            xt, hist, base = f64(outs[i].pred_x_prev), [(t, d0)] + hist, f64(outs[i].corrected_x_t)
        assert torch.equal(outs[-1].pred_x_prev, outs[-1].pred_x_0), "the final step returns x_0"
    print(f"[unipc] order {order}: worst relative L2 against the float64 step {worst:.3e}")
    assert worst <= STEP_BAR


@pytest.mark.parametrize("order", [2, 3])
def test_fused_equals_separate_route(golden, order):
    fu = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    x = _randn(2, (2, 4, 32, 32))
    classes = torch.tensor([1, 2]).cuda()
    for fw, kw in ((fu, {}), (fc, _cond_kwargs(golden))):
        s = samplers.UniPcSampler(fw)
        torch.manual_seed(5)
        a = s.sample(2, noise=x, classes=classes, steps=8, order=order, strength=0.5, verbose=False, **kw).samples
        torch.manual_seed(5)
        b = s.sample(2, noise=x, classes=classes, steps=8, order=order, strength=0.5, verbose=False, return_trajectory=True, **kw)
        assert torch.isfinite(a).all()
        assert torch.equal(a, b.samples), type(fw).__name__
        assert torch.equal(b.pred_x_t[-1], b.samples) and torch.equal(b.pred_x_0[-1], b.samples)


@pytest.mark.parametrize("order", [1, 2, 3])
def test_loop_equals_chained_sample_once_and_is_deterministic(golden, order):
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = samplers.UniPcSampler(fw)
    x = _randn(3, (3, 4, 32, 32))
    classes = torch.tensor([1, 2, 3]).cuda()
    chain = _chain(s, x, classes, 10, order, strength=0.5)
    run = lambda xx, cc, **o: s.sample(xx.shape[0], noise=xx, classes=cc, steps=10, order=order, strength=0.5, verbose=False, **o)
    a = run(x, classes).samples
    assert torch.isfinite(a).all()
    assert torch.equal(a, chain[-1].pred_x_prev), "the whole loop equals chaining sample_once"
    traj = run(x, classes, return_trajectory=True)
    assert all(torch.equal(traj.pred_x_t[i], chain[i].pred_x_prev) for i in range(10)), "pred_x_t holds the predictions"
    assert all(torch.equal(traj.pred_x_0[i], chain[i].pred_x_0) for i in range(10))
    assert torch.equal(run(x, classes).samples, a), "two runs give the same bits"
    for i in (0, 2):
        assert torch.equal(run(x[i:i + 1].contiguous(), classes[i:i + 1]).samples, a[i:i + 1]), f"sample {i} depends on its batch"
    # the torch RNG path runs the same steps
    torch.manual_seed(1)
    b = run(x, classes, rng="torch").samples
    assert torch.equal(a, b), "rng='torch' equals the native loop (UniPC draws no step noise)"


def test_trivial_options_change_nothing(golden):
    """cache_interval=1 runs every forward in full and a guidance interval over every model time guides every step: the same
    bits as neither."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = samplers.UniPcSampler(fw)
    x = _randn(4, (2, 4, 32, 32))
    classes = torch.tensor([4, 5]).cuda()
    run = lambda **o: s.sample(2, noise=x, classes=classes, steps=10, order=3, strength=0.5, verbose=False, **o).samples
    a = run()
    assert torch.equal(run(cache_interval=1), a)
    assert torch.equal(run(guidance_interval=(0, T - 1)), a)


LOOP_CASES = {   # name: (model tag, framework, run / step options)
    "inpaint": ("tiny_cond", frameworks.InpaintCFG, {}),
    "superres": ("tiny_sr", frameworks.SuperResCFG, {}),
    "fp8": ("tiny", frameworks.ClassifierFreeGuidance, dict(fp8=True)),
    "interval": ("tiny", frameworks.ClassifierFreeGuidance, dict(interval=(300, 700))),
    "cache": ("tiny", frameworks.ClassifierFreeGuidance, dict(cache=3)),
    "threshold": ("tiny", frameworks.ClassifierFreeGuidance, dict(threshold=(0.995, 4.0))),
}


@pytest.mark.parametrize("case", list(LOOP_CASES))
def test_loop_equals_chain_with_options(golden, case):
    """ivid_sampler_run (host route) == chained sample_once (device route), order 3, with each option UniPC composes with."""
    tag, cls, opt = LOOP_CASES[case]
    fw = _fw(golden, tag, 4321 if tag == "tiny_cond" else 1234, cls)
    if opt.get("fp8"):
        fw.backbone.set_precision("fp8")
    s = samplers.UniPcSampler(fw)
    steps, strength = 10, 3.0
    kw, cn = {}, None
    if tag == "tiny_cond":
        x, kw = torch.from_numpy(golden["step_x_t"]).cuda(), _cond_kwargs(golden)
        cn = _randn(5, (steps,) + tuple(x.shape))
    elif tag == "tiny_sr":
        x, kw = torch.from_numpy(golden["sr_x"]).cuda(), dict(y=torch.from_numpy(golden["sr_y"]).cuda())
    else:
        x = _randn(6, (3, 4, 32, 32), 2.0)
    N = x.shape[0]
    classes = torch.arange(1, N + 1).cuda()
    interval, cache_interval, threshold = opt.get("interval"), opt.get("cache"), opt.get("threshold")
    a = _run_native(s, x, classes, steps, 3, cond_noise_all=cn, interval=interval, cache_interval=cache_interval,
                    threshold=threshold, strength=strength, **kw)
    sched = sampler_ref.ddim_schedule(T, steps)
    reuse = s._reuse_schedule([t - 1 for (t, _) in sched], classes, dict(strength=strength), interval, cache_interval or 0)
    chain = _chain(s, x, classes, steps, 3, cond_noise=cn, reuse=reuse, strength=strength, guidance_interval=interval,
                   dynamic_threshold=threshold, **kw)
    assert torch.isfinite(a).all()
    assert torch.equal(a, chain[-1].pred_x_prev), case
    if cn is None:       # Philox hole noise otherwise: the fused run is compared with itself
        b = s.sample(N, noise=x, classes=classes, steps=steps, order=3, strength=strength, verbose=False, guidance_interval=interval,
                     cache_interval=cache_interval, dynamic_threshold=threshold, **kw).samples
        assert torch.equal(a, b), case + ": fused route"


def test_warm_run_allocates_nothing(golden):
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = samplers.UniPcSampler(fw)
    x = _randn(7, (2, 4, 32, 32))
    classes = torch.tensor([1, 2]).cuda()
    run = lambda: s.sample(2, noise=x, classes=classes, steps=10, order=3, strength=0.5, verbose=False).samples
    run()
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info()[0]
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == before


def test_sample_all_unipc(golden):
    """The multiview pipeline with solver='unipc' on the tiny models, viewset 'random'."""
    fu = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    mvs = build_modelviews("random", 3, rng=np.random.default_rng(1))
    kw = dict(fov=45, near=0.6, far=5, atol=0.03, rtol=0.03, erode_rgb=3)
    outs = list(sample_all(fu, fc, [5, 6, 7], 10, 4, mvs, classes=[1, 2, 3], guidance=0.5, batchsize=2, solver="unipc", **kw))
    assert len(outs) == 3
    for meshes, colors, samples, conds in outs:
        assert samples.shape == (2, 4, 32, 32) and torch.isfinite(samples).all()

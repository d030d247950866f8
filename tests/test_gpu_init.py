"""GPU: runs started from a given image.  The forward diffusion (ivid_sampler_diffuse) against the reference's
GaussianDiffusion.diffuse and its Philox noise; the tail identity of a run started at grid step k (ivid_sampler_run with
start_step = k on the x_k of a full run gives the full run's samples bit for bit, DDPM and DDIM, with the guidance interval
and dynamic thresholding); the multistep solvers started at k against chained sample_once calls with an empty history;
`sample(init=..., init_strength=...)` as diffuse + partial run; and sample_all with given first views."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from ivid_b200.frameworks.utils import get_betas_by_name
from ivid_b200.inference import build_modelviews, sample_all
from ivid_b200.rgbd_3d import DeviceWarp
from oracle import sampler_ref, unet_ref

pytestmark = pytest.mark.gpu
T = 1000
HERE = os.path.dirname(os.path.abspath(__file__))
INIT = np.load(os.path.join(HERE, "golden", "init_golden.npz"))
WARP_KW = dict(fov=45, near=0.6, far=5, atol=0.03, rtol=0.03, erode_rgb=3)


def _fw(golden, tag, seed, cls):
    cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    return cls(net.cuda(), timesteps=T, beta_schedule="linear")


def _randn(seed, shape, scale=1.0):
    return torch.from_numpy((np.random.default_rng(seed).standard_normal(shape) * scale).astype(np.float32)).cuda()


def _diffuse(s, x0, t, noise=None, seed=0):
    out = torch.empty_like(x0)
    _lib.check(_lib.lib().ivid_sampler_diffuse(s._handle, _lib.ptr(x0), _lib.ptr(noise), x0.shape[0], x0[0].numel(), t, seed,
                                               _lib.ptr(out), _lib.cur_stream()))
    torch.cuda.synchronize()
    return out


def _run_from(s, x, classes, steps, start, seed=0, noise_all=None, traj=False, order=0, sde=False, eta=0.0, interval=None,
              cache_interval=None, threshold=None, **kw):
    """ivid_sampler_run from grid step `start` on x (a copy); returns the samples (and the trajectories)."""
    net = s._net()
    img = x.clone().contiguous()
    a, keep = s._step_args(img.device, classes, False, eta, kw, seed=seed, hw=img.shape[-2:], order=order, sde=sde,
                           interval=interval, cache=(cache_interval or 0, 0, 0),
                           threshold=samplers.samplers._check_threshold(threshold, False))
    a.start_step = start
    n = (T if s.KIND == 0 else steps) - start
    t0 = t1 = None
    if traj:
        t0 = torch.empty((n,) + tuple(img.shape), device="cuda")
        t1 = torch.empty((n,) + tuple(img.shape), device="cuda")
    _lib.check(_lib.lib().ivid_sampler_run(s._handle, net._handle, _lib.ptr(img), img.shape[0], steps, ctypes.byref(a),
                                           _lib.ptr(noise_all), None, _lib.ptr(t0), _lib.ptr(t1), _lib.cur_stream()))
    torch.cuda.synchronize()
    del keep
    return (img, t0, t1) if traj else img


def _philox_seed(torch_seed):
    """The Philox seed sample() draws after torch.manual_seed(torch_seed) when no torch draw precedes it."""
    torch.manual_seed(torch_seed)
    return int(torch.randint(0, 2 ** 62, (1,)).item())


# ------------------------------------------------------------------------------------------------------------ diffuse
@pytest.mark.parametrize("schedule", ["linear", "cosine"])
def test_diffuse_matches_reference(schedule):
    """Injected noise: the reference's GaussianDiffusion.diffuse bit for bit (coefficients rounded once to fp32 as extract
    rounds them, then fp32 mul, mul, add), at every t of the fixture."""
    betas = get_betas_by_name(schedule, T).astype(np.float64)
    fw = type("Fw", (), {"betas": betas, "timesteps": T})()
    s = samplers.DdimSampler(fw)
    x0 = torch.from_numpy(INIT["diffuse_x0"]).cuda()
    z = torch.from_numpy(INIT["diffuse_noise"]).cuda()
    for i, t in enumerate(INIT["diffuse_t"]):
        got = _diffuse(s, x0, int(t), z).cpu().numpy()
        ref = INIT[f"diffuse_{schedule}"][i]
        assert np.array_equal(got, ref), f"{schedule} t={t}: max |diff| {np.abs(got - ref).max()}"


def test_diffuse_philox_noise(golden):
    """Philox z: mean 0 and variance 1 within 6 standard errors over 2^20 draws, the same bits call to call, another seed
    gives other noise, and it is uncorrelated with the step noise of stream 0 (the first step of a run) of the same seed."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = samplers.DdimSampler(fw)
    seed = 0x1234567890ABC
    x0 = torch.zeros(256, 4, 32, 32, device="cuda")
    t = T - 1
    b = np.float32(np.sqrt(1.0 - s.alphas_cumprod[t]))
    z = _diffuse(s, x0, t, seed=seed).double() / float(b)
    n = z.numel()
    mean, var = float(z.mean()), float(z.var())
    print(f"[diffuse] Philox z over {n} draws: mean {mean:+.2e}, variance {var:.5f}")
    assert abs(mean) < 6 / np.sqrt(n) and abs(var - 1) < 6 * np.sqrt(2 / n)
    assert torch.equal(_diffuse(s, x0, t, seed=seed), _diffuse(s, x0, t, seed=seed)), "reproducible call to call"
    assert not torch.equal(_diffuse(s, x0, t, seed=seed + 1), _diffuse(s, x0, t, seed=seed))
    # the step noise of stream 0: a 2-step DDIM run at eta = 1 from x, once with Philox and once with injected zero noise;
    # after the first step the two differ by sigma * z_0
    x = _randn(1, (256, 4, 32, 32))
    classes = torch.arange(256, device="cuda") % 10
    _, _, tp = _run_from(s, x, classes, 2, 0, seed=seed, traj=True, eta=1.0, strength=0.5)
    _, _, t0 = _run_from(s, x, classes, 2, 0, seed=seed, traj=True, eta=1.0, strength=0.5,
                         noise_all=torch.zeros(2, 256, 4, 32, 32, device="cuda"))
    z0 = (tp[0] - t0[0]).double()
    r = float(((z0 - z0.mean()) * (z - z.mean())).mean() / (z0.std() * z.std()))
    print(f"[diffuse] correlation with the stream-0 step noise: {r:+.2e}")
    assert float(z0.std()) > 0.1 and abs(r) < 6 / np.sqrt(n)


# ------------------------------------------------------------------------------------------------------- tail identity
TAIL_CASES = {   # name: (sampler, steps, k, options)
    "ddpm": (samplers.DdpmSampler, T, 600, {}),
    "ddpm_interval_threshold": (samplers.DdpmSampler, T, 850, dict(guidance_interval=(200, 700), dynamic_threshold=(0.99, 3.0))),
    "ddim_eta0": (samplers.DdimSampler, 20, 7, {}),
    "ddim_eta1": (samplers.DdimSampler, 20, 12, dict(eta=1.0)),
    "ddim_eta1_interval_threshold": (samplers.DdimSampler, 20, 5, dict(eta=1.0, guidance_interval=(300, 700),
                                                                         dynamic_threshold=0.995)),
}


@pytest.mark.parametrize("case", list(TAIL_CASES))
def test_tail_identity_philox(golden, case):
    """A seeded Philox run's x at grid step k, run on from k with the same seed, ends in the full run's samples bit for bit."""
    cls, steps, k, opt = TAIL_CASES[case]
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = cls(fw)
    x = _randn(2, (2, 4, 32, 32))
    classes = torch.tensor([3, 7]).cuda()
    seed = _philox_seed(11)
    torch.manual_seed(11)
    full = s.sample(2, noise=x, classes=classes, steps=steps, strength=0.5, verbose=False, return_trajectory=True, **opt)
    x_k = full.pred_x_t[k - 1]                    # x after step k - 1: the input of step k
    run_opt = dict(eta=opt.get("eta", 0.0), interval=opt.get("guidance_interval"), threshold=opt.get("dynamic_threshold"))
    tail, t0, t1 = _run_from(s, x_k, classes, steps, k, seed=seed, traj=True, strength=0.5, **run_opt)
    assert torch.isfinite(tail).all()
    assert torch.equal(tail, full.samples), case
    assert t1.shape[0] == len(full.pred_x_t) - k and all(torch.equal(t1[j], full.pred_x_t[k + j]) for j in range(t1.shape[0]))
    # the fused route (no trajectories) gives the same bits
    assert torch.equal(_run_from(s, x_k, classes, steps, k, seed=seed, strength=0.5, **run_opt), full.samples)


# ------------------------------------------------------------------------------------------ multistep: started at k
def _chain_dpm(s, x, classes, sched, noise=None, reuse=None, **kw):
    xa, prev = x.clone(), None
    N = x.shape[0]
    for j, (t, tp) in enumerate(sched):
        out = s.sample_once(xa, torch.full((N,), t, device="cuda"), torch.full((N,), tp, device="cuda"), classes, prev=prev,
                            noise=noise[j] if noise is not None else torch.zeros_like(xa),
                            reuse_features=bool(reuse and reuse[j]), **kw)
        prev, xa = (t, out.pred_x_0), out.pred_x_prev
    return xa


def _chain_unipc(s, x, classes, sched, order, reuse=None, **kw):
    xa, prev, px = x.clone(), [], None
    N = x.shape[0]
    for j, (t, tp) in enumerate(sched):
        out = s.sample_once(xa, torch.full((N,), t, device="cuda"), torch.full((N,), tp, device="cuda"), classes, prev=prev,
                            prev_x=px, order=order, noise=torch.zeros_like(xa), reuse_features=bool(reuse and reuse[j]), **kw)
        prev, px, xa = ([(t, out.pred_x_0)] + prev)[:3], out.corrected_x_t, out.pred_x_prev
    return xa


MULTI_CASES = ["dpmpp", "dpmpp_sde", "unipc1", "unipc2", "unipc3", "dpmpp_cache", "unipc3_cache"]


@pytest.mark.parametrize("case", MULTI_CASES)
def test_multistep_started_at_k_equals_chain(golden, case):
    """DPM-Solver++ (ODE and SDE) and UniPC orders 1-3 run from grid step k = 4 of 12 equal the chain of sample_once calls over
    the same steps with the history starting empty, bit for bit (the run-vs-chain bar of the solvers' own tests); with
    feature reuse the chain reuses where the run does, counted from the first executed step."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    unipc = case.startswith("unipc")
    s = samplers.UniPcSampler(fw) if unipc else samplers.DpmSolverSampler(fw)
    steps, k = 12, 4
    order = int(case[5]) if unipc else 2
    sde = case == "dpmpp_sde"
    cache_interval = 3 if case.endswith("_cache") else None
    x = _randn(3, (3, 4, 32, 32), 0.8)
    classes = torch.tensor([1, 2, 3]).cuda()
    sched = sampler_ref.ddim_schedule(T, steps)[k:]
    noise = _randn(4, (steps - k, 3, 4, 32, 32)) if sde else None
    reuse = s._reuse_schedule([t - 1 for (t, _) in sched], classes, dict(strength=0.5), None, cache_interval or 0)
    assert not cache_interval or (not reuse[0] and any(reuse))
    a = _run_from(s, x, classes, steps, k, noise_all=noise, order=order, sde=sde, cache_interval=cache_interval, strength=0.5)
    if unipc:
        b = _chain_unipc(s, x, classes, sched, order, reuse=reuse, strength=0.5)
    else:
        b = _chain_dpm(s, x, classes, sched, noise=noise, reuse=reuse, sde=sde, strength=0.5)
    assert torch.isfinite(a).all()
    assert torch.equal(a, b), case


# ---------------------------------------------------------------------------------------------------- the Python surface
@pytest.mark.parametrize("cls", [samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler, samplers.UniPcSampler])
def test_sample_init_is_diffuse_then_partial_run(golden, cls):
    """sample(init=x_0, init_strength=s) with rng='philox' is ivid_sampler_diffuse at model time jump * n - 1 with the run's
    seed, then the run from start_step = steps - n: bit for bit, with given noise and with Philox noise."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = cls(fw)
    steps = T if cls is samplers.DdpmSampler else 10
    strength = 0.3
    n = samplers.init_steps(strength, steps)
    jump = 1 if cls is samplers.DdpmSampler else T // steps
    x0 = _randn(5, (2, 4, 32, 32), 0.5).clamp(-1, 1)
    z = _randn(6, (2, 4, 32, 32))
    classes = torch.tensor([2, 9]).cuda()
    extra = dict(order=2) if cls in (samplers.DpmSolverSampler, samplers.UniPcSampler) else {}
    for noise in (z, None):
        seed = _philox_seed(21)
        torch.manual_seed(21)
        res = s.sample(2, init=x0, init_strength=strength, noise=noise, classes=classes, steps=steps, strength=0.5, verbose=False,
                       return_trajectory=True, **extra)
        x_k = _diffuse(s, x0, jump * n - 1, noise, seed)
        if noise is not None:
            assert torch.equal(x_k, fw.diffuse(x0, torch.full((2,), jump * n - 1, device="cuda"), noise)), "diffuse() of the framework"
        ref = _run_from(s, x_k, classes, steps, steps - n, seed=seed, strength=0.5, **extra)
        assert torch.isfinite(res.samples).all()
        assert torch.equal(res.samples, ref), (cls.__name__, noise is None)
        assert len(res.pred_x_t) == n and len(res.pred_x_0) == n and torch.equal(res.pred_x_t[-1], res.samples)
    # strength 1 runs the whole grid from the noised x_0
    torch.manual_seed(3)
    full = s.sample(2, init=x0, init_strength=1.0, noise=z, classes=classes, steps=steps, strength=0.5, verbose=False,
                    return_trajectory=True, **extra)
    assert len(full.pred_x_t) == steps


def test_torch_rng_init_matches_philox_for_ode(golden):
    """rng='torch' with given noise runs the same steps as the native loop for UniPC (no step noise): the same bits; without
    noise it draws z = randn_like(x_0) first."""
    fw = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    s = samplers.UniPcSampler(fw)
    x0 = _randn(7, (2, 4, 32, 32), 0.5)
    z = _randn(8, (2, 4, 32, 32))
    classes = torch.tensor([1, 4]).cuda()
    run = lambda **o: s.sample(2, init=x0, init_strength=0.5, classes=classes, steps=10, order=3, strength=0.5, verbose=False, **o)
    a = run(noise=z).samples
    assert torch.equal(run(noise=z, rng="torch").samples, a)
    torch.manual_seed(4)
    zt = torch.randn_like(x0)
    torch.manual_seed(4)
    assert torch.equal(run(rng="torch").samples, run(noise=zt).samples)


@pytest.mark.parametrize("kind", ["inpaint", "superres"])
def test_conditional_frameworks_with_init(golden, kind):
    """InpaintCFG (with the replace / constrain guidance) and SuperResCFG runs from an image: finite, and equal to their
    sample_once chains from the diffused image (DDIM, injected hole noise)."""
    if kind == "inpaint":
        fw = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
        y = torch.from_numpy(golden["ddim_y"]).cuda(); mask = torch.from_numpy(golden["ddim_mask"]).cuda()
        mask_rgb = torch.from_numpy(golden["ddim_mask_rgb"]).cuda(); convex = torch.from_numpy(golden["ddim_convex"]).cuda()
        kw = dict(y=y, mask=mask, mask_rgb=mask_rgb, replace_rgb=(0.1, y[:, :3], mask_rgb), replace_depth=(0.2, y[:, 3:], mask),
                  constrain_depth=(0.5, convex))
        x0 = y.clone()
    else:
        fw = _fw(golden, "tiny_sr", 1234, frameworks.SuperResCFG)
        x0 = torch.from_numpy(golden["sr_x"]).cuda().clamp(-1, 1)
        kw = dict(y=torch.from_numpy(golden["sr_y"]).cuda())
    s = samplers.DdimSampler(fw)
    N = x0.shape[0]
    classes = torch.arange(1, N + 1).cuda()
    steps, strength = 10, 0.6
    n = samplers.init_steps(strength, steps)
    z = _randn(9, tuple(x0.shape))
    torch.manual_seed(8)
    res = s.sample(N, init=x0, init_strength=strength, noise=z, classes=classes, steps=steps, strength=3.0, verbose=False,
                   rng="torch", **kw)
    assert torch.isfinite(res.samples).all()
    # the torch path draws the hole noise then randn_like(x_t) per step; replay the same draws into the chain
    torch.manual_seed(8)
    xa = _diffuse(s, x0.contiguous(), (T // steps) * n - 1, z)
    for (t, tp) in sampler_ref.ddim_schedule(T, steps)[steps - n:]:
        out = s.sample_once(xa, torch.full((N,), t, device="cuda"), torch.full((N,), tp, device="cuda"), classes, strength=3.0, **kw)
        xa = out.pred_x_prev
    assert torch.equal(res.samples, xa), kind


# ------------------------------------------------------------------------------------------------------------ sample_all
def test_sample_all_given_first_view(golden):
    """init_views without a strength: no unconditional model (framework_uncond is None), view 0 is the given view bit for bit,
    and view 1's conditions are DeviceWarp.aggregate after add_view of the given view, bit for bit."""
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    mvs = build_modelviews("random", 2, rng=np.random.default_rng(3))
    views = _randn(10, (2, 4, 32, 32), 0.5).clamp(-1, 1)
    outs = list(sample_all(None, fc, [5, 6], 10, 4, mvs, classes=[1, 2], guidance=0.5, batchsize=2, init_views=views, **WARP_KW))
    assert len(outs) == 2
    warp = DeviceWarp(2, image_size=32, ssaa=3, max_views=2, device=0)
    warp.reset()
    warp.add_view(views, [mvs[k][0] for k in range(2)], **WARP_KW)
    cond = warp.aggregate([mvs[k][1] for k in range(2)], **WARP_KW)
    for k, (meshes, colors, samples, conds) in enumerate(outs):
        assert samples.shape == (2, 4, 32, 32) and torch.isfinite(samples).all()
        assert torch.equal(samples[0], views[k]), "view 0 is the given view"
        assert torch.equal(conds["color"][0], cond[k, 0:3] * 2 - 1) and torch.equal(conds["depth"][0], cond[k, 3:4] * 2 - 1)


def test_sample_all_sdedit_first_view(golden):
    """init_views with a strength: view 0 is sampler.sample(init=..., init_strength=...) of the unconditional sampler run alone
    with the same seeds."""
    fu = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    mvs = build_modelviews("random", 2, rng=np.random.default_rng(4))
    views = _randn(11, (2, 4, 32, 32), 0.5).clamp(-1, 1)
    seeds, classes = [5, 6], [1, 2]
    outs = list(sample_all(fu, fc, seeds, 10, 4, mvs, classes=classes, guidance=0.5, batchsize=2, init_views=views,
                           init_strength=0.4, **WARP_KW))
    noise = []
    for sd in seeds:
        torch.manual_seed(sd)
        noise.append(torch.randn(1, 4, 32, 32, device="cuda"))
    ref = samplers.DdimSampler(fu).sample(2, noise=torch.cat(noise), classes=torch.tensor(classes).cuda(), steps=10, strength=0.5,
                                          verbose=False, init=views, init_strength=0.4).samples
    for k, (_, _, samples, _) in enumerate(outs):
        assert torch.isfinite(samples).all()
        assert torch.equal(samples[0], ref[k])
        assert not torch.equal(samples[0], views[k])

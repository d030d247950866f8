"""CPU: the DPM-Solver++(2M) sampler's arithmetic (float64 oracle), its convergence order on data with a closed-form
probability-flow ODE, its per-step order pattern, and the host-side error contract of the new sampler kind."""
import ctypes
import json

import numpy as np
import pytest
import torch

import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from oracle import dpm_ref, sampler_ref

T = 1000
ACP = sampler_ref.Tables(sampler_ref.get_betas("linear", T)).alphas_cumprod
TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16], channel_mult=[1, 2], num_head_channels=64)


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b)))


@pytest.mark.parametrize("clip", [False, True])
def test_order1_is_ddim_eta0_with_guidance(monkeypatch, clip):
    """First order is DDIM with eta = 0, algebraically: the oracle step against sampler_ref.ddim_step (its table lookup kept
    in float64, so both sides are float64 throughout), with the multiview replace / constrain guidance at the pipeline's
    weights, on ordinary steps and on the final step to t_prev = 0."""
    monkeypatch.setattr(sampler_ref, "_ex", lambda arr, t, nd: torch.from_numpy(arr)[t].view(-1, *([1] * (nd - 1))))
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", T))
    rng = np.random.default_rng(3)
    N, H = 2, 8
    x_t, eps = rng.standard_normal((N, 4, H, H)), rng.standard_normal((N, 4, H, H))
    y = rng.uniform(-1, 1, (N, 4, H, H))
    mask = (rng.uniform(size=(N, 1, H, H)) > 0.4).astype(np.float64)
    mask_rgb = mask * (rng.uniform(size=(N, 1, H, H)) > 0.3)
    convex = rng.uniform(-1, 1, (N, 1, H, H))
    g_np = dict(replace_rgb=(0.1, y[:, :3], mask_rgb), replace_depth=(0.2, y[:, 3:], mask), constrain_depth=(0.5, convex))
    th = lambda a: torch.from_numpy(a)
    g_t = dict(replace_rgb=(0.1, th(y[:, :3]), th(mask_rgb)), replace_depth=(0.2, th(y[:, 3:]), th(mask)),
               constrain_depth=(0.5, th(convex)))
    for (t, tp) in [(1000, 980), (500, 480), (41, 21), (20, 0), (1000, 0)]:
        for guided in (False, True):
            got, d0 = dpm_ref.step(ACP, x_t, t, tp, eps, clip_denoised=clip, **(g_np if guided else {}))
            ref, x0 = sampler_ref.ddim_step(tb, th(x_t), torch.tensor([t] * N), torch.tensor([tp] * N), th(eps),
                                            torch.zeros(N, 4, H, H, dtype=torch.float64), clip_denoised=clip, eta=0.0,
                                            **(g_t if guided else {}))
            assert ref.dtype == torch.float64
            assert _rel(d0, x0.numpy()) < 1e-13, (t, tp, guided)
            assert _rel(got, ref.numpy()) < 1e-12, (t, tp, guided)
            if tp == 0:
                assert np.array_equal(got, d0), "the final step returns the guided x_0"


def _gaussian_problem(seed=0, D=64):
    """x_0 ~ N(mu, diag(s^2)): E[eps | x_t] is exact and the probability-flow ODE keeps (x - alpha mu) / sqrt(alpha^2 s^2 + sigma^2)
    constant, so x at any time has a closed form."""
    rng = np.random.default_rng(seed)
    mu, s = rng.uniform(-0.5, 0.5, D), rng.uniform(0.1, 1.0, D)

    def eps_fn(x, t_model):
        a, sg = np.sqrt(ACP[t_model]), np.sqrt(1 - ACP[t_model])
        return sg * (x - a * mu) / (a * a * s * s + sg * sg)

    def exact(x, t_from, t_to):
        a0, s0 = np.sqrt(ACP[t_from - 1]), np.sqrt(1 - ACP[t_from - 1])
        a1, s1 = np.sqrt(ACP[t_to - 1]), np.sqrt(1 - ACP[t_to - 1])
        return a1 * mu + np.sqrt(a1 * a1 * s * s + s1 * s1) / np.sqrt(a0 * a0 * s * s + s0 * s0) * (x - a0 * mu)

    return rng.standard_normal(D), eps_fn, exact


def test_convergence_order_on_gaussian_data():
    """Doubling the steps halves the error at order 1 and quarters it at order 2.  Measured at t = 200 (a point of every
    grid used), before the final step, whose x_0 output is not an ODE step."""
    x_T, eps_fn, exact = _gaussian_problem()
    want = exact(x_T, T, 200)
    err = {o: [_rel(dpm_ref.run(ACP, x_T, eps_fn, n, o, stop_at=200), want) for n in (50, 100, 200)] for o in (1, 2)}
    for o, lo, hi in ((1, 1.8, 2.2), (2, 3.3, 5.0)):
        ratios = [err[o][i] / err[o][i + 1] for i in range(2)]
        assert all(lo < r < hi for r in ratios), (o, err[o], ratios)
    assert all(e2 < e1 / 10 for e1, e2 in zip(err[1], err[2])), "second order is far more accurate at equal steps"


def test_order_pattern():
    """First step and the final step to t_prev = 0 are first order; every other step of a 2M run is second order and uses
    the previous step of the grid.  The grid is DdimSampler's."""
    for steps in (1, 2, 3, 10, 50, 1000):
        sch = dpm_ref.schedule(T, steps, 2)
        assert [(t, tp) for (t, tp, _, _) in sch] == sampler_ref.ddim_schedule(T, steps)
        orders = [o for (*_, o) in sch]
        assert orders == ([1] if steps == 1 else [1] + [2] * (steps - 2) + [1]), steps
        assert [tl for (_, _, tl, _) in sch] == [None] + [t for (t, *_) in sch[:-1]]
        assert all(o == 1 for (*_, o) in dpm_ref.schedule(T, steps, 1))
    # coefficients of the final step: x_p = D0 exactly
    assert dpm_ref.coefs(ACP, 20, 0, 40, 2) == (0.0, -1.0, 1.0, 0.0, 1)


def _tiny_fw():
    return frameworks.ClassifierFreeGuidance(backbones.AdmUnet2d(**TINY), timesteps=T, beta_schedule="linear")


def test_python_surface_and_errors():
    fw = _tiny_fw()
    dpm, ddim = samplers.DpmSolverSampler(fw), samplers.DdimSampler(fw)
    for name in ("alphas_cumprod", "alphas_cumprod_prev", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod"):
        assert np.array_equal(getattr(dpm, name), getattr(ddim, name)), name
    for bad in (0, 3, -1):
        with pytest.raises(AssertionError):
            dpm.sample(1, order=bad, verbose=False)
    from ivid_b200.inference import sample_all
    with pytest.raises(AssertionError):
        next(sample_all(fw, None, 1, 10, 10, [None], solver="euler"))


def test_native_error_contract():
    """The C entry points reject a bad DPM-Solver++ request with IVID_ERR_INVALID_ARGUMENT before any device work."""
    L = _lib.lib()
    unet = ctypes.c_void_p()
    _lib.check(L.ivid_unet_create(json.dumps(TINY).encode(), ctypes.byref(unet)))
    s = samplers.DpmSolverSampler(_tiny_fw())
    fake = ctypes.c_void_p(256)        # never dereferenced: every call below fails its argument checks first

    def step(t, tp, **fields):
        a = _lib.StepArgsT()
        a.kind = 2
        for k, v in fields.items():
            setattr(a, k, v)
        return L.ivid_sampler_step(s._handle, unet, fake, fake, None, 1, t, tp, ctypes.byref(a), None)

    try:
        cases = [
            (dict(kind=3), 500, 480, "sampler kind"),
            (dict(order=3), 500, 480, "order"),
            (dict(order=-1), 500, 480, "order"),
            (dict(), 500, 500, "t_prev < t"),
            (dict(), 1001, 980, "t out of range"),
            (dict(prev_x0_dev=256, t_last=500), 500, 480, "t_last > t"),
            (dict(prev_x0_dev=256, t_last=1001), 500, 480, "t_last out of range"),
            (dict(prev_x0_dev=256, t_last=0), 500, 480, "t_last out of range"),
        ]
        for fields, t, tp, msg in cases:
            rc = step(t, tp, **fields)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and msg in _lib.last_error(), (fields, t, tp, _lib.last_error())
        a = _lib.StepArgsT()
        a.kind, a.order = 2, 7
        rc = L.ivid_sampler_run(s._handle, unet, fake, 1, 10, ctypes.byref(a), None, None, None, None, None)
        assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "order" in _lib.last_error()
    finally:
        L.ivid_unet_destroy(unet)

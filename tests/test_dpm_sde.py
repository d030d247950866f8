"""CPU: the stochastic DPM-Solver++(2M) update (SDE variant, `sde=True`) against its float64 statement: order 1 equals DDIM
at eta = 1, the final step, its convergence on Gaussian data whose output moments are known exactly, the Python surface and
the host-side error contract of the `sde` flag."""
import ctypes
import inspect
import json

import numpy as np
import pytest
import torch

import dpm_sde_ref as R
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from oracle import sampler_ref

T = 1000
ACP = sampler_ref.Tables(sampler_ref.get_betas("linear", T)).alphas_cumprod
TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16], channel_mult=[1, 2], num_head_channels=64)


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b)))


@pytest.mark.parametrize("clip", [False, True])
def test_order1_is_ddim_eta1_with_guidance(monkeypatch, clip):
    """First order is DDIM with eta = 1, algebraically: the float64 SDE step against sampler_ref.ddim_step(eta=1) (its table
    lookup kept in float64) from the same x_t, eps and z, with and without the multiview replace / constrain guidance."""
    monkeypatch.setattr(sampler_ref, "_ex", lambda arr, t, nd: torch.from_numpy(arr)[t].view(-1, *([1] * (nd - 1))))
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", T))
    rng = np.random.default_rng(4)
    N, H = 2, 8
    x_t, eps, z = (rng.standard_normal((N, 4, H, H)) for _ in range(3))
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
            got, d0 = R.sde_step(ACP, x_t, t, tp, eps, z, clip_denoised=clip, **(g_np if guided else {}))
            ref, x0 = sampler_ref.ddim_step(tb, th(x_t), torch.tensor([t] * N), torch.tensor([tp] * N), th(eps), th(z),
                                            clip_denoised=clip, eta=1.0, **(g_t if guided else {}))
            assert ref.dtype == torch.float64
            assert _rel(d0, x0.numpy()) < 1e-13, (t, tp, guided)
            assert _rel(got, ref.numpy()) < 1e-12, (t, tp, guided)


def test_final_step_returns_d0_without_noise():
    assert R.sde_coefs(ACP, 20, 0, 40, 2) == (0.0, -1.0, 0.0, 1.0, 0.0, 1)
    rng = np.random.default_rng(5)
    x_t, eps, z, d_prev = (rng.standard_normal((1, 4, 4, 4)) for _ in range(4))
    got, d0 = R.sde_step(ACP, x_t, 20, 0, eps, z, d_prev=d_prev, t_last=40)
    assert np.array_equal(got, d0)
    # every other step draws noise, and the order-2 weights are the ODE solver's
    c = R.sde_coefs(ACP, 500, 480, 520, 2)
    assert c[2] > 0 and c[5] == 2


# var / s^2 - 1 of the output on x_0 ~ N(0.3, 0.25), linear schedule, T = 1000: SDE order 1 (= DDIM eta = 1), SDE 2M, ODE 2M
GAUSS_TABLE = {10: (-5.55e-1, -3.97e-1, -3.45e-1), 25: (-3.38e-1, 9.82e-3, -4.35e-2), 50: (-2.11e-1, 6.08e-2, 2.17e-3),
               100: (-1.23e-1, 3.17e-2, 3.14e-3), 250: (-5.60e-2, 7.61e-3, 4.44e-4), 500: (-2.97e-2, 2.22e-3, -8.94e-5)}


def test_gaussian_convergence():
    """Exact output moments on Gaussian data.  The mean is exact for every solver; the variance error of SDE 2M is below
    that of order 1 at every step count and falls with order >= 1.5 between 250 and 500 steps (order 1: >= 0.8).  SDE 2M's
    error changes sign near 25 steps, so it is not monotone and no monotonicity is asserted."""
    err = {}
    for n, row in GAUSS_TABLE.items():
        got = []
        for (order, sde) in ((1, True), (2, True), (2, False)):
            dm, dv = R.gaussian_moments(ACP, n, order, sde, 0.3, 0.25)
            assert abs(dm) < 1e-14, (n, order, sde, dm)
            got.append(dv)
        for g, want in zip(got, row):
            assert g == pytest.approx(want, rel=6e-3), (n, got, row)
        err[n] = got
        assert abs(got[1]) < abs(got[0]), (n, got)
    p2 = np.log2(abs(err[250][1]) / abs(err[500][1]))
    p1 = np.log2(abs(err[250][0]) / abs(err[500][0]))
    assert p2 >= 1.5 and p1 >= 0.8, (p1, p2)


def test_sde_run_order1_matches_step_chain():
    """sde_run is the chained update: one 5-step first-order run against five explicit DDIM eta = 1 style steps."""
    rng = np.random.default_rng(6)
    x_T = rng.standard_normal(16)
    zs = rng.standard_normal((5, 16))
    eps_fn = lambda x, tm: 0.3 * x
    x = x_T.copy()
    for i, (t, tp) in enumerate(sampler_ref.ddim_schedule(T, 5)):
        x, _ = R.sde_step(ACP, x, t, tp, eps_fn(x, t - 1), zs[i])
    assert np.array_equal(R.sde_run(ACP, x_T, eps_fn, lambda i: zs[i], 5, order=1), x)


def _tiny_fw():
    return frameworks.ClassifierFreeGuidance(backbones.AdmUnet2d(**TINY), timesteps=T, beta_schedule="linear")


class _Stop(Exception):
    pass


def test_python_surface(monkeypatch):
    for fn in (samplers.DpmSolverSampler.sample, samplers.DpmSolverSampler.sample_once):
        p = inspect.signature(fn).parameters["sde"]
        assert p.default is False
    from ivid_b200.inference import sample_all
    calls = []

    def fake_sample(self, *a, **kw):
        calls.append((type(self).__name__, kw.get("sde")))
        raise _Stop

    monkeypatch.setattr(samplers.DpmSolverSampler, "sample", fake_sample)
    monkeypatch.setattr(samplers.DdpmSampler, "sample", fake_sample)
    fw = _tiny_fw()
    for steps_uncond, want in ((10, ("DpmSolverSampler", True)), (1000, ("DdpmSampler", None))):
        with pytest.raises(_Stop):
            next(sample_all(fw, None, 1, steps_uncond, 10, [None], solver="dpmpp_sde"))
        assert calls[-1] == want, calls
    with pytest.raises(AssertionError):
        next(sample_all(fw, None, 1, 10, 10, [None], solver="dpmpp_ode"))


def test_native_error_contract():
    """`sde` other than 0 / 1, or sde = 1 with kind 0 or 1, is IVID_ERR_INVALID_ARGUMENT before any device work."""
    L = _lib.lib()
    unet = ctypes.c_void_p()
    _lib.check(L.ivid_unet_create(json.dumps(TINY).encode(), ctypes.byref(unet)))
    s = samplers.DpmSolverSampler(_tiny_fw())
    fake = ctypes.c_void_p(256)        # never dereferenced: every call below fails its argument checks first

    def args(kind, sde):
        a = _lib.StepArgsT()
        a.kind, a.sde = kind, sde
        return a

    try:
        for kind, sde in ((2, 2), (2, -1), (0, 1), (1, 1)):
            a = args(kind, sde)
            t, tp = (500, 0) if kind == 0 else (500, 480)
            rc = L.ivid_sampler_step(s._handle, unet, fake, fake, None, 1, t, tp, ctypes.byref(a), None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "sde" in _lib.last_error(), (kind, sde, _lib.last_error())
            rc = L.ivid_sampler_run(s._handle, unet, fake, 1, 10, ctypes.byref(a), None, None, None, None, None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "sde" in _lib.last_error(), (kind, sde, _lib.last_error())
    finally:
        L.ivid_unet_destroy(unet)

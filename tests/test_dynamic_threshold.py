"""CPU: dynamic thresholding of x_0 (`dynamic_threshold=p` or `(p, s_max)`): the float64 oracle against numpy / torch and against
the clipped steps of oracle/, and the host side of the option: argument checks on every surface (which run before any device
work or torch draw), the Python signatures, sample_all, the CLI flag and the output directory name."""
import ctypes
import inspect
import json
import math

import numpy as np
import pytest
import torch

import dynamic_threshold_ref as R
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from ivid_b200.inference import sample as sample_cli
from oracle import dpm_ref, sampler_ref

T = 1000
TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16], channel_mult=[1, 2], num_head_channels=64)
BAD = [0.0, -0.5, 1.5, float("nan"), (0.5, 0.5), (0.5, 0.0), (0.9, float("nan")), (0.5, 2.0, 3.0), True, "0.5"]


def _tiny_fw():
    return frameworks.ClassifierFreeGuidance(backbones.AdmUnet2d(**TINY), timesteps=T, beta_schedule="linear")


def test_quantile_equals_numpy_on_float64():
    """numpy's linear method interpolates as v_{k+1} - (1 - f)(v_{k+1} - v_k) when f >= 0.5: the same value, up to its last bit
    there; below f = 0.5 the formulas are the same and the results are equal."""
    rng = np.random.default_rng(0)
    for _ in range(200):
        M = int(rng.integers(1, 3000))
        a = np.abs(rng.standard_normal(M) * rng.uniform(0.1, 10.0))
        a[rng.integers(0, M, M // 4)] = a[0]                       # ties
        for p in (1e-6, 0.1, 0.3, 0.5, 0.75, 0.995, 1.0, float(rng.uniform(0.0, 1.0))):
            ours, ref = R.quantile(a, p), np.quantile(a, p, method="linear")
            f = p * (M - 1) - math.floor(p * (M - 1))
            if f < 0.5:
                assert ours == ref, (M, p)
            else:
                assert abs(ours - ref) <= np.spacing(ref), (M, p)


def test_quantile_within_one_ulp_of_torch_on_float32():
    """torch.quantile forms the position p (M - 1) in the data's precision; at ratios exact in fp32 it agrees to 1 ulp."""
    rng = np.random.default_rng(1)
    for _ in range(200):
        M = int(rng.integers(1, 3000))
        a = np.abs(rng.standard_normal(M) * rng.uniform(0.1, 10.0)).astype(np.float32)
        for p in (0.25, 0.5, 0.75, 1.0):
            ours = R.quantile(a, p)
            ref = torch.quantile(torch.from_numpy(a), p).numpy()
            assert ours.dtype == np.float32
            assert abs(int(ours.view(np.int32)) - int(ref.view(np.int32))) <= 1, (M, p)


def test_threshold_definition():
    x = np.array([[0.5, -0.25, 0.1, 0.0], [3.0, -4.0, 1.0, 2.0]], dtype=np.float32)
    s, y = R.threshold(x, 1.0)
    assert s.tolist() == [1.0, 4.0]                               # max |x|, at least 1
    assert np.array_equal(y[0], x[0]) and np.array_equal(y[1], x[1] / np.float32(4.0))
    s, y = R.threshold(x, 1.0, 2.0)
    assert s.tolist() == [1.0, 2.0] and np.array_equal(y[1], np.clip(x[1], -2, 2) / np.float32(2.0))


def test_smax_one_reproduces_clipped_reference_steps():
    """s_max = 1 forces s = 1: the oracle's steps equal sampler_ref's clipped DDPM / DDIM steps and dpm_ref's clipped D0 bit for
    bit (fp32 torch for DDPM / DDIM as sampler_ref computes them, float64 numpy for D0)."""
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", T))
    g = torch.Generator().manual_seed(0)
    x_t = torch.randn(2, 4, 8, 8, generator=g) * 3
    eps = torch.randn(2, 4, 8, 8, generator=g) * 3
    z = torch.randn(2, 4, 8, 8, generator=g)
    y = torch.rand(2, 4, 8, 8, generator=g) * 2 - 1
    m = (torch.rand(2, 1, 8, 8, generator=g) > 0.5).float()
    guide = dict(replace_rgb=(0.1, y[:, :3], m), replace_depth=(0.2, y[:, 3:], m), constrain_depth=(0.5, y[:, 3:] * 0.5))
    for ti in (999, 500, 0):
        t = torch.tensor([ti, ti])
        a, a0 = sampler_ref.ddpm_step(tb, x_t, t, eps, z, clip_denoised=True)
        b, b0 = R.ddpm_step(tb, x_t, t, eps, z, 0.9, 1.0)
        assert torch.equal(a, b) and torch.equal(a0, b0)
    for (tt, tp) in ((1000, 900), (500, 480), (20, 0)):
        t, tpv = torch.tensor([tt, tt]), torch.tensor([tp, tp])
        for eta in (0.0, 1.0):
            for gk in ({}, guide):
                a, a0 = sampler_ref.ddim_step(tb, x_t, t, tpv, eps, z, clip_denoised=True, eta=eta, **gk)
                b, b0 = R.ddim_step(tb, x_t, t, tpv, eps, z, 0.995, 1.0, eta=eta, **gk)
                assert torch.equal(a, b) and torch.equal(a0, b0), (tt, eta, bool(gk))
        gn = {k: tuple(v.double().numpy() if torch.is_tensor(v) else v for v in val) for k, val in guide.items()}
        xd, ed = x_t.double().numpy(), eps.double().numpy()
        for gk in ({}, gn):
            a = dpm_ref.guided_x0(tb.alphas_cumprod, xd, tt, tp, ed, clip_denoised=True, **gk)
            b = R.dpm_d0(tb.alphas_cumprod, xd, tt, tp, ed, 0.5, 1.0, **gk)
            assert np.array_equal(a, b), (tt, bool(gk))


def test_native_rejects_bad_arguments():
    """A flag other than 0 / 1, a ratio outside (0, 1], threshold_max in (0, 1) or NaN, or the flag with clip_denoised is
    IVID_ERR_INVALID_ARGUMENT on every sampler entry point before any device work (the pointers are never dereferenced); so is
    the op entry's ratio / bound."""
    L = _lib.lib()
    unet = ctypes.c_void_p()
    _lib.check(L.ivid_unet_create(json.dumps(TINY).encode(), ctypes.byref(unet)))
    s = samplers.DdimSampler(_tiny_fw())
    fake = ctypes.c_void_p(256)
    cases = [(2, 0.5, 0.0, 0), (-1, 0.5, 0.0, 0), (1, 0.0, 0.0, 0), (1, 1.5, 0.0, 0), (1, float("nan"), 0.0, 0),
             (1, 0.5, 0.5, 0), (1, 0.5, float("nan"), 0), (1, 0.5, 0.0, 1)]
    try:
        for kind in (0, 1, 2):
            for flag, ratio, mx, clip in cases:
                a = _lib.StepArgsT()
                a.kind, a.dynamic_threshold, a.threshold_ratio, a.threshold_max, a.clip_denoised = kind, flag, ratio, mx, clip
                t, tp = (500, 0) if kind == 0 else (500, 480)
                rc = L.ivid_sampler_step(s._handle, unet, fake, fake, None, 1, t, tp, ctypes.byref(a), None)
                assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "threshold" in _lib.last_error(), (kind, flag, ratio, mx, clip)
                tdev = ctypes.c_void_p(512)
                rc = L.ivid_sampler_step_dev(s._handle, unet, fake, fake, None, 1, tdev, tdev, ctypes.byref(a), None)
                assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "threshold" in _lib.last_error()
                rc = L.ivid_sampler_run(s._handle, unet, fake, 1, 10, ctypes.byref(a), None, None, None, None, None)
                assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "threshold" in _lib.last_error()
        for ratio, mx in ((0.0, 0.0), (1.5, 0.0), (0.5, 0.5)):
            rc = L.ivid_op_dynamic_threshold(fake, 1, 16, ratio, mx, fake, fake, None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "threshold" in _lib.last_error()
    finally:
        L.ivid_unet_destroy(unet)


def test_zeroed_struct_means_off():
    a = _lib.StepArgsT()
    assert (a.dynamic_threshold, a.threshold_ratio, a.threshold_max) == (0, 0.0, 0.0)
    assert [f[0] for f in _lib.StepArgsT._fields_][-3:] == ["dynamic_threshold", "threshold_ratio", "threshold_max"]


@pytest.mark.parametrize("bad", BAD)
def test_python_rejects_bad_thresholds(bad):
    """AssertionError from every sample / sample_once before the network is touched and before any torch draw."""
    fw = _tiny_fw()
    x = torch.zeros(1, 4, 32, 32)
    t = torch.tensor([500])
    for cls in (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler):
        s = cls(fw)
        with pytest.raises(AssertionError, match="dynamic_threshold"):
            s.sample(1, noise=x, steps=10, verbose=False, dynamic_threshold=bad)
        state = torch.get_rng_state()
        with pytest.raises(AssertionError, match="dynamic_threshold"):
            if cls is samplers.DdpmSampler:
                s.sample_once(x, t, dynamic_threshold=bad)
            else:
                s.sample_once(x, t, t - 20, dynamic_threshold=bad)
        assert torch.equal(state, torch.get_rng_state())


def test_python_rejects_clip_with_threshold():
    fw = _tiny_fw()
    x = torch.zeros(1, 4, 32, 32)
    t = torch.tensor([500])
    for cls in (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler):
        s = cls(fw)
        with pytest.raises(AssertionError, match="clip_denoised"):
            s.sample(1, noise=x, steps=10, verbose=False, clip_denoised=True, dynamic_threshold=0.995)
        state = torch.get_rng_state()
        with pytest.raises(AssertionError, match="clip_denoised"):
            if cls is samplers.DdpmSampler:
                s.sample_once(x, t, clip_denoised=True, dynamic_threshold=0.995)
            else:
                s.sample_once(x, t, t - 20, clip_denoised=True, dynamic_threshold=(0.995, 2.0))
        assert torch.equal(state, torch.get_rng_state())


def test_python_surface():
    for cls in (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler):
        for fn in (cls.sample, cls.sample_once):
            assert inspect.signature(fn).parameters["dynamic_threshold"].default is None
    assert inspect.signature(sample_cli.sample_all).parameters["dynamic_threshold"].default is None


class _Stop(Exception):
    pass


def test_sample_all_passes_the_threshold(monkeypatch):
    calls = []

    def fake_sample(self, *a, **kw):
        calls.append((type(self).__name__, kw.get("dynamic_threshold")))
        raise _Stop

    for cls in (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler):
        monkeypatch.setattr(cls, "sample", fake_sample)
    fw = _tiny_fw()
    for steps_uncond, solver, name in ((1000, "ddim", "DdpmSampler"), (10, "ddim", "DdimSampler"), (10, "dpmpp", "DpmSolverSampler")):
        for dt in (None, 0.995, (0.9, 2.0)):
            with pytest.raises(_Stop):
                next(sample_cli.sample_all(fw, None, 1, steps_uncond, 10, [None], solver=solver, dynamic_threshold=dt))
            assert calls[-1] == (name, dt), calls
    for bad in BAD:
        with pytest.raises(AssertionError, match="dynamic_threshold"):
            next(sample_cli.sample_all(fw, None, 1, 10, 10, [None], dynamic_threshold=bad))


def test_cli_parses_dynamic_threshold():
    ap = sample_cli.build_arg_parser()
    assert ap.parse_args([]).dynamic_threshold is None
    assert ap.parse_args(["--dynamic_threshold", "0.995"]).dynamic_threshold == 0.995
    assert ap.parse_args(["--dynamic_threshold", "0.9,2"]).dynamic_threshold == (0.9, 2.0)
    assert ap.parse_args(["--dynamic_threshold", "1"]).dynamic_threshold == 1.0
    for bad in ("0", "1.5", "-0.1", "a", "0.9,0.5", "0.9,2,3", "nan", "0.9,nan"):
        with pytest.raises(SystemExit):
            ap.parse_args(["--dynamic_threshold", bad])


def test_output_dir_name():
    ap = sample_cli.build_arg_parser()
    base = sample_cli.output_dir_name(ap.parse_args([]))
    assert base.endswith("viewset_3x9_steps_u1000_c50_guidance3.0"), "unchanged without the flag"
    assert sample_cli.output_dir_name(ap.parse_args(["--dynamic_threshold", "0.995"])) == base + "_dthresh0.995"
    assert sample_cli.output_dir_name(ap.parse_args(["--dynamic_threshold", "0.9,2"])) == base + "_dthresh0.9-2.0"

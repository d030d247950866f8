"""CPU: the host side of the guidance interval (`guidance_interval=(t_lo, t_hi)`): the argument checks of the C ABI and of
the Python samplers, which run before any device work, the Python surface, sample_all and the CLI flag."""
import ctypes
import inspect
import json

import pytest
import torch

import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from ivid_b200.inference import sample as sample_cli

T = 1000
TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16], channel_mult=[1, 2], num_head_channels=64)
BAD = [(5, 3), (-1, 10), (0, T), (700, 1200)]


def _tiny_fw():
    return frameworks.ClassifierFreeGuidance(backbones.AdmUnet2d(**TINY), timesteps=T, beta_schedule="linear")


def test_native_rejects_bad_intervals():
    """guidance_interval other than 0 / 1, or bounds outside 0 <= t_lo <= t_hi < T, is IVID_ERR_INVALID_ARGUMENT before any
    device work (the pointers below are never dereferenced)."""
    L = _lib.lib()
    unet = ctypes.c_void_p()
    _lib.check(L.ivid_unet_create(json.dumps(TINY).encode(), ctypes.byref(unet)))
    s = samplers.DdimSampler(_tiny_fw())
    fake = ctypes.c_void_p(256)
    cases = [(1, lo, hi) for lo, hi in BAD] + [(2, 0, 10), (-1, 0, 10)]
    try:
        for kind in (0, 1, 2):
            for flag, lo, hi in cases:
                a = _lib.StepArgsT()
                a.kind, a.guidance_interval, a.guidance_t_lo, a.guidance_t_hi = kind, flag, lo, hi
                t, tp = (500, 0) if kind == 0 else (500, 480)
                rc = L.ivid_sampler_step(s._handle, unet, fake, fake, None, 1, t, tp, ctypes.byref(a), None)
                assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "guidance" in _lib.last_error(), (kind, flag, lo, hi)
                tdev = ctypes.c_void_p(512)
                rc = L.ivid_sampler_step_dev(s._handle, unet, fake, fake, None, 1, tdev, tdev, ctypes.byref(a), None)
                assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "guidance" in _lib.last_error(), (kind, flag, lo, hi)
                rc = L.ivid_sampler_run(s._handle, unet, fake, 1, 10, ctypes.byref(a), None, None, None, None, None)
                assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "guidance" in _lib.last_error(), (kind, flag, lo, hi)
    finally:
        L.ivid_unet_destroy(unet)


@pytest.mark.parametrize("interval", BAD + [(1, 2, 3)])
def test_python_rejects_bad_intervals(interval):
    """AssertionError from every sample / sample_once, before the network is touched and before any torch draw."""
    fw = _tiny_fw()
    x = torch.zeros(1, 4, 32, 32)
    t = torch.tensor([500])
    for cls in (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler):
        s = cls(fw)
        with pytest.raises(AssertionError, match="guidance_interval"):
            s.sample(1, noise=x, steps=10, verbose=False, guidance_interval=interval)
        state = torch.get_rng_state()
        with pytest.raises(AssertionError, match="guidance_interval"):
            if cls is samplers.DdpmSampler:
                s.sample_once(x, t, guidance_interval=interval)
            else:
                s.sample_once(x, t, t - 20, guidance_interval=interval)
        assert torch.equal(state, torch.get_rng_state())


def test_python_surface():
    for cls in (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler):
        for fn in (cls.sample, cls.sample_once):
            assert inspect.signature(fn).parameters["guidance_interval"].default is None
    assert inspect.signature(sample_cli.sample_all).parameters["guidance_interval"].default is None
    assert _lib.StepArgsT().guidance_interval == 0, "a zeroed ivid_step_args_t means no interval"


class _Stop(Exception):
    pass


def test_sample_all_passes_the_interval(monkeypatch):
    calls = []

    def fake_sample(self, *a, **kw):
        calls.append((type(self).__name__, kw.get("guidance_interval")))
        raise _Stop

    for cls in (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler):
        monkeypatch.setattr(cls, "sample", fake_sample)
    fw = _tiny_fw()
    for steps_uncond, solver, name in ((1000, "ddim", "DdpmSampler"), (10, "ddim", "DdimSampler"), (10, "dpmpp", "DpmSolverSampler")):
        for gi in (None, (100, 600)):
            with pytest.raises(_Stop):
                next(sample_cli.sample_all(fw, None, 1, steps_uncond, 10, [None], solver=solver, guidance_interval=gi))
            assert calls[-1] == (name, gi), calls


def test_cli_parses_guidance_interval():
    ap = sample_cli.build_arg_parser()
    assert ap.parse_args([]).guidance_interval is None
    assert ap.parse_args(["--guidance_interval", "100,600"]).guidance_interval == (100, 600)
    assert ap.parse_args(["--guidance_interval", "0,0"]).guidance_interval == (0, 0)
    for bad in ("600", "1,2,3", "a,b", "600,100", "-1,5"):
        with pytest.raises(SystemExit):
            ap.parse_args(["--guidance_interval", bad])

"""CPU: the host side of feature reuse between denoising steps (DeepCache): the argument checks of the Python samplers,
sample_all and the CLI, which run before any device work, the flags' way to sample_all and the output directory, the C ABI
symbol, and the oracle's reuse forward against its full forward."""
import argparse
import inspect

import numpy as np
import pytest
import torch

import deepcache_ref
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from ivid_b200.inference import sample as sample_cli
from oracle import unet_ref

T = 1000
TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16], channel_mult=[1, 2], num_head_channels=64)
SAMPLERS = (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler)


def _tiny_fw():
    return frameworks.ClassifierFreeGuidance(backbones.AdmUnet2d(**TINY), timesteps=T, beta_schedule="linear")


@pytest.mark.parametrize("args", [dict(cache_interval=0), dict(cache_interval=-2), dict(cache_interval=2.5),
                                  dict(cache_interval=2, cache_branch=2), dict(cache_interval=2, cache_branch=-1),
                                  dict(cache_branch=5)])
def test_sample_rejects_bad_cache_args(args):
    """AssertionError from every sample(), before the network is packed (there is no GPU here) and before any torch draw."""
    fw = _tiny_fw()
    x = torch.zeros(1, 4, 32, 32)
    for cls in SAMPLERS:
        state = torch.get_rng_state()
        with pytest.raises(AssertionError, match="cache_"):
            cls(fw).sample(1, noise=x, steps=10, verbose=False, **args)
        assert torch.equal(state, torch.get_rng_state())


@pytest.mark.parametrize("branch", [-1, 2, 7, 1.0])
def test_sample_once_rejects_bad_branch(branch):
    fw = _tiny_fw()
    x = torch.zeros(1, 4, 32, 32)
    t = torch.tensor([500])
    for cls in SAMPLERS:
        s = cls(fw)
        state = torch.get_rng_state()
        with pytest.raises(AssertionError, match="cache_branch"):
            if cls is samplers.DdpmSampler:
                s.sample_once(x, t, reuse_features=True, cache_branch=branch)
            else:
                s.sample_once(x, t, t - 20, reuse_features=True, cache_branch=branch)
        assert torch.equal(state, torch.get_rng_state())


def test_python_surface():
    for cls in SAMPLERS:
        p = inspect.signature(cls.sample).parameters
        assert p["cache_interval"].default is None and p["cache_branch"].default == 0
        p = inspect.signature(cls.sample_once).parameters
        assert p["reuse_features"].default is False and p["cache_branch"].default == 0
    p = inspect.signature(sample_cli.sample_all).parameters
    assert p["cache_interval"].default is None and p["cache_branch"].default == 0
    a = _lib.StepArgsT()
    assert (a.cache_interval, a.cache_branch, a.cache_reuse) == (0, 0, 0), "a zeroed ivid_step_args_t means no reuse"


def test_abi_symbol_exported():
    L = _lib.lib()
    assert hasattr(L, "ivid_unet_forward_reuse")
    assert "ivid_unet_forward_reuse" in _lib.SIGNATURES


def test_reuse_schedule_rule():
    """The host copy of ivid_sampler_run's rule: full at step 0, every cache_interval steps after the last full one, and at
    every switch between the guided and the unguided forward."""
    s = samplers.DdimSampler(_tiny_fw())
    cls = torch.tensor([1])
    times = list(range(999, -1, -100))                                      # 10 steps
    assert s._reuse_schedule(times, cls, dict(strength=0.5), None, 1) == [False] * 10
    assert s._reuse_schedule(times, cls, dict(strength=0.5), None, 3) == [False, True, True] * 3 + [False]
    # guided at 699..399 (steps 3 to 6): the switches at steps 3 and 7 are full, and the count restarts there
    got = s._reuse_schedule(times, cls, dict(strength=0.5), (300, 700), 3)
    assert got == [False, True, True, False, True, True, False, False, True, True]
    # no classes: one plan throughout, the interval changes nothing
    assert s._reuse_schedule(times, None, dict(strength=0.5), (300, 700), 3) == [False, True, True] * 3 + [False]


def test_native_rejects_bad_cache_args():
    """Negative cache_interval, a branch outside [0, num_res_blocks] or cache_reuse other than 0 / 1 is
    IVID_ERR_INVALID_ARGUMENT before any device work (the pointers are never dereferenced)."""
    import ctypes
    import json
    L = _lib.lib()
    unet = ctypes.c_void_p()
    _lib.check(L.ivid_unet_create(json.dumps(TINY).encode(), ctypes.byref(unet)))
    s = samplers.DdimSampler(_tiny_fw())
    fake = ctypes.c_void_p(256)
    try:
        for ci, cb, cr in ((-1, 0, 0), (0, 2, 0), (0, -1, 0), (0, 0, 2), (0, 0, -1)):
            a = _lib.StepArgsT()
            a.kind, a.cache_interval, a.cache_branch, a.cache_reuse = 1, ci, cb, cr
            rc = L.ivid_sampler_step(s._handle, unet, fake, fake, None, 1, 500, 480, ctypes.byref(a), None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "cache_" in _lib.last_error(), (ci, cb, cr)
            rc = L.ivid_sampler_run(s._handle, unet, fake, 1, 10, ctypes.byref(a), None, None, None, None, None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "cache_" in _lib.last_error(), (ci, cb, cr)
        rc = L.ivid_unet_forward_reuse(unet, fake, 1, 32, 32, None, fake, None, fake, 1, -1, None)
        assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "cache_branch" in _lib.last_error()
    finally:
        L.ivid_unet_destroy(unet)


class _Stop(Exception):
    pass


def test_sample_all_passes_cache_args(monkeypatch):
    calls = []

    def fake_sample(self, *a, **kw):
        calls.append((type(self).__name__, kw.get("cache_interval"), kw.get("cache_branch")))
        raise _Stop

    for cls in SAMPLERS:
        monkeypatch.setattr(cls, "sample", fake_sample)
    fw = _tiny_fw()
    for steps_uncond, solver, name in ((1000, "ddim", "DdpmSampler"), (10, "ddim", "DdimSampler"), (10, "dpmpp", "DpmSolverSampler")):
        with pytest.raises(_Stop):
            next(sample_cli.sample_all(fw, None, 1, steps_uncond, 10, [None], solver=solver))
        assert calls[-1] == (name, None, None), calls
        with pytest.raises(_Stop):
            next(sample_cli.sample_all(fw, None, 1, steps_uncond, 10, [None], solver=solver, cache_interval=3, cache_branch=1))
        assert calls[-1] == (name, 3, 1), calls
    n = len(calls)
    for bad in (dict(cache_interval=0), dict(cache_interval=2, cache_branch=2)):
        with pytest.raises(AssertionError, match="cache_"):
            next(sample_cli.sample_all(fw, None, 1, 1000, 10, [None], **bad))
    assert len(calls) == n, "checked before any sampler runs"


def test_cli_flags_and_output_dir():
    ap = sample_cli.build_arg_parser()
    o = ap.parse_args([])
    assert o.cache_interval is None and o.cache_branch == 0
    assert "_cache" not in sample_cli.output_dir_name(o)
    o = ap.parse_args(["--cache_interval", "3", "--cache_branch", "1"])
    assert (o.cache_interval, o.cache_branch) == (3, 1)
    assert sample_cli.output_dir_name(o).endswith("_guidance3.0_cache3b1")
    o = ap.parse_args(["--cache_interval", "2", "--solver", "dpmpp", "--guidance_interval", "100,600"])
    assert sample_cli.output_dir_name(o).endswith("_dpmpp_interval100-600_cache2b0")
    for bad in (["--cache_interval", "0"], ["--cache_interval", "x"], ["--cache_branch", "-1"]):
        with pytest.raises(SystemExit):
            ap.parse_args(bad)
    assert sample_cli.output_dir_name(argparse.Namespace(output_dir="o", viewset="3x9", steps_uncond=1000, steps_cond=50,
                                                         guidance=3.0)) == "o/viewset_3x9_steps_u1000_c50_guidance3.0"


ORACLE_CFGS = {
    "tiny": dict(TINY, num_classes=10, has_null_class=True),
    "top_attention": dict(TINY, attention_resolutions=[32, 16], num_res_blocks=2),
    "no_updown": dict(TINY, resblock_updown=False, num_res_blocks=2),
    "one_level": dict(TINY, channel_mult=[1], num_res_blocks=2),
}


@pytest.mark.parametrize("tag", list(ORACLE_CFGS))
def test_oracle_reuse_equals_full(tag):
    """The oracle's reuse forward, given the tensor its full forward captured from the same x, t and classes, computes the full
    forward exactly, at every branch; a different cached tensor changes it."""
    cfg = ORACLE_CFGS[tag]
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=7)
    g = np.random.default_rng(3)
    x = torch.from_numpy(g.standard_normal((2, 4, 32, 32)).astype(np.float32))
    t = torch.tensor([400, 401])
    classes = torch.tensor([1, -1]) if cfg.get("num_classes") else None
    full = unet_ref.unet_forward(cfg, sd, x, t, classes)
    assert torch.equal(deepcache_ref.unet_forward(cfg, sd, x, t, classes), full)
    for b in range(cfg["num_res_blocks"] + 1):
        name = deepcache_ref.cached_block_name(cfg, b)
        eps, h = deepcache_ref.unet_forward(cfg, sd, x, t, classes, capture=name)
        assert torch.equal(eps, full)
        assert torch.equal(deepcache_ref.unet_forward(cfg, sd, x, t, classes, reuse=(b, h)), full), (tag, b)
        assert not torch.equal(deepcache_ref.unet_forward(cfg, sd, x, t, classes, reuse=(b, h * 1.01)), full)

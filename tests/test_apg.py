"""CPU: adaptive projected guidance (APG) - the float64 model's properties, argument checks in Python and at the native ABI,
and the plumbing through sample_all and the CLI.  Every error is raised before any device work and before any torch draw."""
import ctypes
import inspect
import json
import math

import numpy as np
import pytest
import torch

import apg_ref
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from ivid_b200.inference import sample as sample_cli
from ivid_b200.utils import edict

T = 1000
TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16], channel_mult=[1, 2], num_head_channels=64, num_classes=10, has_null_class=True)
TINY_COND = dict(TINY, in_channels=9)
SAMPLERS = (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler, samplers.UniPcSampler)


def _fw(cls=frameworks.ClassifierFreeGuidance, cfg=TINY):
    return cls(backbones.AdmUnet2d(**cfg), timesteps=T, beta_schedule="linear")


def _pair(seed, n=3, shape=(4, 8, 8)):
    rng = np.random.default_rng(seed)
    dc = rng.standard_normal((n,) + shape)
    du = dc + 0.3 * rng.standard_normal((n,) + shape)
    return dc, du


# ---------------------------------------------------------------------------------------------------------------------
# the float64 model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [0.5, 3.0])
def test_model_is_cfg_at_eta1_r0_beta0(s):
    dc, du = _pair(0)
    d, m = apg_ref.apg64(dc, du, s, eta=1.0)
    assert np.allclose(d, (1 + s) * dc - s * du, rtol=0, atol=1e-12)
    assert np.array_equal(m, dc - du)


def test_model_eta0_is_orthogonal_to_dc():
    dc, du = _pair(1)
    d, _ = apg_ref.apg64(dc, du, 3.0, eta=0.0)
    for n in range(dc.shape[0]):
        upd, base = (d - dc)[n].ravel(), dc[n].ravel()
        assert abs(upd @ base) <= 1e-12 * np.linalg.norm(upd) * np.linalg.norm(base)


@pytest.mark.parametrize("r", [0.05, 1.0, 1e3])
def test_model_norm_bound(r):
    dc, du = _pair(2)
    s = 3.0
    d, m = apg_ref.apg64(dc, du, s, eta=1.0, r=r)
    for n in range(dc.shape[0]):
        assert np.linalg.norm((d - dc)[n]) <= s * r * (1 + 1e-12)
        if np.linalg.norm(m[n]) <= r:         # inside the bound the update is the plain one
            assert np.allclose(d[n], dc[n] + s * m[n], rtol=0, atol=1e-12)


def test_model_momentum_over_three_steps():
    rng = np.random.default_rng(3)
    dcs = [rng.standard_normal((2, 4, 4, 4)) for _ in range(3)]
    dus = [x + 0.2 * rng.standard_normal(x.shape) for x in dcs]
    beta, s, eta = -0.5, 2.0, 0.25
    ds, m3 = apg_ref.chain64(dcs, dus, s, eta=eta, beta=beta)
    deltas = [c - u for c, u in zip(dcs, dus)]
    assert np.allclose(m3, deltas[2] + beta * deltas[1] + beta ** 2 * deltas[0], rtol=0, atol=1e-12)
    # each step is the one-step model from the previous step's m
    m = None
    for i in range(3):
        d, m = apg_ref.apg64(dcs[i], dus[i], s, eta=eta, beta=beta, m_prev=m)
        assert np.array_equal(d, ds[i])


def test_model_degenerate_samples():
    """m = 0 (D_c == D_u) gives D = D_c with c = 1; D_c = 0 gives k = 0 (no division by zero)."""
    dc, du = _pair(4)
    du[0] = dc[0]
    dc[1] = 0.0
    d, _ = apg_ref.apg64(dc, du, 3.0, eta=0.0, r=0.5)
    c, k = apg_ref.scalars(dc, dc - du, 3.0, 0.0, 0.5)
    assert np.array_equal(d[0], dc[0]) and c[0] == 1.0
    assert k[1] == 0.0 and np.all(np.isfinite(d))


# ---------------------------------------------------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------------------------------------------------
def test_defaults_are_none():
    for cls in SAMPLERS:
        for fn in (cls.sample, cls.sample_once):
            assert inspect.signature(fn).parameters["apg"].default is None, (cls, fn)
        assert inspect.signature(cls.sample_once).parameters["apg_state"].default is None, cls
    assert inspect.signature(sample_cli.sample_all).parameters["apg"].default is None
    a = _lib.StepArgsT()
    assert (a.apg, a.apg_eta, a.apg_norm, a.apg_momentum) == (0, 0.0, 0.0, 0.0) and not a.apg_state_dev
    assert samplers.samplers._check_apg(0.5, _fw(), [1], 3.0) == (0.5, 0.0, 0.0)
    assert samplers.samplers._check_apg((0, 2), _fw(), [1], 3.0) == (0.0, 2.0, 0.0)
    assert samplers.samplers._check_apg([0.0, 0.0, -0.5], _fw(), [1], 3.0) == (0.0, 0.0, -0.5)


BAD = [
    (dict(apg=-0.1), "eta must be finite"),
    (dict(apg=float("nan")), "eta must be finite"),
    (dict(apg=float("inf")), "eta must be finite"),
    (dict(apg=True), "eta must be finite"),
    (dict(apg=(0.0, -1.0)), "norm bound r must be finite"),
    (dict(apg=(0.0, float("inf"))), "norm bound r must be finite"),
    (dict(apg=(0.0, 0.0, 1.0)), "momentum beta must lie in"),
    (dict(apg=(0.0, 0.0, -1.0)), "momentum beta must lie in"),
    (dict(apg=(0.0, 0.0, float("nan"))), "momentum beta must lie in"),
    (dict(apg=(0.0, 0.0, 0.0, 0.0)), "apg must be eta"),
    (dict(apg=()), "apg must be eta"),
    (dict(apg=0.0, strength=0.0), "strength > 0"),
    (dict(apg=0.0, strength=-0.5), "strength > 0"),
    (dict(apg=0.0, strength=float("inf")), "strength > 0"),
    (dict(apg=0.0, classes=None), "needs classes"),
]


def _no_device(monkeypatch, fw):
    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(type(fw.backbone), "_ensure_packed", no_device)


def _calls(cls, s, x, t, kw):
    kw = dict(kw)
    classes = kw.pop("classes", torch.tensor([1]))
    yield lambda: s.sample(1, steps=10, verbose=False, classes=classes, **kw)
    if cls is samplers.DdpmSampler:
        yield lambda: s.sample_once(x, t, classes, **kw)
    else:
        yield lambda: s.sample_once(x, t, t - 1, classes, **kw)


@pytest.mark.parametrize("kw,msg", BAD, ids=[f"case{i}" for i in range(len(BAD))])
def test_python_rejects_bad_apg(kw, msg, monkeypatch):
    """AssertionError from every sampler's sample and sample_once, before the network is packed and before any torch draw."""
    fw = _fw()
    _no_device(monkeypatch, fw)
    x = torch.zeros(1, 4, 32, 32)
    t = torch.full((1,), 10)
    for cls in SAMPLERS:
        s = cls(fw)
        for call in _calls(cls, s, x, t, kw):
            state = torch.get_rng_state()
            with pytest.raises(AssertionError, match=msg):
                call()
            assert torch.equal(state, torch.get_rng_state())


def test_python_rejects_apg_without_cfg_and_bad_state(monkeypatch):
    fw = _fw(frameworks.GaussianDiffusion, dict(TINY, num_classes=None, has_null_class=False))
    _no_device(monkeypatch, fw)
    x = torch.zeros(1, 4, 32, 32)
    t = torch.full((1,), 10)
    for cls in SAMPLERS:
        for call in _calls(cls, cls(fw), x, t, dict(apg=0.0)):
            with pytest.raises(AssertionError, match="does not have"):
                call()
    fw = _fw()
    _no_device(monkeypatch, fw)
    for cls in SAMPLERS:
        s = cls(fw)
        once = (lambda **k: s.sample_once(x, t, torch.tensor([1]), **k)) if cls is samplers.DdpmSampler else \
            (lambda **k: s.sample_once(x, t, t - 1, torch.tensor([1]), **k))
        with pytest.raises(AssertionError, match="apg_state needs apg"):
            once(apg_state=torch.zeros_like(x))
        with pytest.raises(AssertionError, match="apg_state must have x_t's shape"):
            once(apg=0.0, apg_state=torch.zeros(1, 4, 16, 16))


def test_native_rejects_bad_apg_before_device_work():
    """ivid_sampler_step / _step_dev / _run and ivid_op_apg reject bad APG fields with IVID_ERR_INVALID_ARGUMENT (the fake
    pointers are never dereferenced)."""
    L = _lib.lib()
    unet = ctypes.c_void_p()
    _lib.check(L.ivid_unet_create(json.dumps(TINY).encode(), ctypes.byref(unet)))
    s = samplers.DdimSampler(_fw())
    fake = ctypes.c_void_p(256)
    try:
        # (apg, use_cfg, classes, strength, eta, r, beta)
        cases = [(2, 1, True, 3.0, 0.0, 0.0, 0.0), (1, 0, True, 3.0, 0.0, 0.0, 0.0), (1, 1, False, 3.0, 0.0, 0.0, 0.0),
                 (1, 1, True, 0.0, 0.0, 0.0, 0.0), (1, 1, True, -1.0, 0.0, 0.0, 0.0), (1, 1, True, float("nan"), 0.0, 0.0, 0.0),
                 (1, 1, True, float("inf"), 0.0, 0.0, 0.0), (1, 1, True, 3.0, -0.5, 0.0, 0.0),
                 (1, 1, True, 3.0, float("nan"), 0.0, 0.0), (1, 1, True, 3.0, 0.0, -1.0, 0.0),
                 (1, 1, True, 3.0, 0.0, float("inf"), 0.0), (1, 1, True, 3.0, 0.0, 0.0, 1.0),
                 (1, 1, True, 3.0, 0.0, 0.0, -1.0), (1, 1, True, 3.0, 0.0, 0.0, float("nan"))]
        for apg, use_cfg, cls, strength, eta, r, beta in cases:
            a = _lib.StepArgsT()
            a.kind = 1
            a.use_cfg, a.strength = use_cfg, strength
            a.classes_dev = fake.value if cls else None
            a.apg, a.apg_eta, a.apg_norm, a.apg_momentum = apg, eta, r, beta
            case = (apg, use_cfg, cls, strength, eta, r, beta)
            rc = L.ivid_sampler_step(s._handle, unet, fake, fake, None, 1, 10, 9, ctypes.byref(a), None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "apg" in _lib.last_error(), case
            rc = L.ivid_sampler_step_dev(s._handle, unet, fake, fake, None, 1, fake, fake, ctypes.byref(a), None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "apg" in _lib.last_error(), case
            rc = L.ivid_sampler_run(s._handle, unet, fake, 1, 10, ctypes.byref(a), None, None, None, None, None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "apg" in _lib.last_error(), case
        for N, M, st, eta, r, beta in ((0, 16, 1.0, 0.0, 0.0, 0.0), (1, 0, 1.0, 0.0, 0.0, 0.0), (1, 16, 0.0, 0.0, 0.0, 0.0),
                                       (1, 16, float("nan"), 0.0, 0.0, 0.0), (1, 16, 1.0, -1.0, 0.0, 0.0),
                                       (1, 16, 1.0, 0.0, float("nan"), 0.0), (1, 16, 1.0, 0.0, 0.0, 1.0)):
            rc = L.ivid_op_apg(fake, fake, fake, N, M, st, eta, r, beta, fake, None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "apg" in _lib.last_error(), (N, M, st, eta, r, beta)
        rc = L.ivid_op_apg(fake, fake, None, 1, 16, 1.0, 0.0, 0.0, 0.0, fake, None)
        assert rc == _lib.IVID_ERR_INVALID_ARGUMENT
    finally:
        L.ivid_unet_destroy(unet)


# ---------------------------------------------------------------------------------------------------------------------
# sample_all and the CLI
# ---------------------------------------------------------------------------------------------------------------------
class _Recorder:
    def __init__(self):
        self.calls = []

    def sampler(self, name):
        rec = self

        class Fake:
            def __init__(self, fw):
                self.fw = fw

            def sample(self, num, **kw):
                rec.calls.append((name, type(self.fw).__name__, kw))
                S = self.fw.backbone.image_size
                return edict(samples=torch.zeros(num, 4, S, S))
        return Fake


class _FakeWarp:
    def __init__(self, bs, image_size, **kw):
        self.bs, self.S = bs, image_size

    def reset(self):
        pass

    def aggregate(self, mv, **kw):
        return torch.zeros(self.bs, 7, self.S, self.S)

    def add_view(self, *a, **k):
        pass


def test_sample_all_passes_apg_to_both_samplers(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(sample_cli.samplers, "DdimSampler", rec.sampler("ddim"))
    monkeypatch.setattr(sample_cli.samplers, "DdpmSampler", rec.sampler("ddpm"))
    monkeypatch.setattr(sample_cli, "DeviceWarp", _FakeWarp)
    fw_u, fw_c = _fw(), _fw(frameworks.InpaintCFG, TINY_COND)
    mv = sample_cli.build_modelviews("3x9", 1)
    out = list(sample_cli.sample_all(fw_u, fw_c, 1, 10, 10, mv, classes=[3], apg=(0.0, 1.0, -0.5)))
    assert len(out) == 1
    assert {fw_name for _, fw_name, _ in rec.calls} == {"ClassifierFreeGuidance", "InpaintCFG"}
    for name, fw_name, kw in rec.calls:
        assert kw["apg"] == (0.0, 1.0, -0.5) and kw["strength"] == 3.0, (name, fw_name)
    rec.calls.clear()
    list(sample_cli.sample_all(fw_u, fw_c, 1, 10, 10, mv, classes=[3]))
    assert rec.calls and all("apg" not in kw for _, _, kw in rec.calls)


def test_sample_all_rejects_apg_first():
    fw_g = _fw(frameworks.GaussianDiffusion, dict(TINY, num_classes=None, has_null_class=False))
    fw_c = _fw(frameworks.InpaintCFG, TINY_COND)
    mv = sample_cli.build_modelviews("3x9", 1)
    with pytest.raises(AssertionError, match="does not have"):
        next(sample_cli.sample_all(fw_g, fw_c, 1, 10, 10, mv, classes=[3], apg=0.0))
    with pytest.raises(AssertionError, match="needs classes"):
        next(sample_cli.sample_all(_fw(), fw_c, 1, 10, 10, mv, apg=0.0))
    with pytest.raises(AssertionError, match="momentum beta"):
        next(sample_cli.sample_all(_fw(), fw_c, 1, 10, 10, mv, classes=[3], apg=(0.0, 0.0, 2.0)))
    with pytest.raises(AssertionError, match="strength > 0"):
        next(sample_cli.sample_all(_fw(), fw_c, 1, 10, 10, mv, classes=[3], guidance=0.0, apg=0.0))


def test_cli_flag_and_output_dir():
    o = sample_cli.parse_args(["--apg", "0"])
    assert o.apg == 0.0 and sample_cli.output_dir_name(o).endswith("_apg0.0")
    o = sample_cli.parse_args(["--apg", "0,2"])
    assert o.apg == (0.0, 2.0) and sample_cli.output_dir_name(o).endswith("_apg0.0,2.0")
    o = sample_cli.parse_args(["--apg", "0.5,0,-0.5"])
    assert o.apg == (0.5, 0.0, -0.5) and sample_cli.output_dir_name(o).endswith("_apg0.5,0.0,-0.5")
    plain = sample_cli.parse_args([])
    assert plain.apg is None and "apg" not in sample_cli.output_dir_name(plain)
    for bad in ("-1", "nan", "x", "0,-1", "0,inf", "0,0,1", "0,0,-1", "0,0,0,0", ""):
        with pytest.raises(SystemExit):
            sample_cli.parse_args(["--apg", bad])
    assert math.isfinite(sample_cli.parse_apg("0,0,0.99")[2])

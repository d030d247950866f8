"""CPU: perturbed-attention guidance (PAG) argument checks, defaults, plumbing through sample_all and the CLI, and the float64
mix model.  Every error is raised before any device work and before any torch draw."""
import ctypes
import inspect
import json
import math

import numpy as np
import pytest
import torch

import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
import pag_ref
from ivid_b200 import _lib
from ivid_b200.inference import sample as sample_cli
from ivid_b200.utils import edict

T = 1000
TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16], channel_mult=[1, 2], num_head_channels=64)
TINY_COND = dict(TINY, in_channels=9)
SAMPLERS = (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler, samplers.UniPcSampler)
FRAMEWORKS = (frameworks.GaussianDiffusion, frameworks.ClassifierFreeGuidance, frameworks.InpaintCFG, frameworks.SuperResCFG)


def _fw(cls=frameworks.ClassifierFreeGuidance, cfg=TINY):
    return cls(backbones.AdmUnet2d(**cfg), timesteps=T, beta_schedule="linear")


def test_attention_layer_names_follow_the_state_dict():
    net = backbones.AdmUnet2d(**TINY)
    names = net.attention_layers
    assert "middle_block.1" in names
    assert names == pag_ref.attention_layers(TINY)
    keys = [k for k in net.state_dict() if k.endswith(".qkv.weight")]
    assert names == [k[: -len(".qkv.weight")] for k in keys]
    assert net.pag_layer_indices(["middle_block.1"]) == [names.index("middle_block.1")]
    assert net.pag_layer_indices(list(reversed(names))) == list(reversed(range(len(names))))


def test_defaults_are_none():
    for cls in SAMPLERS:
        for fn in (cls.sample, cls.sample_once):
            p = inspect.signature(fn).parameters
            assert p["pag_scale"].default is None and p["pag_layers"].default is None, (cls, fn)
    for cls in FRAMEWORKS:
        p = inspect.signature(cls.model_inference).parameters
        assert p["pag_scale"].default is None and p["pag_layers"].default is None, cls
    p = inspect.signature(sample_cli.sample_all).parameters
    assert p["pag_scale"].default is None and p["pag_layers"].default is None
    assert inspect.signature(backbones.AdmUnet2d.forward_perturbed).parameters["layers"].default == ("middle_block.1",)
    # AdmUnet2d.forward keeps the reference's signature
    assert list(inspect.signature(backbones.AdmUnet2d.forward).parameters) == ["self", "x", "times", "classes"]
    a = _lib.StepArgsT()
    assert (a.pag, a.pag_scale, a.pag_num_layers) == (0, 0.0, 0) and not a.pag_layers


BAD = [
    (dict(pag_scale=-1.0), "pag_scale must be finite"),
    (dict(pag_scale=float("nan")), "pag_scale must be finite"),
    (dict(pag_scale=float("inf")), "pag_scale must be finite"),
    (dict(pag_scale=True), "pag_scale must be a real"),
    (dict(pag_scale="1"), "pag_scale must be a real"),
    (dict(pag_scale=1.0, pag_layers=[]), "at least one attention layer"),
    (dict(pag_scale=1.0, pag_layers=["middle_block.0"]), "is not an attention layer"),
    (dict(pag_scale=1.0, pag_layers=["nonsense"]), "is not an attention layer"),
    (dict(pag_scale=1.0, pag_layers="middle_block.1"), "sequence of layer names"),
    (dict(pag_scale=1.0, pag_layers=["middle_block.1", "middle_block.1"]), "twice"),
    (dict(pag_layers=["middle_block.1"]), "pag_layers needs pag_scale"),
]


def _no_device(monkeypatch, fw):
    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(type(fw.backbone), "_ensure_packed", no_device)


@pytest.mark.parametrize("kw,msg", BAD, ids=[f"case{i}" for i in range(len(BAD))])
def test_python_rejects_bad_pag(kw, msg, monkeypatch):
    """AssertionError from every sampler's sample and sample_once and from every framework's model_inference, before the
    network is packed and before any torch draw."""
    fw = _fw()
    _no_device(monkeypatch, fw)
    x = torch.zeros(1, 4, 32, 32)
    t = torch.full((1,), 10)
    for cls in SAMPLERS:
        s = cls(fw)
        state = torch.get_rng_state()
        with pytest.raises(AssertionError, match=msg):
            s.sample(1, steps=10, verbose=False, **kw)
        with pytest.raises(AssertionError, match=msg):
            if cls is samplers.DdpmSampler:
                s.sample_once(x, t, **kw)
            else:
                s.sample_once(x, t, t - 1, **kw)
        assert torch.equal(state, torch.get_rng_state())
    for fcls in FRAMEWORKS:
        f = _fw(fcls, TINY_COND if fcls is frameworks.InpaintCFG else (dict(TINY, in_channels=8) if fcls is frameworks.SuperResCFG else TINY))
        _no_device(monkeypatch, f)
        extra = dict(y=torch.zeros(1, 4, 32, 32), mask=torch.zeros(1, 1, 32, 32)) if fcls is frameworks.InpaintCFG else \
            (dict(y=torch.zeros(1, 4, 16, 16)) if fcls is frameworks.SuperResCFG else {})
        state = torch.get_rng_state()
        with pytest.raises(AssertionError, match=msg):
            f.model_inference(x, t, **extra, **kw)
        assert torch.equal(state, torch.get_rng_state())
    if kw.get("pag_layers") is not None and kw.get("pag_scale") == 1.0:
        with pytest.raises(AssertionError, match=msg):
            fw.backbone.forward_perturbed(x, t, layers=kw["pag_layers"])


def test_native_rejects_bad_pag_before_device_work():
    """ivid_sampler_step / _step_dev / _run and ivid_unet_forward_perturbed reject bad PAG fields with
    IVID_ERR_INVALID_ARGUMENT (the fake pointers are never dereferenced)."""
    L = _lib.lib()
    unet = ctypes.c_void_p()
    _lib.check(L.ivid_unet_create(json.dumps(TINY).encode(), ctypes.byref(unet)))
    s = samplers.DdimSampler(_fw())
    fake = ctypes.c_void_p(256)
    nattn = len(pag_ref.attention_layers(TINY))
    try:
        cases = [(2, 1.0, [0]), (1, -0.5, [0]), (1, float("nan"), [0]), (1, float("inf"), [0]), (1, 1.0, []),
                 (1, 1.0, [nattn]), (1, 1.0, [-1]), (1, 1.0, [0, 0])]
        for pag, w, layers in cases:
            a = _lib.StepArgsT()
            a.kind = 1
            arr = (ctypes.c_int * max(len(layers), 1))(*layers)
            a.pag, a.pag_scale, a.pag_layers, a.pag_num_layers = pag, w, arr if layers else None, len(layers)
            rc = L.ivid_sampler_step(s._handle, unet, fake, fake, None, 1, 10, 9, ctypes.byref(a), None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "pag" in _lib.last_error(), (pag, w, layers)
            rc = L.ivid_sampler_step_dev(s._handle, unet, fake, fake, None, 1, fake, fake, ctypes.byref(a), None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "pag" in _lib.last_error(), (pag, w, layers)
            rc = L.ivid_sampler_run(s._handle, unet, fake, 1, 10, ctypes.byref(a), None, None, None, None, None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "pag" in _lib.last_error(), (pag, w, layers)
        for row0, layers in ((-1, [0]), (3, [0]), (1, []), (1, [nattn]), (1, [0, 0])):
            arr = (ctypes.c_int * max(len(layers), 1))(*layers)
            rc = L.ivid_unet_forward_perturbed(unet, fake, 2, 32, 32, None, fake, None, fake, 2, row0, arr if layers else None,
                                               len(layers), -1, None)
            assert rc in (_lib.IVID_ERR_INVALID_ARGUMENT, _lib.IVID_ERR_STATE), (row0, layers)
            if layers and row0 in (-1, 3):
                assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "row0" in _lib.last_error()
        for cfg, pag, w in ((3, 1, 1.0), (1, 2, 1.0), (1, 1, -1.0), (0, 1, float("nan"))):
            rc = L.ivid_guidance_mix(fake, 16, cfg, 1.0, pag, w, fake, None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "guidance mix" in _lib.last_error(), (cfg, pag, w)
        rc = L.ivid_op_attention_perturbed(fake, 2, 64, 64, 64, 3, fake, None)
        assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "row0" in _lib.last_error()
    finally:
        L.ivid_unet_destroy(unet)


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


@pytest.mark.parametrize("uncond_cls", [frameworks.GaussianDiffusion, frameworks.ClassifierFreeGuidance])
def test_sample_all_passes_pag_to_both_samplers(uncond_cls, monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(sample_cli.samplers, "DdimSampler", rec.sampler("ddim"))
    monkeypatch.setattr(sample_cli.samplers, "DdpmSampler", rec.sampler("ddpm"))
    monkeypatch.setattr(sample_cli, "DeviceWarp", _FakeWarp)
    fw_u = _fw(uncond_cls)
    fw_c = _fw(frameworks.InpaintCFG, TINY_COND)
    mv = sample_cli.build_modelviews("3x9", 1)
    cls = [3] if uncond_cls is frameworks.ClassifierFreeGuidance else None
    layers = ("middle_block.1", fw_u.backbone.attention_layers[0])
    out = list(sample_cli.sample_all(fw_u, fw_c, 1, 10, 10, mv, classes=cls, pag_scale=2.0, pag_layers=layers,
                                     guidance_interval=(100, 900)))
    assert len(out) == 1
    assert rec.calls and rec.calls[0][0] == "ddim" and rec.calls[0][1] == uncond_cls.__name__
    for name, fw_name, kw in rec.calls:
        assert kw["pag_scale"] == 2.0 and tuple(kw["pag_layers"]) == layers, (name, fw_name)
        assert kw["guidance_interval"] == (100, 900), "the interval gates PAG on every network"
    # without PAG nothing new is passed, and a GaussianDiffusion still gets no strength and no interval
    rec.calls.clear()
    list(sample_cli.sample_all(fw_u, fw_c, 1, 10, 10, mv, classes=cls, guidance_interval=(100, 900)))
    for name, fw_name, kw in rec.calls:
        assert "pag_scale" not in kw and "pag_layers" not in kw
        if fw_name == "GaussianDiffusion":
            assert "strength" not in kw and "guidance_interval" not in kw


def test_sample_all_rejects_bad_pag_first():
    fw = _fw()
    mv = sample_cli.build_modelviews("uncond", 1)
    with pytest.raises(AssertionError, match="not an attention layer"):
        next(sample_cli.sample_all(fw, None, 1, 10, 10, mv, pag_scale=1.0, pag_layers=["out"]))
    with pytest.raises(AssertionError, match="pag_scale must be finite"):
        next(sample_cli.sample_all(fw, None, 1, 10, 10, mv, pag_scale=-2.0))


def test_cli_flags_and_output_dir():
    o = sample_cli.parse_args(["--pag_scale", "3"])
    assert o.pag_scale == 3.0 and o.pag_layers is None
    assert sample_cli.output_dir_name(o).endswith("_pag3.0")
    o = sample_cli.parse_args(["--pag_scale", "1.5", "--pag_layers", "input_blocks.7.1,middle_block.1"])
    assert o.pag_layers == ("input_blocks.7.1", "middle_block.1")
    assert sample_cli.output_dir_name(o).endswith("_pag1.5-input_blocks.7.1+middle_block.1")
    o = sample_cli.parse_args(["--pag_scale", "2", "--pag_layers", "middle_block.1"])
    assert sample_cli.output_dir_name(o).endswith("_pag2.0")
    plain = sample_cli.parse_args([])
    assert plain.pag_scale is None and plain.pag_layers is None and "pag" not in sample_cli.output_dir_name(plain)
    for bad in (["--pag_scale", "-1"], ["--pag_scale", "nan"], ["--pag_scale", "inf"], ["--pag_scale", "x"],
                ["--pag_layers", "middle_block.1"], ["--pag_scale", "1", "--pag_layers", "a,,b"]):
        with pytest.raises(SystemExit):
            sample_cli.parse_args(bad)


@pytest.mark.parametrize("cfg", [0, 1, 2])
def test_mix_model_reduces_to_todays_mix_at_w0(cfg):
    rng = np.random.default_rng(cfg)
    ec, eu, ep = (rng.standard_normal(4096).astype(np.float32) for _ in range(3))
    s = 0.7 if cfg == 1 else -0.3
    g64 = {0: ec.astype(np.float64), 1: (1 + s) * ec.astype(np.float64) - s * eu.astype(np.float64),
           2: (1 + s) * ec.astype(np.float64)}[cfg]
    assert np.array_equal(pag_ref.mix64(ec, ep, 0.0, cfg, s, eu), g64)
    g32 = pag_ref.mix32(ec, ep, 0.0, cfg, s, eu)
    assert g32.dtype == np.float32
    assert np.abs(g32 - g64).max() <= 4 * np.finfo(np.float32).eps * (np.abs(g64).max() + 1)
    # and the w term is the float64 one to fp32 accuracy
    w = 2.5
    d = pag_ref.mix32(ec, ep, w, cfg, s, eu) - pag_ref.mix64(ec, ep, w, cfg, s, eu)
    assert np.abs(d).max() <= 16 * np.finfo(np.float32).eps * (np.abs(pag_ref.mix64(ec, ep, w, cfg, s, eu)).max() + 1)
    assert math.isfinite(float(d.sum()))


def test_identity_attention_model_outputs_v():
    """The model's identity attention is x + proj_out(V) with V the [head][q|k|v][d] value channels."""
    from oracle import unet_ref
    torch.manual_seed(0)
    C, d, T_ = 128, 64, 9
    sd = {"a.norm.weight": torch.ones(C), "a.norm.bias": torch.zeros(C), "a.qkv.weight": torch.randn(3 * C, C, 1),
          "a.qkv.bias": torch.randn(3 * C), "a.proj_out.weight": torch.eye(C)[:, :, None], "a.proj_out.bias": torch.zeros(C)}
    x = torch.randn(2, C, 3, 3)
    out = pag_ref.identity_attention(x, sd, "a", 32, d)
    qkv = torch.nn.functional.conv1d(unet_ref._group_norm(x.reshape(2, C, -1), sd, "a.norm", 32), sd["a.qkv.weight"], sd["a.qkv.bias"])
    v = torch.cat([qkv[:, 3 * d * h + 2 * d: 3 * d * h + 3 * d] for h in range(C // d)], dim=1)
    assert torch.allclose(out.reshape(2, C, -1), x.reshape(2, C, -1) + v, atol=1e-6)
    # the oracle's own attention is back in place after a perturbed forward
    before = unet_ref._attention
    with pag_ref._perturbed(["a"]):
        assert unet_ref._attention is not before
    assert unet_ref._attention is before

"""CPU: AdmUnet2d at channel widths that are not multiples of 64 — the golden eps of the unmodified reference
(widths_golden.npz) against the oracle, the state-dict schema and load_state_dict, and the width error contract
(num_groups must divide every width: AssertionError; widths that are not multiples of 8: NotImplementedError).  No GPU
calls."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import ivid_b200.backbones as backbones
from ivid_b200 import _lib
from oracle import sampler_ref, unet_ref

UNET_TAGS = ["mc96", "mc32", "frac", "g8", "narrow8", "legacy96"]
STRENGTH = 0.5


@pytest.fixture(scope="module")
def wid():
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "widths_golden.npz")))


def _cfg(g, tag):
    return json.loads(bytes(g[f"{tag}_cfg"]).decode())


def _T(g, tag, k):
    return torch.from_numpy(g[f"{tag}_{k}"])


@pytest.mark.parametrize("tag", UNET_TAGS)
def test_golden_matches_oracle(wid, tag):
    cfg = _cfg(wid, tag)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    ora = unet_ref.unet_forward(cfg, sd, _T(wid, tag, "x"), _T(wid, tag, "t"), _T(wid, tag, "c"))
    assert torch.equal(ora, _T(wid, tag, "eps"))


def test_inpaint_golden_matches_oracle(wid):
    cfg = _cfg(wid, "inpaint96")
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    g = lambda k: _T(wid, "inpaint96", k)
    noise = g("noise")
    ci = sampler_ref.make_inpaint_inputs(g("x"), g("y"), g("mask"), g("mask_rgb"), noise[:, :3], noise[:, 3:])
    model = lambda xx, tt, cc: unet_ref.unet_forward(cfg, sd, xx, tt, cc)
    assert torch.equal(sampler_ref.cond_eps(model, ci, g("t"), g("c"), STRENGTH), g("eps"))


def _widths(cfg):
    blocks, final = unet_ref._topology(cfg)
    ws = {final}
    for b in blocks:
        for layer in b["layers"]:
            ws.update(v for v in layer[3 if layer[0] == "conv" else 2:] if isinstance(v, int))    # not the stem's input
    return ws


@pytest.mark.parametrize("tag", UNET_TAGS + ["inpaint96"])
def test_construction_and_schema(wid, tag):
    cfg = _cfg(wid, tag)
    assert any(w % 64 for w in _widths(cfg)), "every case has a width that is not a multiple of 64"
    net = backbones.AdmUnet2d(**cfg)
    want = [(k, tuple(v.shape)) for k, v in unet_ref.make_synthetic_state_dict(cfg, seed=77).items()]
    got = [(k, tuple(v.shape)) for k, v in net.state_dict().items()]
    assert got == want
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=77))


def _create_code(cfg):
    h = ctypes.c_void_p()
    L = _lib.lib()
    rc = L.ivid_unet_create(json.dumps(cfg).encode(), ctypes.byref(h))
    if rc == 0:
        L.ivid_unet_destroy(h)
    return rc


def test_width_not_multiple_of_8_is_not_implemented(wid):
    """num_groups=4, model_channels=20, channel_mult=[1, 3.2]: widths 20, 64, 84 and 40, all divisible by 4, so the
    reference runs it (the fixture generator checks that); 20 and 84 are not multiples of 8."""
    cfg = _cfg(wid, "g4_20")
    assert _widths(cfg) == {20, 40, 64, 84, 128}
    with pytest.raises(NotImplementedError):
        backbones.AdmUnet2d(**cfg)
    assert _create_code(cfg) == _lib.IVID_ERR_NOT_IMPLEMENTED


@pytest.mark.parametrize("extra", [dict(model_channels=48),                               # 48 % 32 != 0
                                   dict(model_channels=96, channel_mult=[1, 1.25, 2]),   # level width 120
                                   dict(num_groups=3, model_channels=20, channel_mult=[1, 3.2])])   # 20 % 3: checked before % 8
def test_width_not_divisible_by_num_groups_asserts(extra):
    cfg = dict(dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1, attention_resolutions=[],
                    channel_mult=[1, 2], num_classes=10, has_null_class=True, num_groups=32, num_heads=None,
                    num_head_channels=64, dropout=0.0, use_fp16=False), **extra)
    with pytest.raises(AssertionError):
        backbones.AdmUnet2d(**cfg)
    assert _create_code(cfg) == _lib.IVID_ERR_INVALID_ARGUMENT

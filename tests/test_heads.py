"""CPU: AdmUnet2d at attention head widths other than 64 — the golden eps of the unmodified reference (heads_golden.npz)
against the oracle, construction and state-dict schema, and the reference's error contract for num_heads /
num_head_channels.  No GPU calls."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import ivid_b200.backbones as backbones
from ivid_b200 import _lib
from oracle import unet_ref

TAGS = ["hc128", "nh4", "single"]
TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16, 8], channel_mult=[1, 2, 2], num_classes=10, has_null_class=True,
            num_groups=32, dropout=0.0, use_fp16=False)


@pytest.fixture(scope="module")
def heads_golden():
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "heads_golden.npz")))


def _cfg(g, tag):
    return json.loads(bytes(g[f"{tag}_cfg"]).decode())


@pytest.mark.parametrize("tag", TAGS)
def test_golden_matches_oracle(heads_golden, tag):
    g = heads_golden
    cfg = _cfg(g, tag)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    ora = unet_ref.unet_forward(cfg, sd, torch.from_numpy(g[f"{tag}_x"]), torch.from_numpy(g[f"{tag}_t"]),
                                torch.from_numpy(g[f"{tag}_c"]))
    assert torch.equal(ora, torch.from_numpy(g[f"{tag}_eps"]))


@pytest.mark.parametrize("tag", TAGS)
def test_construction_and_schema(heads_golden, tag):
    cfg = _cfg(heads_golden, tag)
    net = backbones.AdmUnet2d(**cfg)
    want = [(k, tuple(v.shape)) for k, v in unet_ref.make_synthetic_state_dict(cfg, seed=77).items()]
    got = [(k, tuple(v.shape)) for k, v in net.state_dict().items()]
    assert sorted(got) == sorted(want)
    assert len(got) == len(want)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=77))


def test_num_heads_none_means_one():
    """num_heads=None with num_head_channels=-1 is one head per block, as in the oracle's _cfg_defaults: here 64 channels."""
    cfg = dict(TINY, channel_mult=[1, 1], attention_resolutions=[32, 16], num_heads=None, num_head_channels=-1)
    assert unet_ref._cfg_defaults(cfg)["num_heads"] == 1
    backbones.AdmUnet2d(**cfg)
    # the same network with two heads per block would be 32 channels wide: not supported, so None really means 1
    with pytest.raises(NotImplementedError):
        backbones.AdmUnet2d(**dict(cfg, num_heads=2))


def test_head_channels_must_divide_channels():
    """adm.py:272: channels % num_head_channels != 0 -> AssertionError (192 does not divide 64 or 128)."""
    with pytest.raises(AssertionError):
        backbones.AdmUnet2d(**dict(TINY, num_heads=None, num_head_channels=192))


def test_num_heads_must_divide_channels():
    """adm.py:244: channels % num_heads != 0 -> AssertionError (raised at construction here, at the first forward there)."""
    with pytest.raises(AssertionError):
        backbones.AdmUnet2d(**dict(TINY, num_heads=3, num_head_channels=-1))


@pytest.mark.parametrize("hc", [32, 96])
def test_head_width_not_multiple_of_64(hc):
    cfg = dict(TINY, model_channels=192, channel_mult=[1, 2, 2], num_heads=None, num_head_channels=hc)
    with pytest.raises(NotImplementedError):
        backbones.AdmUnet2d(**cfg)
    L = _lib.lib()
    h = ctypes.c_void_p()
    assert L.ivid_unet_create(json.dumps(cfg).encode(), ctypes.byref(h)) == _lib.IVID_ERR_NOT_IMPLEMENTED

"""CPU: AdmUnet2d and the frameworks at input sizes other than a square power of two — the golden eps of the unmodified
reference (geometry_golden.npz) against the oracle, the state-dict schema, the implicit-GEMM conv tile rule (host-side
query ivid_conv_tile) and the super-resolution scale contract.  No GPU calls."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import ivid_b200.backbones as backbones
from ivid_b200 import _lib
from ivid_b200.frameworks import SuperResCFG
from oracle import sampler_ref, unet_ref

UNET_TAGS = ["np2", "np2_single", "short", "rect", "big"]
SR_TAGS = ["sr4", "sr3"]
SR_STRENGTH = 0.5


@pytest.fixture(scope="module")
def geo():
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "geometry_golden.npz")))


def _cfg(g, tag):
    return json.loads(bytes(g[f"{tag}_cfg"]).decode())


def _T(g, tag, k):
    return torch.from_numpy(g[f"{tag}_{k}"])


@pytest.mark.parametrize("tag", UNET_TAGS)
def test_golden_matches_oracle(geo, tag):
    cfg = _cfg(geo, tag)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    ora = unet_ref.unet_forward(cfg, sd, _T(geo, tag, "x"), _T(geo, tag, "t"), _T(geo, tag, "c"))
    assert torch.equal(ora, _T(geo, tag, "eps"))


@pytest.mark.parametrize("tag", SR_TAGS)
def test_sr_golden_matches_oracle(geo, tag):
    cfg = _cfg(geo, tag)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    x, y = _T(geo, tag, "x"), _T(geo, tag, "y")
    ci = sampler_ref.make_sr_inputs(x, y)
    assert torch.equal(ci, torch.cat([x, _T(geo, tag, "up")], dim=1))
    model = lambda xx, tt, cc: unet_ref.unet_forward(cfg, sd, xx, tt, cc)
    ora = sampler_ref.cond_eps(model, ci, _T(geo, tag, "t"), _T(geo, tag, "c"), SR_STRENGTH)
    assert torch.equal(ora, _T(geo, tag, "eps"))


@pytest.mark.parametrize("tag", SR_TAGS)
def test_sr_make_cond_inputs(geo, tag):
    """make_cond_inputs upsamples by the integer scale_factor, as sr_cfg.py:31-36 does."""
    fw = SuperResCFG.__new__(SuperResCFG)          # make_cond_inputs needs no backbone
    x, y = _T(geo, tag, "x"), _T(geo, tag, "y")
    assert torch.equal(fw.make_cond_inputs(x, y), torch.cat([x, _T(geo, tag, "up")], dim=1))


@pytest.mark.parametrize("tag", ["np2", "np2_single", "short"])
def test_construction_and_schema(geo, tag):
    cfg = _cfg(geo, tag)
    net = backbones.AdmUnet2d(**cfg)
    want = [(k, tuple(v.shape)) for k, v in unet_ref.make_synthetic_state_dict(cfg, seed=77).items()]
    got = [(k, tuple(v.shape)) for k, v in net.state_dict().items()]
    assert got == want
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=77))


def _tile(H, W):
    tw, th, tn, fs = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.lib().ivid_conv_tile(H, W, ctypes.byref(tw), ctypes.byref(th), ctypes.byref(tn), ctypes.byref(fs)))
    return tw.value, th.value, tn.value, bool(fs.value)


def _levels(H, W, n):
    return [(H >> i, W >> i) for i in range(n)]


def test_tile_rule_keeps_power_of_two_tiles(golden):
    """For every power-of-two layer of the four real configs the tile is the one used before any-size support:
    TW = min(W, 16), TH = min(H, 128 / TW), TN = 128 / (TW * TH); statistics fuse iff TW * TH >= 32."""
    seen = set()
    for k in golden:
        if not k.startswith("schemacfg_"):
            continue
        cfg = json.loads(bytes(golden[k]).decode())
        seen.update(_levels(cfg["image_size"], cfg["image_size"], len(cfg["channel_mult"])))
    seen.update((h, w) for h in (1, 2, 4, 8, 16, 32, 64, 128, 256) for w in (1, 2, 4, 8, 16, 32, 64, 128, 256))
    for H, W in sorted(seen):
        tw = min(W, 16); th = min(H, 128 // tw)
        assert _tile(H, W) == (tw, th, 128 // (tw * th), tw * th >= 32), (H, W)


def test_tile_rule_never_overhangs(geo):
    """Tiles divide every layer of the golden geometries (only the batch tail is masked), and the examples of the rule."""
    sizes = [(48, 48), (40, 24), (64, 64), (32, 32), (96, 96), (160, 96), (3, 5), (12, 20), (6, 10), (48, 80)]
    for tag in UNET_TAGS + SR_TAGS:
        x = geo[f"{tag}_x"]
        sizes += _levels(x.shape[2], x.shape[3], len(_cfg(geo, tag)["channel_mult"]))
    for H, W in sizes:
        tw, th, tn, fs = _tile(H, W)
        assert W % tw == 0 and H % th == 0 and tw * th * tn == 128, (H, W)
        assert tw == 16 or W % (2 * tw) != 0, (H, W)                 # the largest power of two <= 16 dividing W
        assert th == 128 // tw or H % (2 * th) != 0, (H, W)
        assert fs == (tw * th >= 32)
    assert _tile(24, 40)[:3] == (8, 8, 2)
    assert _tile(3, 5)[:3] == (1, 1, 128)
    assert _tile(12, 20)[:3] == (4, 4, 8) and not _tile(12, 20)[3]
    with pytest.raises(AssertionError):
        _tile(0, 8)


@pytest.mark.parametrize("xs,ys", [((30, 30), (8, 8)), ((32, 32), (8, 16)), ((32, 24), (8, 8)), ((8, 8), (16, 16))])
def test_sr_scale_must_be_an_integer_multiple(xs, ys):
    with pytest.raises(RuntimeError):
        SuperResCFG._scale(torch.empty(1, 4, *xs), torch.empty(1, 4, *ys))


@pytest.mark.parametrize("xs,ys,s", [((32, 32), (8, 8), 4), ((48, 48), (16, 16), 3), ((40, 24), (20, 12), 2), ((8, 8), (8, 8), 1)])
def test_sr_scale(xs, ys, s):
    assert SuperResCFG._scale(torch.empty(1, 4, *xs), torch.empty(1, 4, *ys)) == s

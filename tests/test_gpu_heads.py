"""GPU: attention at head widths other than 64 (attention_hd_kernel) — the op against an fp32 torch computation, the whole
AdmUnet2d against the unmodified reference's eps (heads_golden.npz) and the oracle's per-block taps, the large config with the
reference's single-head default, and bitwise determinism / batch invariance.  Eps bars follow tests/test_gpu_unet.py."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch

import gpu_util as G
import ivid_b200.backbones as backbones
import precision_model as PM
from ivid_b200 import _lib
from oracle import unet_ref

pytestmark = pytest.mark.gpu
NORTH_STAR = 1e-3
HARD_CAP = 1.6e-3
TAGS = ["hc128", "nh4", "single"]


def _bar(floor):
    return min(max(NORTH_STAR, 1.15 * floor), HARD_CAP)


@pytest.fixture(scope="module")
def heads_golden():
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "heads_golden.npz")))


def _attention_heads(qkv_f16, C, d):
    N, T, _ = qkv_f16.shape
    out = torch.empty((N, T, C), dtype=torch.float16, device="cuda")
    _lib.check(_lib.lib().ivid_op_attention_heads(_lib.ptr(qkv_f16), N, T, C, d, _lib.ptr(out), _lib.cur_stream()))
    return out


def _qkv(N, T, C, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(N, 3 * C, T, generator=g).half()          # reference layout [N, 3C, T]


def _torch_attention(qh, C, d):
    """QKVAttention (adm.py:233-253) in fp32 on the fp16 inputs."""
    N, _, T = qh.shape
    q, k, v = qh.float().reshape(N * (C // d), 3 * d, T).split(d, dim=1)
    s = 1 / math.sqrt(math.sqrt(d))
    w = torch.softmax(torch.einsum("bct,bcs->bts", q * s, k * s), dim=-1)
    return torch.einsum("bts,bcs->bct", w, v).reshape(N, C, T)


OP_CASES = [(d, T) for d in (128, 192, 256, 384, 512, 1024) for T in (64, 256, 1024)] + [(d, 4096) for d in (128, 192, 256)]


@pytest.mark.parametrize("d,T", OP_CASES)
def test_attention_heads_matches_torch(d, T):
    C = 2 * d if d <= 512 else d
    N = 1 if T == 4096 else 2
    qh = _qkv(N, T, C, d * 7 + T).cuda()
    ref = _torch_attention(qh, C, d)
    out = _attention_heads(qh.permute(0, 2, 1).contiguous(), C, d)
    r = G.report(f"attention_heads N{N} T{T} C{C} d{d}", out.float().permute(0, 2, 1), ref)
    assert r < 2e-3


@pytest.mark.parametrize("N,T,C", [(2, 256, 128), (1, 1024, 512)])
def test_attention_heads_d64_is_attention(N, T, C):
    """Head width 64 through the new entry point is the existing kernel: the same bits."""
    qkv = _qkv(N, T, C, 3).permute(0, 2, 1).contiguous().cuda()
    assert torch.equal(_attention_heads(qkv, C, 64), G.attention(qkv, C))


def test_attention_heads_rejects_bad_widths():
    qkv = torch.zeros(1, 64, 3 * 192, dtype=torch.float16, device="cuda")
    with pytest.raises(NotImplementedError):
        _attention_heads(qkv, 192, 96)
    with pytest.raises(AssertionError):
        _attention_heads(qkv, 192, 128)


def _load(cfg, sd):
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(sd)
    return net.cuda()


def _tap(net, N, name):
    L = _lib.lib()
    C, H, W = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), None, 0, ctypes.byref(C), ctypes.byref(H), ctypes.byref(W)))
    out = torch.empty((N, C.value, H.value, W.value), dtype=torch.float32)
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), _lib.ptr(out), out.numel(), None, None, None))
    return out


def _check(name, got, ref, cfg, sd, x, t, c):
    floor = PM.rel(PM.forward(cfg, sd, x, t, c, PM.TF32_CLASS), ref)
    err = G.report(name, got, ref)
    print(f"[parity] {name}: eps rel {err:.3e}  TF32-class floor {floor:.3e}  bar {_bar(floor):.3e}")
    assert err <= _bar(floor), f"{name}: eps rel {err:.3e} > bar {_bar(floor):.3e} (floor {floor:.3e})"


@pytest.mark.parametrize("tag", TAGS)
def test_unet_heads_vs_reference_golden(heads_golden, tag):
    g = heads_golden
    cfg = json.loads(bytes(g[f"{tag}_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    net = _load(cfg, sd)
    x = torch.from_numpy(g[f"{tag}_x"]); t = torch.from_numpy(g[f"{tag}_t"]); c = torch.from_numpy(g[f"{tag}_c"])
    got = net(x.cuda(), t.cuda(), c.cuda())
    _check(f"{tag} eps", got, torch.from_numpy(g[f"{tag}_eps"]), cfg, sd, x, t, c)
    taps = {}
    unet_ref.unet_forward(cfg, sd, x, t, c, taps=taps)
    blocks, _ = unet_ref._topology(cfg)
    worst = 0.0
    for name in [l[1] for b in blocks for l in b["layers"] if l[0] == "attn"]:
        r = G.rel(_tap(net, 2, name), taps[name])
        print(f"[tap] {tag} {name} rel {r:.3e}")
        worst = max(worst, r)
    assert worst < HARD_CAP


def test_large_config_single_head(golden):
    """rgbd_imagenet_adm_128_large_cfg with the reference's defaults num_heads=1, num_head_channels=-1: one head of
    512 / 768 / 1024 channels at T = 1024 / 256 / 64 (the sliced, Q-streaming path)."""
    cfg = json.loads(bytes(golden["schemacfg_rgbd_imagenet_adm_128_large_cfg"]).decode())
    cfg = dict(cfg, num_heads=1, num_head_channels=-1)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    net = _load(cfg, sd)
    rng = np.random.default_rng(11)
    x = torch.from_numpy(rng.standard_normal((1, 4, 128, 128)).astype(np.float32))
    t = torch.tensor([999]); c = torch.tensor([3])
    ref = unet_ref.unet_forward(cfg, sd, x, t, c)
    _check("large single-head eps", net(x.cuda(), t.cuda(), c.cuda()), ref, cfg, sd, x, t, c)


@pytest.mark.parametrize("tag", ["single", "nh4"])
def test_heads_deterministic_and_batch_invariant(heads_golden, tag):
    cfg = json.loads(bytes(heads_golden[f"{tag}_cfg"]).decode())
    net = _load(cfg, unet_ref.make_synthetic_state_dict(cfg, seed=77))
    N = 8
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, 4, 32, 32, generator=g).cuda()
    t = torch.arange(N, device="cuda") * 120 + 3; c = torch.arange(N, device="cuda") % 10
    first = net(x, t, c).clone()
    bad = sum(0 if torch.equal(net(x, t, c), first) else 1 for _ in range(10))
    assert bad == 0, f"{bad} of 10 forwards differ from the first"
    for i in (0, 5):
        one = net(x[i:i + 1].contiguous(), t[i:i + 1], c[i:i + 1])
        assert torch.equal(one, first[i:i + 1]), f"sample {i}: eps depends on the batch"

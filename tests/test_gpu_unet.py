"""GPU parity of the whole AdmUnet2d forward (through the reference-facing class and the C ABI) against
 (a) the committed golden vectors produced by the unmodified reference (tiny configs),
 (b) the CPU oracle on the real configs (small / large / cond / SR), computed in-test,
 (c) the oracle's per-layer taps (ivid_unet_debug_tap).

Tolerance on eps (relative L2 against the strict-fp32 oracle).  The tensor-core operands are fp16 (10-bit mantissa, the
mantissa of TF32); everything between the GEMMs is fp32 or a single extra fp16 rounding (tests/precision_model.py lists
every one).  The bar per case is

        max(1e-3, 1.15 x floor)        and never above 1.6e-3,

where `floor` is computed IN THE SAME TEST: the oracle with only its conv / GEMM operands rounded to a 10-bit mantissa —
what the unmodified reference itself computes on the A100 it was tested on (PyTorch 1.11 runs fp32 convolutions and
matmuls in TF32 by default).  For most cases the floor is below 0.87e-3 and the bar is the north star's 1e-3; where the
reference's own GPU arithmetic is already further than 1e-3 from strict fp32 (tiny_cond: 1.2e-3) no 10-bit-operand
implementation can do better, and the test says so instead of hiding it behind a loose constant.
Per denoising step (x_{t-1}) the 1e-3 bar is met with a wide margin: tests/test_gpu_sampler.py."""
import ctypes
import json

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


def _bar(floor):
    return min(max(NORTH_STAR, 1.15 * floor), HARD_CAP)


def _load(cfg, sd):
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(sd)
    return net.cuda()


def _check(name, got, ref, cfg, sd, x, t, c):
    floor = PM.rel(PM.forward(cfg, sd, x, t, c, PM.TF32_CLASS), ref)
    err = G.report(name, got, ref)
    print(f"[parity] {name}: eps rel {err:.3e}  TF32-class floor {floor:.3e}  bar {_bar(floor):.3e}")
    assert err <= _bar(floor), f"{name}: eps rel {err:.3e} > bar {_bar(floor):.3e} (floor {floor:.3e})"
    return err, floor


@pytest.mark.parametrize("tag", ["tiny", "tiny_cond", "tiny_sr"])
def test_tiny_unet_vs_reference_golden(golden, tag):
    cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    net = _load(cfg, sd)
    x = torch.from_numpy(golden[f"{tag}_x"]); t = torch.from_numpy(golden[f"{tag}_t"]); c = torch.from_numpy(golden[f"{tag}_classes"])
    _check(f"{tag} unet eps (classes)", net(x.cuda(), t.cuda(), c.cuda()), torch.from_numpy(golden[f"{tag}_eps"]), cfg, sd, x, t, c)
    _check(f"{tag} unet eps (None)", net(x.cuda(), t.cuda(), None), torch.from_numpy(golden[f"{tag}_eps_none"]), cfg, sd, x, t, None)
    # determinism: same inputs, same bits (eager first call, CUDA-graph replays afterwards)
    a = net(x.cuda(), t.cuda(), c.cuda())
    assert torch.equal(a, net(x.cuda(), t.cuda(), c.cuda())) and torch.equal(a, net(x.cuda(), t.cuda(), c.cuda()))


def test_eps_seeds_and_timesteps_fp32_tiny(golden):
    """use_fp16=False config, 3 weight/input seeds x t in {999, 500, 37}: every case within its bar."""
    cfg = json.loads(bytes(golden["tiny_cfg"]).decode())
    assert not cfg["use_fp16"]
    worst = 0.0
    for seed in (1234, 99, 7):
        sd = unet_ref.make_synthetic_state_dict(cfg, seed=seed)
        net = _load(cfg, sd)
        rng = np.random.default_rng(seed)
        x = torch.from_numpy(rng.standard_normal((2, 4, 32, 32)).astype(np.float32))
        c = torch.tensor([4, -1])
        for tt in (999, 500, 37):
            t = torch.tensor([tt, tt])
            ref = unet_ref.unet_forward(cfg, sd, x, t, c)
            err, _ = _check(f"tiny seed{seed} t={tt}", net(x.cuda(), t.cuda(), c.cuda()), ref, cfg, sd, x, t, c)
            worst = max(worst, err)
    print(f"[parity] tiny fp32, 3 seeds x 3 timesteps: worst eps rel {worst:.3e}")


@pytest.mark.parametrize("name,N", [("rgbd_singlecategory_adm_128_small", 1), ("rgbd_imagenet_adm_128_large_cfg", 2),
                                    ("rgbd_imagenet_adm_128_large_cond", 1), ("rgbd_imagenet_adm_256_128_small_sr", 1)])
def test_real_config_vs_oracle(golden, name, N):
    cfg = json.loads(bytes(golden[f"schemacfg_{name}"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    net = _load(cfg, sd)
    rng = np.random.default_rng(11)
    S = cfg["image_size"]
    x = torch.from_numpy(rng.standard_normal((N, cfg["in_channels"], S, S)).astype(np.float32))
    t = torch.tensor([999, 37][:N])
    c = torch.tensor([3, -1][:N]) if cfg.get("num_classes") else None
    ref = unet_ref.unet_forward(cfg, sd, x, t, c)
    got = net(x.cuda(), t.cuda(), c.cuda() if c is not None else None)
    _check(f"{name} N={N} eps", got, ref, cfg, sd, x, t, c)


def test_large_fp32_config_three_timesteps(golden):
    """The headline model (rgbd_imagenet_adm_128_large_cfg, use_fp16=False) at t in {999, 500, 37}, fresh input seed each."""
    cfg = json.loads(bytes(golden["schemacfg_rgbd_imagenet_adm_128_large_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    net = _load(cfg, sd)
    for seed, tt in ((21, 999), (22, 500), (23, 37)):
        rng = np.random.default_rng(seed)
        x = torch.from_numpy(rng.standard_normal((1, 4, 128, 128)).astype(np.float32))
        t = torch.tensor([tt]); c = torch.tensor([seed])
        ref = unet_ref.unet_forward(cfg, sd, x, t, c)
        _check(f"large seed{seed} t={tt}", net(x.cuda(), t.cuda(), c.cuda()), ref, cfg, sd, x, t, c)


def _tap(net, N, name):
    L = _lib.lib()
    C, H, W = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), None, 0, ctypes.byref(C), ctypes.byref(H), ctypes.byref(W)))
    out = torch.empty((N, C.value, H.value, W.value), dtype=torch.float32)
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), _lib.ptr(out), out.numel(), None, None, None))
    return out


@pytest.mark.parametrize("which", ["tiny", "large"])
def test_layerwise_taps(golden, which):
    """Per-layer drift: the output of EVERY ResBlock / AttentionBlock / the stem against the oracle's taps.  Shows where the
    eps error is accumulated (it grows smoothly along the depth: no single layer is off) and pins each block on its own."""
    key = "tiny_cfg" if which == "tiny" else "schemacfg_rgbd_imagenet_adm_128_large_cfg"
    cfg = json.loads(bytes(golden[key]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=99 if which == "tiny" else 1234)
    net = _load(cfg, sd)
    S = cfg["image_size"]
    rng = np.random.default_rng(3)
    x = torch.from_numpy(rng.standard_normal((1, 4, S, S)).astype(np.float32))
    t = torch.tensor([250]); c = torch.tensor([4])
    taps = {}
    ref = unet_ref.unet_forward(cfg, sd, x, t, c, taps=taps)
    got = net(x.cuda(), t.cuda(), c.cuda())
    worst, worst_name = 0.0, ""
    for name, want in taps.items():
        if name == "emb":
            continue
        r = G.rel(_tap(net, 1, name), want)
        print(f"[tap] {which:5s} {name:24s} {tuple(want.shape)!s:22s} rel {r:.3e}")
        if r > worst:
            worst, worst_name = r, name
    # PosEncoding -> time_embed (+ label_emb, null class -> zeros) is fp32 end to end (adm.py:11-33,357-365,545-555)
    r_emb = G.rel(_tap(net, 1, "emb")[:, :, 0, 0], taps["emb"])
    print(f"[tap] {which:5s} emb (time + class embedding) rel {r_emb:.3e}")
    assert r_emb < 2e-6
    # the stem carries a two-term split of x and W: it must be far inside fp16 precision
    assert G.rel(_tap(net, 1, "input_blocks.0.0"), taps["input_blocks.0.0"]) < 2e-5
    assert worst < 1.2e-3, f"layer {worst_name} is {worst:.3e} from the oracle"
    _check(f"{which} taps run eps", got, ref, cfg, sd, x, t, c)


def test_embeddings_and_film_table_fp32(golden):
    """PosEncoding / time_embed / label_emb incl. the null class, and the stacked emb_layers ("FiLM table") of every ResBlock,
    against the oracle in fp32 (SURVEY 8a row 6)."""
    import torch.nn.functional as F
    cfg = json.loads(bytes(golden["tiny_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    net = _load(cfg, sd)
    x = torch.zeros(3, 4, 32, 32)
    t = torch.tensor([999, 0, 421]); c = torch.tensor([9, -1, 0])
    taps = {}
    unet_ref.unet_forward(cfg, sd, x, t, c, taps=taps)
    net(x.cuda(), t.cuda(), c.cuda())
    emb = _tap(net, 3, "emb")[:, :, 0, 0]
    assert G.report("emb [N, 4*mc] (t = 999 / 0 / 421, classes 9 / null / 0)", emb, taps["emb"]) < 2e-6
    blocks, _ = unet_ref._topology(cfg)
    want = torch.cat([F.linear(F.silu(taps["emb"]), sd[l[1] + ".emb_layers.1.weight"], sd[l[1] + ".emb_layers.1.bias"])
                      for b in blocks for l in b["layers"] if l[0] == "res"], dim=1)
    film = _tap(net, 3, "film")[:, :, 0, 0]
    assert film.shape == want.shape
    assert G.report("FiLM table (all emb_layers stacked)", film, want) < 5e-6
    # classes=None: zero class embedding (adm.py:554-555)
    unet_ref.unet_forward(cfg, sd, x, t, None, taps=taps)
    net(x.cuda(), t.cuda(), None)
    assert G.report("emb, classes=None", _tap(net, 3, "emb")[:, :, 0, 0], taps["emb"]) < 2e-6


def test_large_model_batch32_deterministic_and_batch_invariant(golden):
    """Size-independent properties at the benchmark batch (CFG batch 32 of the large model, every SM busy): the forward is bitwise
    reproducible run to run (eager first call, then CUDA-graph replays) and a sample's eps does not depend on the batch it is
    computed in (same bits alone and inside the batch of 32).  Regression test for the attention barrier alias fixed in round 2
    (one launch in ten returned a few wrong 32-row groups, eps off by 5e-4 relative)."""
    cfg = json.loads(bytes(golden["schemacfg_rgbd_imagenet_adm_128_large_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    net = _load(cfg, sd)
    N = 32
    g = torch.Generator().manual_seed(3)
    x = torch.randn(N, 4, 128, 128, generator=g).cuda()
    t = torch.full((N,), 500, device="cuda"); c = torch.arange(N, device="cuda") % 1000
    first = net(x, t, c).clone()
    bad = sum(0 if torch.equal(net(x, t, c), first) else 1 for _ in range(40))
    assert bad == 0, f"{bad} of 40 forwards differ from the first"
    for i in (0, 13, 31):
        one = net(x[i:i + 1].contiguous(), t[i:i + 1], c[i:i + 1])
        assert torch.equal(one, first[i:i + 1]), f"sample {i}: eps depends on the batch"


@pytest.mark.parametrize("tag", ["noshift", "plainconv", "plainpool"])
def test_backbone_options(tag):
    """Backbone options no shipped config sets, against the unmodified reference's eps (options_golden.npz) and the oracle's
    per-block taps.
      noshift    use_scale_shift_norm=False (adm.py:219-221): the embedding is ADDED before out_layers' GroupNorm; the plan derives
                 the moments of h + e from the per-channel statistics of the conv epilogue and folds e into the apply affine
      plainconv  resblock_updown=False, conv_resample=True: Downsample2d = 3x3 stride-2 conv (im2col + 1x1 GEMM over 9C),
                 Upsample2d = nearest 2x + 3x3 conv (adm.py:60-117)
      plainpool  resblock_updown=False, conv_resample=False (+ use_scale_shift_norm=False): AvgPool2d(2) / nearest 2x"""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "options_golden.npz"))
    cfg = json.loads(bytes(g[f"{tag}_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    net = _load(cfg, sd)
    x = torch.from_numpy(g[f"{tag}_x"]); t = torch.from_numpy(g[f"{tag}_t"]); c = torch.from_numpy(g[f"{tag}_c"])
    got = net(x.cuda(), t.cuda(), c.cuda())
    r = G.report(f"eps, {tag}", got, torch.from_numpy(g[f"{tag}_eps"]))
    assert r < HARD_CAP
    taps = {}
    unet_ref.unet_forward(cfg, sd, x, t, c, taps=taps)
    blocks, _ = unet_ref._topology(cfg)
    names = [l[1] for b in blocks for l in b["layers"] if l[0] in ("res", "attn", "down", "up")]
    worst = 0.0
    for name in names:
        rt = G.rel(_tap(net, 2, name), taps[name])
        worst = max(worst, rt)
        print(f"[{tag}] {name} rel {rt:.3e}")
    assert worst < HARD_CAP


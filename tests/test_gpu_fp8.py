"""GPU: the fp8 (e4m3) precision mode of the ResBlock convs (AdmUnet2d.set_precision("fp8"), DESIGN.md §2).

The conv kernel's A8 instantiations and the gn_apply e4m3 output against float64 emulations of exactly what they are
specified to compute; whole forwards against the fp32 oracle at 1.15 x the fp8 emulation's own distance
(tests/precision_model_fp8.py); the
bitwise properties of the plan in fp8 mode; mode toggling; and which convs run e4m3."""
import ctypes
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
import precision_model as PM
import precision_model_fp8 as P8
from ivid_b200 import _lib
from oracle import unet_ref

pytestmark = pytest.mark.gpu


def _e4m3(t):
    return t.clamp(-448.0, 448.0).to(torch.float8_e4m3fn)


def _conv8(a8, w, b, k, act2=None, w2=None, b2=None, residual=None, out_fp16=False):
    N, H, W, Cin = a8.shape
    Cout = w.shape[0]
    out = torch.empty((N, H, W, Cout), dtype=torch.float16 if out_fp16 else torch.float32, device="cuda")
    wc = w.float().contiguous(); bc = b.float().contiguous()
    w2c = w2.float().contiguous() if w2 is not None else None
    b2c = b2.float().contiguous() if b2 is not None else None
    e = ctypes.c_int()
    _lib.check(_lib.lib().ivid_op_conv2d_e4m3(_lib.ptr(a8), N, H, W, Cin, _lib.ptr(wc), _lib.ptr(bc), Cout, k,
                                              _lib.ptr(act2), act2.shape[-1] if act2 is not None else 0, _lib.ptr(w2c),
                                              _lib.ptr(b2c), _lib.ptr(residual), _lib.ptr(out), 1 if out_fp16 else 0,
                                              ctypes.byref(e), _lib.cur_stream()))
    return out, e.value


def _emulate(a8, w, b, k, e, act2=None, w2=None, b2=None, residual=None):
    """float64: dequantized e4m3 operands x 2^-e, plus the fp16 skip terms with weights fp16(w2 * 2^e) * 2^-e."""
    a = a8.float().double().permute(0, 3, 1, 2).cpu()
    wq = _e4m3(w * 2.0 ** e).float().double() * 2.0 ** -e
    y = F.conv2d(a, wq, b.double(), padding=k // 2)
    if act2 is not None:
        w2q = (w2 * 2.0 ** e).half().double() * 2.0 ** -e
        y = y + F.conv2d(act2.double().permute(0, 3, 1, 2).cpu(), w2q.reshape(w2.shape[0], -1, 1, 1), b2.double())
    if residual is not None:
        y = y + residual.double().permute(0, 3, 1, 2).cpu()
    return y.permute(0, 2, 3, 1)


# tag, N, H (= W), Cin, Cout, k, Cin2 (1x1 fp16 skip segment), residual, out_fp16
CONV_CASES = [
    ("128^2 3x3 256->256 fp16 out", 2, 128, 256, 256, 3, 0, False, True),
    ("128^2 3x3 256 + skip 512 -> 256", 2, 128, 256, 256, 3, 512, False, False),
    ("128^2 3x3 256->256 residual", 2, 128, 256, 256, 3, 0, True, False),
    ("64^2 3x3 256->256", 2, 64, 256, 256, 3, 0, False, False),
    ("32^2 3x3 512->512", 2, 32, 512, 512, 3, 0, False, False),
    ("16^2 3x3 768->768", 2, 16, 768, 768, 3, 0, False, False),
    ("8^2 3x3 1024->1024, batch tail", 3, 8, 1024, 1024, 3, 0, False, False),
    ("32^2 3x3 96->128 (padded chunk)", 2, 32, 96, 128, 3, 0, False, False),
    ("32^2 3x3 160->192 (two chunks, padded)", 2, 32, 160, 192, 3, 0, False, False),
    ("16^2 1x1 128->64 (one k-block)", 2, 16, 128, 64, 1, 0, False, False),
    ("16^2 1x1 256->64 (two k-blocks)", 2, 16, 256, 64, 1, 0, False, False),
    ("16^2 3x3 48->40 (BN 16), skip 40, residual", 5, 16, 48, 40, 3, 40, True, False),
    ("32^2 3x3 160 + skip 96 -> 160, residual, fp16 out", 2, 32, 160, 160, 3, 96, True, True),
]


# Hopper's fp8 wgmma does not accumulate at full fp32 precision (the product sums are truncated inside the instruction), so
# the kernel differs from the float64 emulation by more than summation order: measured 1.2e-4 at K = 128, 7.6e-4 at K = 2304
# and 2.0e-3 at K = 9216 (relative L2, H100).  That is 30x below the e4m3 operand rounding the mode introduces (the
# forward tests below compare the whole network against an emulation that rounds operands only, within 1.15x).
CONV_BAR = 3e-3


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_e4m3_vs_float64_emulation(case):
    tag, N, H, Cin, Cout, k, Cin2, res, out16 = case
    g = torch.Generator().manual_seed(sum(map(ord, tag)))
    a8 = _e4m3(torch.randn(N, H, H, Cin, generator=g) * 1.5).cuda()
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    act2 = torch.randn(N, H, H, Cin2, generator=g).half().cuda() if Cin2 else None
    w2 = torch.randn(Cout, Cin2, generator=g) / max(Cin2, 1) ** 0.5 if Cin2 else None
    b2 = torch.randn(Cout, generator=g) * 0.1 if Cin2 else None
    r = torch.randn(N, H, H, Cout, generator=g).cuda() if res else None
    got, e = _conv8(a8, w, b, k, act2, w2, b2, r, out16)
    assert 224 < float(w.abs().max()) * 2.0 ** e <= 448
    want = _emulate(a8, w, b, k, e, act2, w2, b2, r)
    err = G.report(f"conv e4m3 {tag}", got.float(), want)
    assert err < CONV_BAR


def test_conv_e4m3_rejects_unaligned_channels():
    a8 = torch.zeros(1, 16, 16, 40, dtype=torch.uint8, device="cuda")
    out = torch.empty(1, 16, 16, 64, device="cuda")
    w = torch.zeros(64, 40, 3, 3); b = torch.zeros(64)
    rc = _lib.lib().ivid_op_conv2d_e4m3(_lib.ptr(a8), 1, 16, 16, 40, _lib.ptr(w), _lib.ptr(b), 64, 3, None, 0, None, None, None,
                                        _lib.ptr(out), 0, None, _lib.cur_stream())
    assert rc == _lib.IVID_ERR_INVALID_ARGUMENT


def _ulp_codes(q):
    """e4m3 bytes -> integers ordered like the values (adjacent representable values differ by 1)."""
    q = q.view(torch.uint8).to(torch.int32)
    mag = q & 0x7F
    return torch.where(q >= 128, -mag, mag)


@pytest.mark.parametrize("mode,C0,C1,gain", [(0, 256, 0, 1.0), (0, 192, 128, 1.0), (1, 128, 0, 1.0), (2, 256, 0, 1.0),
                                             (0, 128, 0, 400.0)])
def test_group_norm_e4m3_vs_emulation(mode, C0, C1, gain):
    N, H, W, groups = 2, 32, 32, 32
    g = torch.Generator().manual_seed(C0 + C1 + mode)
    x0 = (torch.randn(N, H, W, C0, generator=g) * 2 + 0.3).cuda()
    x1 = (torch.randn(N, H, W, C1, generator=g) - 0.2).cuda() if C1 else None
    C = C0 + C1
    gamma = (torch.rand(C, generator=g) + 0.5) * gain
    beta = torch.randn(C, generator=g) * 0.2
    film = torch.randn(N, 2 * C, generator=g).cuda() * 0.3
    Ho, Wo = (H * 2, W * 2) if mode == 1 else ((H // 2, W // 2) if mode == 2 else (H, W))
    out = torch.empty(N, Ho, Wo, C, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib().ivid_op_group_norm_e4m3(_lib.ptr(x0), C0, _lib.ptr(x1), C1, N, H, W, groups, 1e-5, _lib.ptr(gamma),
                                                  _lib.ptr(beta), _lib.ptr(film), 1, mode, _lib.ptr(out), _lib.cur_stream()))
    x = torch.cat([x0, x1], -1) if C1 else x0
    x = x.double().permute(0, 3, 1, 2).cpu()
    f = film.double().cpu()
    y = F.group_norm(x, groups, gamma.double(), beta.double(), 1e-5) * (1 + f[:, :C, None, None]) + f[:, C:, None, None]
    y = F.silu(y)
    if mode == 1:
        y = F.interpolate(y, scale_factor=2, mode="nearest")
    elif mode == 2:
        y = F.avg_pool2d(y, 2)
    want = _e4m3(y.permute(0, 2, 3, 1).float())
    d = (_ulp_codes(out.cpu()) - _ulp_codes(want)).abs()
    n1 = int((d == 1).sum())
    print(f"[fp8] gn_apply e4m3 mode {mode} C {C0}+{C1} gamma x{gain}: max ulp {int(d.max())}, off by one ulp {n1} of {d.numel()}, "
          f"saturated {int(((out.cpu() & 0x7F) == 0x7E).sum())}")
    assert int(d.max()) <= 1 and n1 < 1e-3 * d.numel()
    if gain > 100:
        assert int(((out.cpu() & 0x7F) == 0x7E).sum()) > 0, "the large-gamma case saturates"


def _net(cfg, sd, precision="fp8"):
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(sd)
    net = net.cuda()
    net.set_precision(precision)
    return net


def _forward_case(name, cfg, sd, x, t, c):
    net = _net(cfg, sd)
    got = net(x.cuda(), t.cuda(), c.cuda() if c is not None else None)
    ref = unet_ref.unet_forward(cfg, sd, x, t, c)
    floor = PM.rel(P8.forward(cfg, sd, x, t, c), ref)
    err = G.report(f"{name} fp8 eps", got, ref)
    print(f"[fp8] {name}: eps rel to fp32 {err:.3e}, fp8 emulation {floor:.3e}, bar {1.15 * floor:.3e}")
    assert torch.isfinite(got).all()
    assert err <= 1.15 * floor


@pytest.mark.parametrize("tag", ["tiny", "tiny_cond", "tiny_sr"])
def test_forward_fp8_vs_oracle_tiny(golden, tag):
    cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    x = torch.from_numpy(golden[f"{tag}_x"]); t = torch.from_numpy(golden[f"{tag}_t"]); c = torch.from_numpy(golden[f"{tag}_classes"])
    _forward_case(tag, cfg, sd, x, t, c)


def test_forward_fp8_vs_oracle_large(golden):
    cfg = json.loads(bytes(golden["schemacfg_rgbd_imagenet_adm_128_large_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    rng = np.random.default_rng(11)
    x = torch.from_numpy(rng.standard_normal((2, 4, 128, 128)).astype(np.float32))
    _forward_case("large N=2", cfg, sd, x, torch.tensor([999, 37]), torch.tensor([3, -1]))


def test_fp8_bitwise_properties(golden):
    """Run to run, batch invariance at batch 32, and the fused head step == the separate step route (DDIM, DPM-Solver++)."""
    cfg = json.loads(bytes(golden["schemacfg_rgbd_imagenet_adm_128_large_cfg"]).decode())
    net = _net(cfg, unet_ref.make_synthetic_state_dict(cfg, seed=1234))
    N = 32
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(N, 4, 128, 128, generator=gen).cuda()
    t = torch.full((N,), 500, device="cuda"); c = torch.arange(N, device="cuda") % 1000
    first = net(x, t, c).clone()
    assert all(torch.equal(net(x, t, c), first) for _ in range(5))
    for i in (0, 31):
        assert torch.equal(net(x[i:i + 1].contiguous(), t[i:i + 1], c[i:i + 1]), first[i:i + 1]), f"sample {i} depends on the batch"
    tcfg = json.loads(bytes(golden["tiny_cfg"]).decode())
    fw = frameworks.ClassifierFreeGuidance(_net(tcfg, unet_ref.make_synthetic_state_dict(tcfg, seed=1234)), timesteps=1000,
                                           beta_schedule="linear")
    xs = torch.from_numpy(np.random.default_rng(2).standard_normal((2, 4, 32, 32)).astype(np.float32)).cuda()
    cls = torch.tensor([1, 2]).cuda()
    for S in (samplers.DdimSampler, samplers.DpmSolverSampler):
        s = S(fw)
        a = s.sample(2, noise=xs, classes=cls, steps=8, strength=0.5, verbose=False).samples
        b = s.sample(2, noise=xs, classes=cls, steps=8, strength=0.5, verbose=False, return_trajectory=True).samples
        assert torch.isfinite(a).all() and torch.equal(a, b), f"{S.__name__}: fused and separate routes differ in fp8 mode"


def test_precision_toggle_restores_fp16_bits(golden):
    cfg = json.loads(bytes(golden["tiny_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    x = torch.from_numpy(golden["tiny_x"]).cuda(); t = torch.from_numpy(golden["tiny_t"]).cuda()
    c = torch.from_numpy(golden["tiny_classes"]).cuda()
    plain = _net(cfg, sd, "fp16")
    want = plain(x, t, c).clone()
    net = _net(cfg, sd, "fp16")
    assert torch.equal(net(x, t, c), want)
    net.set_precision("fp8")
    e8 = net(x, t, c).clone()
    assert not torch.equal(e8, want)
    net.set_precision("fp16")
    assert torch.equal(net(x, t, c), want)


def _profile_families(net, x, t, c):
    L = _lib.lib()
    net(x, t, c)
    torch.cuda.synchronize()
    _lib.check(L.ivid_unet_profile_begin(net._handle))
    net(x, t, c)
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(L.ivid_unet_profile_end(net._handle, buf, len(buf)))
    return json.loads(buf.value.decode())


def _e4m3_launches(fam):
    return sum(v["launches"] for k, v in fam.items() if k.startswith("conv_gemm<") and k.endswith(",e4m3>"))


def _resblock_conv_inputs(net):
    sd = net.state_dict()
    return [int(v.shape[1]) for k, v in sd.items() if k.endswith((".in_layers.2.weight", ".out_layers.3.weight"))]


def test_fp8_coverage():
    import bench
    net = _net(bench.MODELS["L"], unet_ref.make_synthetic_state_dict(bench.MODELS["L"], seed=1234))
    x = torch.randn(2, 4, 128, 128, device="cuda"); t = torch.tensor([500, 10], device="cuda"); c = torch.tensor([1, 2], device="cuda")
    fam = _profile_families(net, x, t, c)
    n_res = len(_resblock_conv_inputs(net))
    print(f"[fp8] config-2 families: " + ", ".join(f"{k} {v['launches']}" for k, v in sorted(fam.items()) if k.startswith("conv")))
    assert _e4m3_launches(fam) == n_res
    # widths 40 (not a multiple of 16) and 128; up-path concatenations 256, 168 (not a multiple of 16) and 80
    cfg = dict(image_size=32, in_channels=4, model_channels=40, out_channels=4, num_res_blocks=1, attention_resolutions=[],
               channel_mult=[1, 3.2], num_groups=8, num_head_channels=64)
    net = _net(cfg, unet_ref.make_synthetic_state_dict(cfg, seed=5))
    x = torch.randn(2, 4, 32, 32, device="cuda"); t = torch.tensor([500, 10], device="cuda")
    fam = _profile_families(net, x, t, None)
    widths = _resblock_conv_inputs(net)
    want = sum(1 for w in widths if w % 16 == 0)
    print(f"[fp8] widths-40 net: ResBlock conv inputs {widths}, e4m3 launches {_e4m3_launches(fam)} (expected {want})")
    assert 0 < want < len(widths) and _e4m3_launches(fam) == want


def test_skip_range_fallback_runs_fp16(golden):
    """A conv whose skip weights are > 300 x its 3x3 weights would overflow fp16 once scaled (300 > 65504 / 224): it stays
    fp16.  The e4m3 family loses exactly those convs, and the net stays within the bar of the fp8 emulation that keeps
    them fp16."""
    cfg = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1, attention_resolutions=[],
               channel_mult=[1, 2], num_groups=32)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=9)
    for k in list(sd):
        if k.endswith(".skip_connection.weight"):
            w3 = k.replace("skip_connection", "out_layers.3")
            sd[w3] = sd[w3] * (float(sd[k].abs().max()) / (400.0 * float(sd[w3].abs().max())))
    x = torch.randn(2, 4, 32, 32, device="cuda"); t = torch.tensor([500, 10], device="cuda")
    n8 = _net(cfg, sd, "fp8")
    fam = _profile_families(n8, x, t, None)
    n_skip = sum(1 for k in sd if k.endswith(".skip_connection.weight"))
    assert n_skip > 0 and _e4m3_launches(fam) == len(_resblock_conv_inputs(n8)) - n_skip
    ref = unet_ref.unet_forward(cfg, sd, x.cpu(), t.cpu(), None)
    got = n8(x, t, None)
    floor = PM.rel(P8.forward(cfg, sd, x.cpu(), t.cpu(), None), ref)
    err = G.report("skip-fallback net fp8 eps", got, ref)
    print(f"[fp8] skip-fallback net: eps rel {err:.3e}, fp8 emulation {floor:.3e}")
    assert err <= 1.15 * floor

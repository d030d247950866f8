"""GPU: the network's two ends and its embedding path against float64, per element (bounds: tests/network_ends_model.py).

  a/b  the stem: the packed two-term split of the network input, unconditional at in_channels 4, 3 and 7 and with the
       inpaint / super-resolution inputs assembled in cond_pack_kernel, read through the stem tap;
  c    the output head: GroupNorm from the block's fp16 copy, the split 1x1 GEMM over 9 * Co tap columns and the tap
       shift-and-add, or the fp16 conv for out_channels > 7, read as eps; with IVID_NO_OUTSPLIT the split bound must fail;
  d    the time / class embedding and the FiLM table at N = 1 ... 65, through every embedding kernel a network reaches;
  e    forwards of more than 32 rows: a sample's eps is the same bits alone and inside the batch.

Where a rounding is coherent it is made coherent (positive stem and out.2 weights and inputs just off the fp16 grid), so
a dropped split term moves every element.  Each case prints the worst |got - ref| / bound and where it is."""
import ctypes

import pytest
import torch

import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
import network_ends_model as NM
from ivid_b200 import _lib
from oracle import sampler_ref, unet_ref

pytestmark = pytest.mark.gpu
CFGS = NM.golden_cfgs()
T = 1000


def _net(cfg, sd):
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(sd)
    net = net.cuda()
    net._ensure_packed()
    return net


_LARGE = {}


def _large():
    """The large model (256 channels, FiLM table 40960 wide) is built once for the tests that use it."""
    if not _LARGE:
        cfg = CFGS["large"]
        sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
        _LARGE.update(cfg=cfg, sd=sd, net=_net(cfg, sd))
    return _LARGE["cfg"], _LARGE["sd"], _LARGE["net"]


def _forward(net, x, N, t, classes, cond=None, out_channels=4):
    """ivid_unet_forward_hw over N rows; row n reads x[n % Nx] (and the conditional inputs of that sample)."""
    H, W = x.shape[-2:]
    eps = torch.empty((N, out_channels, H, W), device="cuda")
    c = ctypes.byref(cond) if cond is not None else None
    _lib.check(_lib.lib().ivid_unet_forward_hw(net._handle, _lib.ptr(x), x.shape[0], H, W, c, _lib.ptr(t), _lib.ptr(classes),
                                               _lib.ptr(eps), N, _lib.cur_stream()))
    torch.cuda.synchronize()
    return eps


def _tap(net, N, name):
    L = _lib.lib()
    C, H, W = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), None, 0, ctypes.byref(C), ctypes.byref(H), ctypes.byref(W)))
    out = torch.empty((N, C.value, H.value, W.value), dtype=torch.float32)
    _lib.check(L.ivid_unet_debug_tap(net._handle, N, name.encode(), _lib.ptr(out), out.numel(), None, None, None))
    return out


def _report(family, case, got, ref, bound):
    r, at = NM.worst(got, ref, bound)
    print(f"[ends] {family:10s} {case:34s} worst |got - ref| / bound {r:.3e} at {at}")
    assert r <= 1.0, f"{family} {case}: {r:.3e} x the bound at {at}"
    return r


def _guided(N, t, classes):
    """t and classes of a guidance forward over 2N rows: rows n + N are the unconditional halves (null class)."""
    return torch.cat([t, t]), torch.cat([classes, torch.full_like(classes, -1)])


# ----------------------------------------------------------------------------------------------------------------------
# a. stem, unconditional
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cin", [4, 3, 7])
def test_stem_unconditional(cin):
    """in_channels 3 and 7 make the hi | lo | hi segments straddle the kernel's 8-channel store groups.  The batch-2 guidance
    forward reads x[n % 1] for both rows: their stem outputs are the same bits."""
    cfg = dict(CFGS["tiny"], in_channels=cin)
    sd = NM.coherent_state_dict(cfg)
    net = _net(cfg, sd)
    x = NM.stem_input(1, cin, 32, 32, seed=cin)
    w, b = sd["input_blocks.0.0.weight"], sd["input_blocks.0.0.bias"]
    ref, S = NM.stem_reference(x, w, b)
    bound = NM.stem_bound(S, w, b)
    t, c = torch.tensor([500], device="cuda"), torch.tensor([3], device="cuda")
    _forward(net, x.cuda(), 1, t, c)
    _report("stem", f"Cin={cin} N=1", _tap(net, 1, "input_blocks.0.0"), ref, bound)
    tg, cg = _guided(1, t, c)
    _forward(net, x.cuda(), 2, tg, cg)
    two = _tap(net, 2, "input_blocks.0.0")
    assert torch.equal(two[0], two[1]), "the two guidance rows of one sample differ at the stem"
    _report("stem", f"Cin={cin} guided 2 rows", two, ref.expand(2, -1, -1, -1), bound.expand(2, -1, -1, -1))


# ----------------------------------------------------------------------------------------------------------------------
# b. stem, conditional inputs
# ----------------------------------------------------------------------------------------------------------------------
def _mask(N, H, W, seed, band_rows):
    """Mostly 0 / 1, with a band of rows of fractional values."""
    g = torch.Generator().manual_seed(seed)
    m = (torch.rand(N, 1, H, W, generator=g) > 0.5).float()
    m[:, :, band_rows] = torch.rand(N, 1, len(range(H)[band_rows]), W, generator=g)
    return m


def _cond_stem(cfg, x, xin, delta, cond, Nx, case):
    """Forward N = 2 Nx rows (row n reads sample n % Nx) and check the stem of every row against the reference of its
    sample; rows n and n + Nx are the same bits."""
    sd = NM.coherent_state_dict(cfg)
    net = _net(cfg, sd)
    w, b = sd["input_blocks.0.0.weight"], sd["input_blocks.0.0.bias"]
    ref, S = NM.stem_reference(xin, w, b)
    bound = NM.stem_bound(S, w, b, delta)
    t = torch.full((Nx,), 500, device="cuda")
    c = torch.arange(Nx, device="cuda") % cfg["num_classes"]
    tg, cg = _guided(Nx, t, c)
    _forward(net, x.cuda(), 2 * Nx, tg, cg, cond=cond)
    got = _tap(net, 2 * Nx, "input_blocks.0.0")
    assert torch.equal(got[:Nx], got[Nx:]), f"{case}: rows n and n + Nx differ at the stem"
    return _report("cond stem", case, got, torch.cat([ref, ref]), torch.cat([bound, bound]))


@pytest.mark.parametrize("mask_rgb", [True, False], ids=["10ch_mask_rgb", "9ch"])
def test_stem_inpaint(mask_rgb):
    N, H, W = 2, 32, 32
    cfg = dict(CFGS["tiny_cond"], in_channels=10 if mask_rgb else 9)
    x, y, z = (NM.stem_input(N, 4, H, W, seed=s) for s in (10, 11, 12))
    m = _mask(N, H, W, 13, slice(8, 14))
    mr = _mask(N, H, W, 14, slice(20, 23)) if mask_rgb else None
    xin = sampler_ref.make_inpaint_inputs(x, y, m, mr, z[:, :3], z[:, 3:])
    delta = NM.cond_delta("inpaint", x, y, m, mr, z)
    dev = [v.cuda() for v in (y, m, z)] + ([mr.cuda()] if mask_rgb else [])
    cond = _lib.CondT(kind=1, y_dev=dev[0].data_ptr(), mask_dev=dev[1].data_ptr(),
                      mask_rgb_dev=dev[3].data_ptr() if mask_rgb else None, noise_dev=dev[2].data_ptr())
    _cond_stem(cfg, x, xin, delta, cond, N, f"inpaint {'10' if mask_rgb else '9'} channels")


@pytest.mark.parametrize("scale,H,W", [(2, 32, 32), (3, 24, 36), (4, 32, 32), (4, 8, 4)])
def test_stem_superres(scale, H, W):
    """Scales 2, 3 and 4; 24x36 is non-square; at 8x4 / 4 the low-resolution input is 2x1, so the bilinear stencil is
    clamped at both borders of both axes."""
    N = 2
    cfg = CFGS["tiny_sr"]
    x = NM.stem_input(N, 4, H, W, seed=20 + scale)
    y = torch.randn(N, 4, H // scale, W // scale, generator=torch.Generator().manual_seed(30 + scale))
    xin = sampler_ref.make_sr_inputs(x, y)
    delta = NM.cond_delta("sr", x, y)
    yd = y.cuda()
    cond = _lib.CondT(kind=2, y_dev=yd.data_ptr(), sr_scale=scale)
    _cond_stem(cfg, x, xin, delta, cond, N, f"super-res x{scale} {H}x{W}")


# ----------------------------------------------------------------------------------------------------------------------
# c. output head
# ----------------------------------------------------------------------------------------------------------------------
def _head(cfg, H, W):
    """eps of a forward, the float64 head of the GPU's own last block output, and the head's split and fp16 bounds."""
    sd = NM.coherent_state_dict(cfg)
    net = _net(cfg, sd)
    N = 2
    x = torch.randn(N, cfg["in_channels"], H, W, generator=torch.Generator().manual_seed(H * W)).cuda()
    t = torch.tensor([999, 37], device="cuda")
    c = torch.tensor([3, -1], device="cuda")
    eps = _forward(net, x, N, t, c, out_channels=cfg["out_channels"]).cpu()
    blocks, _ = unet_ref._topology(cfg)
    ref, y, dy = NM.head_reference(_tap(net, N, blocks[-1]["layers"][-1][1]), sd, cfg["num_groups"])
    w, b = sd["out.2.weight"], sd["out.2.bias"]
    return eps, ref, NM.head_bound(y, dy, w, b, split=True), NM.head_bound(y, dy, w, b, split=False)


HEAD_CASES = {
    "tiny 32x32": (CFGS["tiny"], 32, 32),
    "final width 96 (K pad 128)": (CFGS["mc96"], 32, 32),
    "two levels at 10x6": (dict(CFGS["tiny"], channel_mult=[1, 2]), 10, 6),
    "out_channels 3": (dict(CFGS["tiny"], out_channels=3), 32, 32),
}


@pytest.mark.parametrize("case", list(HEAD_CASES))
def test_head_split(case):
    cfg, H, W = HEAD_CASES[case]
    eps, ref, split, _ = _head(cfg, H, W)
    _report("head", case, eps, ref, split)


def test_head_unsplit_out_channels_8():
    """9 * 8 tap columns do not fit the split GEMM's 64: the head is conv_gemm<16> over fp16 y and W, and is held to the
    fp16 operand rounding."""
    eps, ref, _, fp16 = _head(dict(CFGS["tiny"], out_channels=8), 32, 32)
    _report("head fp16", "out_channels 8", eps, ref, fp16)


def test_head_without_split_fails_the_split_bound(monkeypatch):
    """IVID_NO_OUTSPLIT=1 on a fresh network runs the fp16 head: it meets the fp16 bound and exceeds the split one, so the
    split test can see the split."""
    monkeypatch.setenv("IVID_NO_OUTSPLIT", "1")
    eps, ref, split, fp16 = _head(CFGS["tiny"], 32, 32)
    r, at = NM.worst(eps, ref, split)
    print(f"[ends] head control IVID_NO_OUTSPLIT=1 against the split bound: worst ratio {r:.3e} at {at}")
    assert r > 1.0, "the fp16 head passes the split bound: the head test cannot see the split"
    _report("head fp16", "tiny, IVID_NO_OUTSPLIT=1", eps, ref, fp16)


# ----------------------------------------------------------------------------------------------------------------------
# d. embedding and FiLM table
# ----------------------------------------------------------------------------------------------------------------------
def _embed_inputs(cfg, N, with_classes):
    t = torch.tensor([0, 1, 500, T - 2, T - 1] * 14)[:N]
    if not with_classes:
        return t, None
    c = torch.arange(N) * 7 % cfg["num_classes"]
    c[1::3] = -1
    return t, c


@pytest.mark.parametrize("tag", ["tiny", "single", "large", "g8", "g4_40", "mc96"])
def test_embedding_and_film_table(tag):
    """emb and film taps against float64 at N = 1, 31, 32, 33, 65 (per-row t 0, 1, 500, T-2, T-1; real labels, the null
    class and classes=None).  tests/test_network_ends_model.py says which kernel each configuration reaches."""
    if tag == "large":
        cfg, sd, net = _large()
    else:
        cfg = CFGS[tag]
        sd = unet_ref.make_synthetic_state_dict(cfg, seed=7)
        net = _net(cfg, sd)
    side = 2 ** (len(cfg["channel_mult"]) - 1)          # the smallest input: the embedding does not depend on it
    worst_e = worst_f = 0.0
    for N in (1, 31, 32, 33, 65):
        for with_classes in ((True, False) if N in (33, 65) else (True,)):
            t, c = _embed_inputs(cfg, N, with_classes)
            x = torch.zeros(N, cfg["in_channels"], side, side, device="cuda")
            _forward(net, x, N, t.cuda(), c.cuda() if c is not None else None)
            emb = _tap(net, N, "emb")[:, :, 0, 0]
            ref, bound = NM.embedding_reference(cfg, sd, t, c)
            case = f"{tag} N={N}" + ("" if with_classes else " classes=None")
            worst_e = max(worst_e, _report("emb", case, emb, ref, bound))
            fref, fbound = NM.film_reference(cfg, sd, emb)
            worst_f = max(worst_f, _report("film", case, _tap(net, N, "film")[:, :, 0, 0], fref, fbound))
    print(f"[ends] {tag}: worst emb {worst_e:.3e}, worst film {worst_f:.3e}, kernels {NM.embedding_kernels(cfg)}")


# ----------------------------------------------------------------------------------------------------------------------
# e. more than 32 rows
# ----------------------------------------------------------------------------------------------------------------------
def _batch_net(tag):
    if tag == "large":
        return _large()
    cfg = CFGS[tag]
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    return cfg, sd, _net(cfg, sd)


@pytest.mark.parametrize("tag", ["tiny", "tiny_cond", "large"])
def test_batch_past_32_rows_is_bitwise_per_sample(tag):
    """N = 33 and 65, plain and with guidance (66 and 130 rows): rows 0, 31, 32 and N - 1 (and their guidance halves)
    have the bits of the same sample run alone."""
    cfg, sd, net = _batch_net(tag)
    H = W = 64 if tag == "large" else 32
    for N in (33, 65):
        g = torch.Generator().manual_seed(N)
        x = torch.randn(N, 4, H, W, generator=g).cuda()
        t = torch.tensor([0, 1, 500, T - 2, T - 1] * 14)[:N].cuda()
        c = (torch.arange(N) % cfg["num_classes"]).cuda()
        cond, parts = None, []
        if tag == "tiny_cond":
            parts = [torch.randn(N, 4, H, W, generator=g).cuda(), (torch.rand(N, 1, H, W, generator=g) > 0.5).float().cuda(),
                     (torch.rand(N, 1, H, W, generator=g) > 0.5).float().cuda(), torch.randn(N, 4, H, W, generator=g).cuda()]
        def cond_of(i=None):
            if not parts:
                return None
            p = [v[i:i + 1].contiguous() if i is not None else v for v in parts]
            cond_of.keep.append(p)
            return _lib.CondT(kind=1, y_dev=p[0].data_ptr(), mask_dev=p[1].data_ptr(), mask_rgb_dev=p[2].data_ptr(),
                              noise_dev=p[3].data_ptr())
        cond_of.keep = []
        for guided in (False, True):
            tt, cc = _guided(N, t, c) if guided else (t, c)
            rows = 2 * N if guided else N
            eps = _forward(net, x, rows, tt, cc, cond=cond_of()).clone()
            for i in (0, 31, 32, N - 1):
                ti, ci = t[i:i + 1], c[i:i + 1]
                if guided:
                    ti, ci = _guided(1, ti, ci)
                one = _forward(net, x[i:i + 1].contiguous(), 2 if guided else 1, ti, ci, cond=cond_of(i))
                assert torch.equal(one[0], eps[i]), f"{tag} N={N} guided={guided}: row {i} depends on the batch"
                if guided:
                    assert torch.equal(one[1], eps[N + i]), f"{tag} N={N}: unconditional row {N + i} depends on the batch"
            print(f"[ends] batch {tag} N={N} {'guided ' + str(rows) + ' rows' if guided else 'plain'}: rows 0, 31, 32, {N - 1} bitwise")


def test_ddim_sample_of_33_is_bitwise_per_sample():
    """A 10-step guided DDIM run of 33 samples (66-row forwards, the output head's fused step) equals each sample run alone
    at the same seed, from the same injected x_T."""
    cfg, sd, net = _batch_net("tiny")
    s = samplers.DdimSampler(frameworks.ClassifierFreeGuidance(net, timesteps=T, beta_schedule="linear"))
    N = 33
    x = torch.randn(N, 4, 32, 32, generator=torch.Generator().manual_seed(5)).cuda()
    c = (torch.arange(N) % cfg["num_classes"]).cuda()
    torch.manual_seed(0)
    all_ = s.sample(N, noise=x, classes=c, steps=10, strength=0.5, verbose=False).samples.clone()
    for i in range(N):
        torch.manual_seed(0)
        one = s.sample(1, noise=x[i:i + 1].contiguous(), classes=c[i:i + 1], steps=10, strength=0.5, verbose=False).samples
        assert torch.equal(one[0], all_[i]), f"sample {i} depends on the batch"
    print("[ends] DDIM-10 of 33 guided samples: every sample bitwise equal to its own run")

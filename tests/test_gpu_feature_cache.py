"""GPU: feature reuse between denoising steps (DeepCache, include/ivid_b200.h: ivid_unet_forward_reuse and the cache_* fields
of ivid_step_args_t).

A reuse forward runs the kept blocks' ops of the full forward's plan on the tensor the last full forward left in place, so a
reuse forward right after a full forward with the same inputs computes the same bits.  A reuse forward at other inputs is
checked against the oracle's reuse forward (tests/deepcache_ref.py) fed the GPU's own cached tensor, at the forward parity
bar of tests/test_gpu_unet.py.  Whole runs are checked bitwise against chained sample_once calls that follow the schedule
rule, which the test builds itself."""
import ctypes
import json

import numpy as np
import pytest
import torch

import deepcache_ref
import gpu_util as G
import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
import precision_model as PM
from ivid_b200 import _lib
from oracle import sampler_ref, unet_ref

pytestmark = pytest.mark.gpu
T = 1000
S = 0.5
NORTH_STAR, HARD_CAP = 1e-3, 1.6e-3


def _randn(seed, shape):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal(shape).astype(np.float32)).cuda()


def _golden_cfg(golden, tag):
    return json.loads(bytes(golden[tag]).decode())


def _cfgs(golden):
    tiny = _golden_cfg(golden, "tiny_cfg")
    return {
        "tiny": tiny,
        "tiny_cond": _golden_cfg(golden, "tiny_cond_cfg"),
        "tiny_sr": _golden_cfg(golden, "tiny_sr_cfg"),
        "large": _golden_cfg(golden, "schemacfg_rgbd_imagenet_adm_128_large_cfg"),
        "fp8": tiny,
        "non_square": tiny,
        "no_updown": dict(tiny, resblock_updown=False, num_res_blocks=2),
        "top_attention": dict(tiny, attention_resolutions=[32, 16], num_res_blocks=2),
    }


def _net(cfg, seed=1234, precision="fp16"):
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    net = net.cuda()
    if precision != "fp16":
        net.set_precision(precision)
    net._ensure_packed()
    return net


class _Inputs:
    """x, t, classes and the conditional inputs (injected hole noise for InpaintCFG) of one forward."""

    def __init__(self, cfg, N, H, W, seed, kind=0):
        self.N, self.H, self.W = N, H, W
        self.x = _randn(seed, (N, 4 if kind else cfg["in_channels"], H, W))
        self.t = torch.full((N,), 300 + seed, dtype=torch.int64, device="cuda")
        self.classes = (torch.arange(N, device="cuda") % cfg["num_classes"]) if cfg.get("num_classes") else None
        self.cond = None
        self._keep = []
        if kind == 1:
            y, mask = _randn(seed + 1, (N, 4, H, W)), (_randn(seed + 2, (N, 1, H, W)) > 0).float()
            mask_rgb, noise = (_randn(seed + 3, (N, 1, H, W)) > 0).float(), _randn(seed + 4, (N, 4, H, W))
            self._keep = [y, mask, mask_rgb, noise]
            self.cond = _lib.CondT(kind=1, y_dev=y.data_ptr(), mask_dev=mask.data_ptr(), mask_rgb_dev=mask_rgb.data_ptr(),
                                   noise_dev=noise.data_ptr())
        elif kind == 2:
            y = _randn(seed + 1, (N, 4, H // 2, W // 2))
            self._keep = [y]
            self.cond = _lib.CondT(kind=2, y_dev=y.data_ptr())


def _forward(net, inp, branch=None):
    eps = torch.empty((inp.N, 4, inp.H, inp.W), device="cuda")
    L = _lib.lib()
    cond = ctypes.byref(inp.cond) if inp.cond is not None else None
    args = (net._handle, _lib.ptr(inp.x), inp.N, inp.H, inp.W, cond, _lib.ptr(inp.t), _lib.ptr(inp.classes), _lib.ptr(eps), inp.N)
    if branch is None:
        _lib.check(L.ivid_unet_forward_hw(*args, _lib.cur_stream()))
    else:
        _lib.check(L.ivid_unet_forward_reuse(*args, branch, _lib.cur_stream()))
    torch.cuda.synchronize()
    return eps


def _case(golden, tag):
    cfg = _cfgs(golden)[tag]
    kind = {"tiny_cond": 1, "tiny_sr": 2}.get(tag, 0)
    H, W = (32, 48) if tag == "non_square" else (cfg["image_size"],) * 2
    N = 2 if tag == "large" else 3
    return cfg, _net(cfg, precision="fp8" if tag == "fp8" else "fp16"), _Inputs(cfg, N, H, W, 5, kind)


@pytest.mark.parametrize("tag", ["tiny", "tiny_cond", "tiny_sr", "large", "fp8", "non_square", "no_updown", "top_attention"])
def test_reuse_after_full_is_bitwise_full(golden, tag):
    """Right after a full forward with the same inputs, a reuse forward at every branch returns the full forward's eps bit for
    bit (eager first call, then CUDA-graph captures and replays)."""
    cfg, net, inp = _case(golden, tag)
    full = _forward(net, inp)
    assert torch.isfinite(full).all()
    for rnd in range(2):
        for b in range(cfg["num_res_blocks"] + 1):
            assert torch.equal(_forward(net, inp, b), full), f"{tag}: branch {b}, round {rnd}"
        assert torch.equal(_forward(net, inp), full)


def _last_layer(cfg, block):
    blocks, _ = unet_ref._topology(cfg)
    return [b for b in blocks if b["prefix"] == block][0]["layers"][-1][1]


@pytest.mark.parametrize("tag", ["tiny", "top_attention"])
def test_reuse_vs_oracle(golden, tag):
    """A reuse forward at another x and t, against the oracle's reuse forward fed the cached tensor read back with
    ivid_unet_debug_tap, within the forward parity bar."""
    cfg = _cfgs(golden)[tag]
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    net = _net(cfg)
    N = 2
    for b in range(cfg["num_res_blocks"] + 1):
        a, other = _Inputs(cfg, N, 32, 32, 11), _Inputs(cfg, N, 32, 32, 12 + b)
        _forward(net, a)
        layer = _last_layer(cfg, deepcache_ref.cached_block_name(cfg, b))
        C, H, W = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        _lib.check(_lib.lib().ivid_unet_debug_tap(net._handle, N, layer.encode(), None, 0, ctypes.byref(C), ctypes.byref(H), ctypes.byref(W)))
        cached = torch.empty((N, C.value, H.value, W.value))
        _lib.check(_lib.lib().ivid_unet_debug_tap(net._handle, N, layer.encode(), _lib.ptr(cached), cached.numel(), None, None, None))
        got = _forward(net, other, b)
        x, t, c = other.x.cpu(), other.t.cpu(), other.classes.cpu() if other.classes is not None else None
        ref = deepcache_ref.unet_forward(cfg, sd, x, t, c, reuse=(b, cached))
        full = unet_ref.unet_forward(cfg, sd, x, t, c)
        floor = PM.rel(PM.forward(cfg, sd, x, t, c, PM.TF32_CLASS), full)
        bar = min(max(NORTH_STAR, 1.15 * floor), HARD_CAP)
        err = G.report(f"{tag} reuse forward branch {b}", got, ref)
        assert err <= bar, f"branch {b}: rel {err:.3e} > bar {bar:.3e}"
        assert G.rel(ref, full) > 3 * bar, "the cached tensor came from other inputs, so the reuse forward differs"


# sampler kinds: (class, sample() kwargs)
KINDS = {
    "ddpm": (samplers.DdpmSampler, {}),
    "ddim": (samplers.DdimSampler, dict(eta=1.0)),
    "dpm_ode": (samplers.DpmSolverSampler, {}),
    "dpm_sde": (samplers.DpmSolverSampler, dict(sde=True)),
}


def _fw(golden, tag, cls, precision="fp16", seed=1234):
    cfg = _cfgs(golden)[tag]
    net = _net(cfg, seed=seed, precision=precision)
    return cls(net, timesteps=T, beta_schedule="linear")


def _schedule(s, steps):
    """(t, t_prev, model time) of every step of a run, as ivid_sampler_run walks them."""
    if s.KIND == 0:
        return [(t, 0, t) for t in reversed(range(T))]
    return [(t, tp, t - 1) for (t, tp) in sampler_ref.ddim_schedule(T, steps)]


def _reuse_steps(sched, every, guided_at):
    """The schedule rule, restated: full at step 0, where the forward switches between the guided and the unguided plan, and
    `every` steps after the last full step; reuse elsewhere."""
    out, last_full, last_g = [], 0, None
    for i, (_, _, tm) in enumerate(sched):
        g = guided_at(tm)
        full = every <= 1 or i == 0 or g != last_g or i - last_full >= every
        if full:
            last_full = i
        last_g = g
        out.append(not full)
    return out


def _run_injected(s, x, classes, steps, noise_all, cache_interval=0, branch=0, interval=None, cond_noise_all=None, eta=0.0,
                  sde=False, **kw):
    """ivid_sampler_run with the per-step draws injected (separate step kernel)."""
    net = s._net()
    img = x.clone().contiguous()
    a, keep = s._step_args(img.device, classes, False, eta, kw, seed=0, hw=img.shape[-2:], order=2, sde=sde, interval=interval,
                           cache=(cache_interval, branch, 0))
    ca = cond_noise_all.contiguous() if cond_noise_all is not None else None
    _lib.check(_lib.lib().ivid_sampler_run(s._handle, net._handle, _lib.ptr(img), img.shape[0], steps, ctypes.byref(a),
                                           _lib.ptr(noise_all.contiguous()), _lib.ptr(ca), None, None, _lib.cur_stream()))
    torch.cuda.synchronize()
    del keep
    return img


def _chained(s, x, classes, steps, noise_all, every, branch=0, interval=None, cond_noise_all=None, eta=0.0, sde=False, **kw):
    """Chained sample_once calls with reuse_features set by the schedule rule."""
    N = x.shape[0]
    sched = _schedule(s, steps)
    lo, hi = interval if interval is not None else (0, T - 1)
    reuse = _reuse_steps(sched, every, lambda tm: lo <= tm <= hi)
    xa, prev = x.clone(), None
    for i, (t, tp, _) in enumerate(sched):
        k = dict(kw, strength=S, noise=noise_all[i], guidance_interval=interval, reuse_features=reuse[i], cache_branch=branch)
        if cond_noise_all is not None:
            k["cond_noise"] = cond_noise_all[i]
        tt = torch.full((N,), t, device="cuda")
        if s.KIND == 0:
            out = s.sample_once(xa, tt, classes, **k)
        elif s.KIND == 1:
            out = s.sample_once(xa, tt, torch.full((N,), tp, device="cuda"), classes, eta=eta, **k)
        else:
            out = s.sample_once(xa, tt, torch.full((N,), tp, device="cuda"), classes, prev=prev, sde=sde, **k)
            prev = (t, out.pred_x_0)
        xa = out.pred_x_prev
    return xa, sum(reuse)


@pytest.mark.parametrize("kind", list(KINDS))
def test_interval_one_equals_no_caching(golden, kind):
    """cache_interval=1 runs every forward in full: the bits of a run without caching, on the fused route (Philox noise) and on
    the separate step kernel (injected noise)."""
    cls, kw = KINDS[kind]
    s = cls(_fw(golden, "tiny", frameworks.ClassifierFreeGuidance))
    x = _randn(1, (2, 4, 32, 32)); classes = torch.tensor([1, 2]).cuda()
    steps = T if kind == "ddpm" else 10
    runs = []
    for ci in (None, 1):
        torch.manual_seed(3)
        runs.append(s.sample(2, noise=x, classes=classes, steps=10, strength=S, verbose=False, cache_interval=ci, **kw).samples)
    assert torch.isfinite(runs[0]).all() and torch.equal(runs[0], runs[1])
    noise_all = _randn(2, (steps, 2, 4, 32, 32))
    assert torch.equal(_run_injected(s, x, classes, steps, noise_all, 0, strength=S, **kw),
                       _run_injected(s, x, classes, steps, noise_all, 1, strength=S, **kw))


@pytest.mark.parametrize("kind", list(KINDS))
def test_run_equals_chained_steps(golden, kind):
    """ivid_sampler_run with injected noise == chained sample_once whose reuse_features follows the schedule rule, and reuse
    changes the result."""
    cls, kw = KINDS[kind]
    s = cls(_fw(golden, "tiny", frameworks.ClassifierFreeGuidance))
    steps = T if kind == "ddpm" else 10
    x = _randn(5, (2, 4, 32, 32)); noise_all = _randn(6, (steps, 2, 4, 32, 32)); classes = torch.tensor([5, 6]).cuda()
    a = _run_injected(s, x, classes, steps, noise_all, 3, strength=S, **kw)
    b, n_reuse = _chained(s, x, classes, steps, noise_all, 3, **kw)
    c = _run_injected(s, x, classes, steps, noise_all, 0, strength=S, **kw)
    assert n_reuse > 0 and torch.isfinite(a).all()
    assert torch.equal(a, b)
    assert not torch.equal(a, c), "reuse forwards change eps"


@pytest.mark.parametrize("case", ["interval_ddim", "interval_dpm_sde", "fp8_ddim", "branch1_ddpm"])
def test_run_equals_chained_variants(golden, case):
    """The same with a guidance interval (full steps forced at the batch switches), in fp8, and at branch 1."""
    kind = case.split("_", 1)[1]
    cls, kw = KINDS[kind]
    cfg_tag = "top_attention" if case.startswith("branch1") else "tiny"
    s = cls(_fw(golden, cfg_tag, frameworks.ClassifierFreeGuidance, precision="fp8" if case.startswith("fp8") else "fp16"))
    steps = T if kind == "ddpm" else 10
    interval = (300, 700) if case.startswith("interval") else None
    branch = 1 if case.startswith("branch1") else 0
    x = _randn(7, (2, 4, 32, 32)); noise_all = _randn(8, (steps, 2, 4, 32, 32)); classes = torch.tensor([3, 4]).cuda()
    a = _run_injected(s, x, classes, steps, noise_all, 3, branch, interval=interval, strength=S, **kw)
    b, n_reuse = _chained(s, x, classes, steps, noise_all, 3, branch, interval=interval, **kw)
    assert n_reuse > 0 and torch.isfinite(a).all()
    assert torch.equal(a, b)


def _guidance(golden):
    y = torch.from_numpy(golden["ddim_y"]).cuda(); mask = torch.from_numpy(golden["ddim_mask"]).cuda()
    mask_rgb = torch.from_numpy(golden["ddim_mask_rgb"]).cuda(); convex = torch.from_numpy(golden["ddim_convex"]).cuda()
    return dict(y=y, mask=mask, mask_rgb=mask_rgb, replace_rgb=(0.1, y[:, :3], mask_rgb), replace_depth=(0.2, y[:, 3:], mask),
                constrain_depth=(0.5, convex))


@pytest.mark.parametrize("kind", ["ddim", "dpm_ode"])
@pytest.mark.parametrize("tag", ["tiny_cond", "tiny_sr"])
def test_run_equals_chained_conditional(golden, tag, kind):
    """InpaintCFG (hole noise injected, multiview replace / constrain guidance) and SuperResCFG."""
    cls, kw = KINDS[kind]
    if tag == "tiny_cond":
        fw = _fw(golden, tag, frameworks.InpaintCFG, seed=4321)
        x = torch.from_numpy(golden["step_x_t"]).cuda()
        extra = _guidance(golden)
        cond_noise_all = _randn(9, (6,) + tuple(x.shape))
    else:
        fw = _fw(golden, tag, frameworks.SuperResCFG)
        x = torch.from_numpy(golden["sr_x"]).cuda()
        extra = dict(y=torch.from_numpy(golden["sr_y"]).cuda())
        cond_noise_all = None
    s = cls(fw)
    classes = torch.arange(1, x.shape[0] + 1).cuda()
    noise_all = _randn(10, (6,) + tuple(x.shape))
    a = _run_injected(s, x, classes, 6, noise_all, 2, cond_noise_all=cond_noise_all, strength=S, **kw, **extra)
    b, n_reuse = _chained(s, x, classes, 6, noise_all, 2, cond_noise_all=cond_noise_all, **kw, **extra)
    assert n_reuse > 0 and torch.isfinite(a).all()
    assert torch.equal(a, b)


@pytest.mark.parametrize("kind", list(KINDS))
def test_fused_route_equals_separate_route(golden, kind):
    """Reuse steps give the same bits with the update fused into the output head (Philox noise) and with the separate step
    kernel (the same run keeping its trajectory)."""
    cls, kw = KINDS[kind]
    s = cls(_fw(golden, "tiny", frameworks.ClassifierFreeGuidance))
    x = _randn(11, (2, 4, 32, 32)); classes = torch.tensor([7, 8]).cuda()
    out = []
    for traj in (False, True):
        torch.manual_seed(5)
        out.append(s.sample(2, noise=x, classes=classes, steps=10, strength=S, verbose=False, cache_interval=3,
                            return_trajectory=traj, **kw).samples)
    assert torch.isfinite(out[0]).all() and torch.equal(out[0], out[1])


def test_full_after_reuse_equals_fresh_handle(golden):
    cfg, net, inp = _case(golden, "tiny")
    other = _Inputs(cfg, inp.N, inp.H, inp.W, 21)
    _forward(net, other)
    for b in range(cfg["num_res_blocks"] + 1):
        _forward(net, inp, b)
    after = _forward(net, inp)
    fresh = _forward(_net(cfg), inp)
    assert torch.equal(after, fresh)


def test_errors(golden):
    cfg, net, inp = _case(golden, "tiny")
    with pytest.raises(RuntimeError, match="reuse forward"):
        _forward(net, inp, 0)                                   # no full forward on this plan yet
    _forward(net, inp)
    _forward(net, inp, 0)
    with pytest.raises(AssertionError, match="cache_branch"):
        _forward(net, inp, cfg["num_res_blocks"] + 1)
    small = _Inputs(cfg, inp.N, 16, 16, 3)
    with pytest.raises(RuntimeError, match="reuse forward"):
        _forward(net, small, 0)                                 # another plan
    net.repack()                                                # finalize drops every plan and its cache
    with pytest.raises(RuntimeError, match="reuse forward"):
        _forward(net, inp, 0)
    s = samplers.DdimSampler(frameworks.ClassifierFreeGuidance(net, timesteps=T, beta_schedule="linear"))
    x = _randn(3, (2, 4, 32, 32)); t = torch.full((2,), 500, device="cuda")
    with pytest.raises(RuntimeError, match="reuse forward"):
        s.sample_once(x, t, t - 100, torch.tensor([1, 2]).cuda(), strength=S, reuse_features=True)
    for bad in (dict(cache_interval=0), dict(cache_interval=2, cache_branch=2)):
        with pytest.raises(AssertionError, match="cache_"):
            s.sample(2, noise=x, steps=10, verbose=False, **bad)


def _conv_flops(net, fn):
    L = _lib.lib()
    _lib.check(L.ivid_unet_profile_begin(net._handle))
    fn()
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(L.ivid_unet_profile_end(net._handle, buf, len(buf)))
    return sum(v["flops"] for k, v in json.loads(buf.value.decode()).items() if k.startswith("conv"))


def _expected_conv_flops(cfg, N, H, W, branch=None):
    """Algorithmic conv FLOPs of the layers a forward runs, from their shapes (every kept layer of a reuse forward is at the
    input resolution: the top level has no resampling)."""
    blocks, final_ch = unet_ref._topology(cfg)
    n_in = sum(b["group"] == "input" for b in blocks)
    L = sum(b["group"] == "output" for b in blocks)
    M = N * H * W
    total = 2.0 * M * 9 * final_ch * cfg["out_channels"]                    # output head
    for bi, b in enumerate(blocks):
        if branch is not None and not (bi <= branch or bi >= n_in + L - branch):
            continue
        for l in b["layers"]:
            assert branch is None or l[0] in ("conv", "res", "attn")
            if l[0] == "conv":
                total += 2.0 * M * 9 * l[2] * l[3]
            elif l[0] == "res":
                _, _, cin, cout, mode = l
                assert mode == "same" or branch is None
                total += 2.0 * M * 9 * cin * cout + 2.0 * M * (9 * cout + (cin if cin != cout else 0)) * cout
            elif l[0] == "attn":
                total += 2.0 * M * l[2] * 4 * l[2]                          # qkv (3C) + proj_out (C)
    return total


@pytest.mark.parametrize("tag", ["tiny", "top_attention"])
def test_reuse_conv_flops(golden, tag):
    cfg = _cfgs(golden)[tag]
    net = _net(cfg)
    inp = _Inputs(cfg, 2, 32, 32, 4)
    _forward(net, inp)
    for b in range(cfg["num_res_blocks"] + 1):
        got = _conv_flops(net, lambda: _forward(net, inp, b))
        want = _expected_conv_flops(cfg, 2, 32, 32, b)
        print(f"[flops] {tag} branch {b}: profiled {got:.6e} expected {want:.6e}")
        assert got == pytest.approx(want, rel=1e-6)                 # the profile JSON prints 7 significant digits
    full = _conv_flops(net, lambda: _forward(net, inp))
    assert full > got


def test_reuse_allocates_nothing(golden):
    cfg, net, inp = _case(golden, "large")
    _forward(net, inp)
    for b in range(cfg["num_res_blocks"] + 1):                   # eager, then captured: the graphs exist afterwards
        _forward(net, inp, b)
        _forward(net, inp, b)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        for b in range(cfg["num_res_blocks"] + 1):
            _forward(net, inp, b)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0


def test_torch_rng_stream_unchanged(golden):
    """rng='torch' with caching draws exactly what it draws without, and runs the schedule ivid_sampler_run runs."""
    s = samplers.DdimSampler(_fw(golden, "tiny", frameworks.ClassifierFreeGuidance))
    x = _randn(14, (2, 4, 32, 32)); classes = torch.tensor([1, 2]).cuda()
    torch.manual_seed(21)
    a = s.sample(2, noise=x, classes=classes, steps=10, strength=S, eta=1.0, verbose=False, rng="torch", cache_interval=3,
                 guidance_interval=(300, 700))
    after = torch.randn(4, device="cuda")
    torch.manual_seed(21)
    noise_all = torch.stack([torch.randn_like(x) for _ in range(10)])
    assert torch.equal(after, torch.randn(4, device="cuda")), "the torch RNG is consumed as without caching"
    assert torch.equal(a.samples, _run_injected(s, x, classes, 10, noise_all, 3, interval=(300, 700), eta=1.0, strength=S))

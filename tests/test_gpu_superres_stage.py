"""GPU: the super-resolution stage of the multiview pipeline (superresolve_views, sample_all(framework_sr=...), the upsample
entry point) on the tiny golden networks at 32^2 -> 64^2, checked bit for bit against direct sampler calls and an
independently built DeviceWarp; and the device warp at 64^2 and 256^2 against the CPU oracle."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from conftest import ROOT
from ivid_b200.inference import build_modelviews, load_scene_views, sample_all, superresolve_views
from ivid_b200.rgbd_3d import DeviceWarp
from oracle import unet_ref, warp_ref

pytestmark = pytest.mark.gpu

WARP_KW = dict(fov=45, near=0.6, far=5, atol=0.03, rtol=0.03, erode_rgb=3)
SR_WARP_KW = dict(WARP_KW, erode_rgb=3 * 2)          # erode_rgb * s at 64^2
STEPS, GUIDANCE = 4, 0.5


def _fw(golden, tag, seed, cls):
    cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    return cls(net.cuda(), timesteps=1000, beta_schedule="linear")


@pytest.fixture(scope="module")
def nets(golden):
    return (_fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance), _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG),
            _fw(golden, "tiny_sr", 1234, frameworks.SuperResCFG))


def _rows(seeds, V, S=64):
    """The stage's seeded x_T: row v of randn(V, 4, S, S) of each sample's own generator -> [B, V, 4, S, S] on the GPU."""
    return torch.stack([torch.randn(V, 4, S, S, generator=torch.Generator().manual_seed(sd)) for sd in seeds]).cuda()


def _smooth_views(B, V, n=32, seed=0):
    """Smooth synthetic RGBD views in model space [B, V, 4, n, n] (a random-weight sampler's depth is noise, which the warp
    meshes as all discontinuities)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:n, 0:n] / n
    out = np.empty((B, V, 4, n, n), np.float32)
    for b in range(B):
        for v in range(V):
            z = 0.55 + 0.08 * np.sin(6 * xx + rng.uniform(0, 6)) * np.cos(5 * yy + rng.uniform(0, 6))
            out[b, v, :3] = np.stack([0.5 + 0.5 * np.sin(9 * xx + i + v) * np.cos(7 * yy - i) for i in range(3)])
            out[b, v, 3] = z
    return torch.from_numpy(out * 2 - 1).cuda()


def _direct(fw, B, y, noise, classes, replace=None, **kw):
    s = samplers.DdimSampler(fw)
    args = {}
    if replace is not None:
        w, c = replace
        args = dict(replace_rgb=(w[0], c[:, :3] * 2 - 1, c[:, 5:6]), replace_depth=(w[1], c[:, 3:4] * 2 - 1, c[:, 4:5]))
    return s.sample(B, y=y, noise=noise, classes=classes, steps=STEPS, strength=GUIDANCE, verbose=False, **args, **kw).samples


def _pipeline(nets, viewset, sr, seeds=(5, 6, 7)):
    fu, fc, fsr = nets
    mvs = build_modelviews(viewset, len(seeds), rng=np.random.default_rng(1))
    kw = dict(classes=[1, 2, 3][:len(seeds)], guidance=GUIDANCE, batchsize=2, **WARP_KW)
    if sr:
        kw.update(framework_sr=fsr, steps_sr=STEPS, sr_size=64)
    return mvs, list(sample_all(fu, fc if viewset != "uncond" else None, list(seeds), 6, 3, mvs, **kw))


# 1 -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("viewset", ["random", "uncond"])
def test_lowres_views_are_the_pipeline_without_the_stage(nets, viewset):
    _, plain = _pipeline(nets, viewset, False)
    _, outs = _pipeline(nets, viewset, True)
    assert len(outs) == len(plain) == 3
    for (_, _, s0, c0), (meshes, colors, s1, c1) in zip(plain, outs):
        V = s0.shape[0]
        assert torch.equal(c1["lowres"], s0), viewset
        assert s1.shape == (V, 4, 64, 64) and torch.isfinite(s1).all()
        assert meshes[0].depth.shape == (64, 64, 1) and colors[-1].shape == (64, 64, 3)
        if c0 is not None:
            assert torch.equal(c1["color"], c0["color"]) and torch.equal(c1["depth"], c0["depth"])


# 2, 3 ----------------------------------------------------------------------------------------------------------------
def test_pipeline_views_equal_direct_calls(nets):
    """viewset random: view 0 of a batch is the direct SR sampler call with the seeded rows, view 1 the direct call with
    replace guidance from an independently built DeviceWarp(B, image_size=64) fed the stage's view 0."""
    fsr = nets[2]
    mvs, outs = _pipeline(nets, "random", True)
    B = 2                                                           # the first batch: samples 0 and 1
    lowres = torch.stack([outs[k][3]["lowres"] for k in range(B)])
    sr = torch.stack([outs[k][2] for k in range(B)])
    noise = _rows([5, 6], 2)
    classes = torch.tensor([1, 2]).cuda()
    v0 = _direct(fsr, B, lowres[:, 0], noise[:, 0], classes)
    assert torch.equal(sr[:, 0], v0)
    w = DeviceWarp(B, image_size=64, ssaa=3, max_views=2)
    w.add_view(sr[:, 0], [mvs[k][0] for k in range(B)], **SR_WARP_KW)
    c = w.aggregate([mvs[k][1] for k in range(B)], **SR_WARP_KW)
    v1 = _direct(fsr, B, lowres[:, 1], noise[:, 1], classes, replace=((0.1, 0.2), c))
    assert torch.equal(sr[:, 1], v1)


def test_three_view_list_equals_direct_calls(nets):
    fsr = nets[2]
    B, V = 2, 3
    views = _smooth_views(B, V)
    mvs = build_modelviews("3x9", 1)[:V]
    seeds = [11, 12]
    classes = torch.tensor([3, 4]).cuda()
    sr = superresolve_views(fsr, views, mvs, steps=STEPS, size=64, classes=[3, 4], guidance=GUIDANCE, seeds=seeds, **WARP_KW)
    assert sr.shape == (B, V, 4, 64, 64)
    noise = _rows(seeds, V)
    w = DeviceWarp(B, image_size=64, ssaa=3, max_views=V)
    for j in range(V):
        c = w.aggregate(mvs[j], **SR_WARP_KW) if j > 0 else None
        want = _direct(fsr, B, views[:, j], noise[:, j], classes, replace=((0.1, 0.2), c) if c is not None else None)
        assert torch.equal(sr[:, j], want), j
        w.add_view(sr[:, j], mvs[j], **SR_WARP_KW)


# 4 -------------------------------------------------------------------------------------------------------------------
def test_no_replace_runs_views_independently(nets):
    fsr = nets[2]
    B, V = 2, 3
    views = _smooth_views(B, V, seed=1)
    mvs = build_modelviews("3x9", 1)[:V]
    sr = superresolve_views(fsr, views, mvs, steps=STEPS, size=64, classes=[3, 4], guidance=GUIDANCE, seeds=[1, 2], replace=None)
    noise = _rows([1, 2], V)
    for j in range(V):
        assert torch.equal(sr[:, j], _direct(fsr, B, views[:, j], noise[:, j], torch.tensor([3, 4]).cuda())), j


def test_unseeded_views_are_drawn_at_the_output_size(nets):
    """Without seeds each view's x_T is drawn by its sampler at S' (64, not the backbone's image_size 32): the views equal
    direct calls with image_size=64 from the same torch RNG, and the warp of a replace run takes them."""
    fsr = nets[2]
    B, V = 2, 2
    views = _smooth_views(B, V, seed=4)
    mvs = build_modelviews("3x9", 1)[:V]
    torch.manual_seed(41)
    sr = superresolve_views(fsr, views, mvs, steps=STEPS, size=64, classes=[3, 4], guidance=GUIDANCE, replace=None)
    assert sr.shape == (B, V, 4, 64, 64)
    torch.manual_seed(41)
    for j in range(V):
        want = _direct(fsr, B, views[:, j], None, torch.tensor([3, 4]).cuda(), image_size=64)
        assert torch.equal(sr[:, j], want), j
    out = superresolve_views(fsr, _smooth_views(B, 3, seed=5), build_modelviews("3x9", 1)[:3], steps=STEPS, size=64,
                             classes=[3, 4], guidance=GUIDANCE, **WARP_KW)
    assert out.shape == (B, 3, 4, 64, 64) and torch.isfinite(out).all()


def test_unseeded_pipeline_keeps_the_lowres_views(nets):
    """num_samples without seeds: the stage draws from a reseeded fork of the torch RNG, so every batch's 128^2 views are
    those of the same run without it."""
    fu, fc, fsr = nets
    mvs = build_modelviews("random", 3, rng=np.random.default_rng(2))
    kw = dict(classes=[1, 2, 3], guidance=GUIDANCE, batchsize=2, **WARP_KW)
    torch.manual_seed(7)
    plain = list(sample_all(fu, fc, 3, 6, 3, mvs, **kw))
    torch.manual_seed(7)
    outs = list(sample_all(fu, fc, 3, 6, 3, mvs, framework_sr=fsr, steps_sr=STEPS, sr_size=64, **kw))
    for (_, _, s0, _), (_, _, s1, c1) in zip(plain, outs):
        assert torch.equal(c1["lowres"], s0) and s1.shape == (2, 4, 64, 64) and torch.isfinite(s1).all()


# 5 -------------------------------------------------------------------------------------------------------------------
def test_batch_invariance(nets):
    fsr = nets[2]
    views = _smooth_views(2, 3, seed=2)
    mvs = [build_modelviews("3x9", 1)[:3], build_modelviews("3x9", 1)[3:6]]
    kw = dict(steps=STEPS, size=64, guidance=GUIDANCE, **WARP_KW)
    both = superresolve_views(fsr, views, mvs, classes=[5, 6], seeds=[21, 22], **kw)
    alone = superresolve_views(fsr, views[1:], mvs[1:], classes=[6], seeds=[22], **kw)
    assert torch.equal(both[1], alone[0])


# 6 -------------------------------------------------------------------------------------------------------------------
OPTIONS = {
    "dpmpp": (dict(solver="dpmpp"), samplers.DpmSolverSampler, {}),
    "unipc": (dict(solver="unipc"), samplers.UniPcSampler, {}),
    "fp8": (dict(precision="fp8"), samplers.DdimSampler, {}),
    "cache": (dict(cache_interval=2), samplers.DdimSampler, dict(cache_interval=2, cache_branch=0)),
    "interval": (dict(guidance_interval=(0, 500)), samplers.DdimSampler, dict(guidance_interval=(0, 500))),
    "threshold": (dict(dynamic_threshold=0.9), samplers.DdimSampler, dict(dynamic_threshold=0.9)),
}


@pytest.mark.parametrize("name", list(OPTIONS))
def test_options_pass_through(golden, name):
    fsr = _fw(golden, "tiny_sr", 1234, frameworks.SuperResCFG)           # its own network: fp8 changes the precision
    stage_kw, cls, direct_kw = OPTIONS[name]
    views = _smooth_views(2, 2, seed=3)
    sr = superresolve_views(fsr, views, build_modelviews("3x9", 1)[:2], steps=STEPS, size=64, classes=[1, 2], guidance=GUIDANCE,
                            seeds=[31, 32], **stage_kw, **WARP_KW)
    assert fsr.backbone.precision == stage_kw.get("precision", "fp16")
    want = cls(fsr).sample(2, y=views[:, 0], noise=_rows([31, 32], 2)[:, 0], classes=torch.tensor([1, 2]).cuda(), steps=STEPS,
                           strength=GUIDANCE, verbose=False, **direct_kw).samples
    assert torch.equal(sr[:, 0], want), name
    base = superresolve_views(fsr, views, build_modelviews("3x9", 1)[:2], steps=STEPS, size=64, classes=[1, 2], guidance=GUIDANCE,
                              seeds=[31, 32], precision=stage_kw.get("precision", "fp16"), **WARP_KW)
    if name != "fp8":
        assert not torch.equal(base[:, 0], sr[:, 0]), f"{name} changes the result"


# 7 -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [64, 256])
def test_warp_at_other_sizes_matches_oracle(n):
    """DeviceWarp.aggregate at image_size 64 and 256 (192^2 and 768^2 renders) after two source views, against the whole
    oracle pipeline, as test_gpu_warp checks it at 128."""
    wg = {k: v for i in (0, 1) for k, v in np.load(os.path.join(ROOT, "tests", "golden", f"warp_golden_part{i}.npz")).items()}
    near, far, fov, atol, rtol, erode = [float(v) for v in wg["params"]]
    p = dict(fov=fov, near=near, far=far, atol=atol, rtol=rtol, erode_rgb=int(erode))
    xs = [F.interpolate(torch.from_numpy(wg[f"rgbd{i}"].transpose(2, 0, 1)[None] * 2 - 1).float(), size=(n, n), mode="bilinear",
                        align_corners=False).cuda() for i in range(2)]
    dw = DeviceWarp(1, image_size=n, ssaa=3, max_views=3)
    rend = warp_ref.SoftwareAggregationRenderer(3 * n, n)
    ms, cs = [], []
    for j in range(2):
        r01 = xs[j].cpu().numpy().transpose(0, 2, 3, 1)[0] * 0.5 + 0.5
        ms.append(warp_ref.depth_to_mesh(warp_ref.linearize_depth(r01[:, :, 3:], near, far), fov=fov, modelview=wg["views"][j],
                                         atol=atol, rtol=rtol, erode_rgb=p["erode_rgb"]))
        cs.append(r01[:, :, :3])
        dw.add_view(xs[j], wg["views"][j], **p)
    cond = dw.aggregate(wg["views"][2], **p)[0].permute(1, 2, 0).cpu().numpy()
    ref = warp_ref.aggregate_conditions(rend, ms, cs, wg["views"][2], **p)
    m_eq = (cond[:, :, 4:5] == ref["mask"]).mean(); mr_eq = (cond[:, :, 5:6] == ref["mask_rgb"]).mean()
    agree = cond[:, :, 4] == ref["mask"][:, :, 0]
    dd = np.abs(cond[:, :, 3:4] - ref["depth"])[agree]; dc = np.abs(cond[:, :, :3] - ref["color"])
    print(f"[parity] device warp at {n}^2 ({3 * n}^2 render): mask agree {m_eq:.5f}, mask_rgb agree {mr_eq:.5f}, "
          f"coverage {float(cond[:, :, 4].mean()):.3f}, depth max {dd.max():.2e}, colour pixels off by more than one 8-bit step "
          f"{(dc > 1.5 / 255).mean():.2e}")
    assert float(cond[:, :, 4].mean()) > 0.3
    assert m_eq > 0.999 and mr_eq > 0.999
    assert dd.max() < 1e-4 and (dc > 1.5 / 255).mean() < 1e-3


# 8 -------------------------------------------------------------------------------------------------------------------
def test_upsample_saved_scenes_end_to_end(nets, golden, tmp_path):
    """A 3x9 scene written by sample_all + async_save, super-resolved by the upsample entry point, equals superresolve_views on
    its decoded views (both stored the same way), and renders to 64^2 frames."""
    from ivid_b200 import rgbd_3d
    from ivid_b200.inference import render, swing_trajectory, upsample
    from ivid_b200.inference.sample import async_save
    from ivid_b200.inference.utils import save_scene
    from ivid_b200.utils import edict
    fu, fc, _ = nets
    out = os.path.join(tmp_path, "run")
    for sub in ("results", "grids", "conds", "scenes"):
        os.makedirs(os.path.join(out, sub))
    mvs = build_modelviews("3x9", 1)
    for i, (meshes, colors, samples, conds) in enumerate(sample_all(fu, fc, [8], 6, 2, mvs, classes=[7], guidance=GUIDANCE, **WARP_KW)):
        async_save(meshes, colors, samples, conds, "class007_seed00008", edict(output_dir=out, viewset="3x9")).join()
    cfg64 = dict(json.loads(bytes(golden["tiny_sr_cfg"]).decode()), image_size=64)   # its image_size is the stage's output size
    cp = os.path.join(tmp_path, "sr.json")
    json.dump({"backbone": {"name": "AdmUnet2d", "args": cfg64},
               "framework": {"name": "SuperResCFG", "args": {"timesteps": 1000, "beta_schedule": "linear"}}}, open(cp, "w"))
    kp = os.path.join(tmp_path, "sr.pt")
    torch.save(unet_ref.make_synthetic_state_dict(cfg64, seed=1234), kp)
    upsample.main(["--scene_dir", out, "--config_sr", cp, "--ckpt_sr", kp, "--steps_sr", str(STEPS), "--guidance", str(GUIDANCE)])
    got_path = os.path.join(out + f"_sr{STEPS}", "scenes", "scene_class007_seed00008.npz")
    assert os.path.exists(os.path.join(out + f"_sr{STEPS}", "results", "rgb_class007_seed00008.png"))
    got = load_scene_views(got_path)
    assert len(got) == 27 and got[0].color.shape == (64, 64, 3)
    # the same stage on the decoded views, stored the same way
    net = backbones.AdmUnet2d(**cfg64)
    net.load_state_dict(torch.load(kp))
    fsr = frameworks.SuperResCFG(net.cuda(), timesteps=1000, beta_schedule="linear")
    views = load_scene_views(os.path.join(out, "scenes", "scene_class007_seed00008.npz"))
    x = torch.stack([torch.from_numpy(np.concatenate([v.color.astype(np.float32) * 2 - 1,
                                                      rgbd_3d.utils.project_depth(v.depth, 0.6, 5).astype(np.float32) * 2 - 1], -1))
                     .permute(2, 0, 1) for v in views])[None].cuda()
    sr = superresolve_views(fsr, x, [v.modelview for v in views], steps=STEPS, classes=[7], guidance=GUIDANCE, seeds=[8],
                            fov=float(views[0].fov))
    rgbd = sr[0].permute(0, 2, 3, 1).cpu().numpy() * 0.5 + 0.5
    ref_path = os.path.join(tmp_path, "ref.npz")
    save_scene(ref_path, [edict(depth=rgbd_3d.utils.linearize_depth(rgbd[v, :, :, 3:], 0.6, 5), fov=views[v].fov,
                                modelview=views[v].modelview) for v in range(27)], [rgbd[v, :, :, :3] for v in range(27)])
    want = load_scene_views(ref_path)
    for g, w in zip(got, want):
        assert np.array_equal(g.color, w.color) and np.array_equal(g.depth, w.depth)
    assert render.scene_image_size(got_path) == 64
    renderer = rgbd_3d.AggregationRenderer(64 * render.SSAA, 64, near=0.1, far=200)
    cols, deps = render.render_scene(renderer, got_path, swing_trajectory(3))
    assert cols.shape == (3, 64, 64, 3) and deps.shape == (3, 64, 64, 3) and cols.dtype == np.uint8

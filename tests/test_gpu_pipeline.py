"""GPU: the whole multiview loop (uncond sampler -> device warp -> conditional sampler with guidance) on tiny models,
through the reference-facing driver `sample_all`, checked against a manual chain of the same public pieces."""
import json
import os

import numpy as np
import pytest
import torch

import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200.inference import build_modelviews, sample_all
from ivid_b200.rgbd_3d import DeviceWarp
from oracle import unet_ref

pytestmark = pytest.mark.gpu


def _fw(golden, tag, seed, cls):
    cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
    return cls(net.cuda(), timesteps=1000, beta_schedule="linear")


def test_sample_all_two_views(golden):
    fu = _fw(golden, "tiny", 1234, frameworks.ClassifierFreeGuidance)
    fc = _fw(golden, "tiny_cond", 4321, frameworks.InpaintCFG)
    mvs = build_modelviews("random", 3, rng=np.random.default_rng(1))
    kw = dict(fov=45, near=0.6, far=5, atol=0.03, rtol=0.03, erode_rgb=3)
    outs = list(sample_all(fu, fc, [5, 6, 7], 10, 4, mvs, classes=[1, 2, 3], guidance=0.5, batchsize=2, **kw))
    assert len(outs) == 3
    for meshes, colors, samples, conds in outs:
        assert samples.shape == (2, 4, 32, 32) and torch.isfinite(samples).all()
        assert conds["color"].shape == (1, 3, 32, 32) and conds["depth"].shape == (1, 1, 32, 32)
        assert len(meshes) == 2 and meshes[0].depth.shape == (32, 32, 1) and colors[1].shape == (32, 32, 3)
    # manual chain for the first batch: same seeds, same Philox draws?  Philox seeds come from torch's generator, so
    # compare the deterministic parts: view 0 depends only on (seed noise, sampler seed); re-run with rng='torch'
    torch.manual_seed(0)
    a = list(sample_all(fu, fc, [5], 6, 3, [mvs[0]], classes=[1], guidance=0.5, batchsize=1, rng="torch", **kw))[0][2]
    torch.manual_seed(0)
    b = list(sample_all(fu, fc, [5], 6, 3, [mvs[0]], classes=[1], guidance=0.5, batchsize=1, rng="torch", **kw))[0][2]
    assert torch.equal(a, b), "the pipeline is deterministic given the torch RNG state"
    # the warp inside the loop equals a stand-alone DeviceWarp fed with the same view-0 sample
    w = DeviceWarp(1, image_size=32, ssaa=3, max_views=2)
    w.add_view(a[0:1], mvs[0][0], **kw)
    cond = w.aggregate(mvs[0][1], **kw)
    # (random-weight samples are depth noise: almost everything is a discontinuity, so coverage is tiny but well-formed)
    assert cond.shape == (1, 7, 32, 32) and torch.isfinite(cond).all()
    assert torch.all(cond[:, 5] <= cond[:, 4]), 'mask_rgb is a subset of mask (utils.py:464)'
    assert torch.all((cond[:, 4] == 0) | (cond[:, 4] == 1))


def test_large_models_two_view_pipeline(golden):
    """BASELINE config 3 shape at reduced step counts: rgbd_imagenet_adm_128_large_cfg (uncond, DDIM 6 steps) ->
    device warp -> rgbd_imagenet_adm_128_large_cond (InpaintCFG, DDIM 3 steps, replace/constrain guidance), batch 2,
    viewset 'random', guidance 0.5, synthetic weights.  Checks the whole multiview loop runs on the real architectures."""
    def fw(name, seed, cls):
        cfg = json.loads(bytes(golden[f"schemacfg_{name}"]).decode())
        net = backbones.AdmUnet2d(**cfg)
        net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=seed))
        return cls(net.cuda(), timesteps=1000, beta_schedule="linear")
    fu = fw("rgbd_imagenet_adm_128_large_cfg", 1234, frameworks.ClassifierFreeGuidance)
    fc = fw("rgbd_imagenet_adm_128_large_cond", 4321, frameworks.InpaintCFG)
    mvs = build_modelviews("random", 2, rng=np.random.default_rng(3))
    outs = list(sample_all(fu, fc, [11, 12], 6, 3, mvs, classes=[11, 12], guidance=0.5, batchsize=2, erode_rgb=3))
    assert len(outs) == 2
    for meshes, colors, samples, conds in outs:
        assert samples.shape == (2, 4, 128, 128) and torch.isfinite(samples).all()
        assert conds["color"].shape == (1, 3, 128, 128) and len(meshes) == 2 and meshes[1].depth.shape == (128, 128, 1)


# ----------------------------------------------------------------------------------------------------------------------
# Teacher-forced parity of the multiview chain on the REAL architectures (BASELINE configs 3 / 4: view j of a sample) and
# of BASELINE config 1 (small model, DDIM-10).  Every stage gets the ORACLE's output of the previous stage as input, so
# each comparison isolates one stage: warp -> condition maps (exact masks), condition maps -> one guided DDIM step of the
# conditional model (x_{t-1} within the north star's 1e-3).
#   reference: inference/sample.py:75-139 (view loop), rgbd_3d/utils.py:420-477 (aggregate_conditions),
#              diffusion/frameworks/inpaint_cfg.py:61-83, diffusion/samplers/ddim.py:81-103
# ----------------------------------------------------------------------------------------------------------------------
def _real_fw(golden, name, seed, cls):
    cfg = json.loads(bytes(golden[f"schemacfg_{name}"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=seed)
    net = backbones.AdmUnet2d(**cfg)
    net.load_state_dict(sd)
    return cfg, sd, cls(net.cuda(), timesteps=1000, beta_schedule="linear")


def test_multiview_chain_teacher_forced_large_models(golden):
    import gpu_util as G
    from conftest import ROOT
    from oracle import sampler_ref, warp_ref
    wg = {k: v for i in (0, 1) for k, v in np.load(os.path.join(ROOT, "tests", "golden", f"warp_golden_part{i}.npz")).items()}
    near, far, fov, atol, rtol, erode = [float(v) for v in wg["params"]]
    p = dict(fov=fov, near=near, far=far, atol=atol, rtol=rtol, erode_rgb=int(erode))
    # stage 0: "view 0" of two samples = the smooth synthetic RGBD images of the warp fixture (a random-weight sampler would
    # produce depth noise, i.e. a degenerate all-discontinuity mesh), in model space [-1, 1]
    x0 = torch.cat([torch.from_numpy(wg[f"rgbd{i}"].transpose(2, 0, 1)[None] * 2 - 1).float() for i in range(2)], 0).cuda()
    mv0, mv1 = wg["views"][0], wg["views"][1]
    # stage 1: warp.  CUDA DeviceWarp (mesh build + rasterise + aggregate + post-filters) vs the oracle pipeline
    dw = DeviceWarp(2, image_size=128, ssaa=3, max_views=2)
    dw.add_view(x0, mv0, **p)
    cond = dw.aggregate(mv1, **p)                                             # [2,7,128,128]
    r01 = x0.cpu().numpy().transpose(0, 2, 3, 1) * 0.5 + 0.5
    rend = [warp_ref.SoftwareAggregationRenderer(384, 128) for _ in range(2)]
    conds_ref = []
    for b in range(2):
        m = warp_ref.depth_to_mesh(warp_ref.linearize_depth(r01[b][:, :, 3:], near, far), fov=fov, modelview=mv0, atol=atol, rtol=rtol,
                                   erode_rgb=int(erode))
        ref = warp_ref.aggregate_conditions(rend[b], [m], [r01[b][:, :, :3]], mv1, **p)
        got = cond[b].permute(1, 2, 0).cpu().numpy()
        # coverage is decided by exact integer edge functions on both sides; the CUDA mesh is within one float32 ulp of the
        # oracle's float64 mesh, so at most a handful of boundary pixels may differ
        m_eq = (got[:, :, 4:5] == np.asarray(ref["mask"], np.float32)).mean()
        mr_eq = (got[:, :, 5:6] == np.asarray(ref["mask_rgb"], np.float32)).mean()
        agree = got[:, :, 4] == np.asarray(ref["mask"], np.float32)[:, :, 0]
        dd = np.abs(got[:, :, 3:4] - ref["depth"])[agree].max(); dc = np.abs(got[:, :, :3] - ref["color"])
        print(f"[parity] chain warp sample {b}: mask agree {m_eq:.6f}, mask_rgb agree {mr_eq:.6f}, depth max {dd:.2e}, "
              f"colour pixels off by > one 8-bit step {(dc > 1.5 / 255).mean():.2e}")
        assert m_eq > 0.9995 and mr_eq > 0.9995
        assert dd < 1e-4 and (dc > 1.5 / 255).mean() < 1e-3
        conds_ref.append(np.concatenate([np.asarray(ref[k], np.float32) for k in ("color", "depth", "mask", "mask_rgb", "depth_convex")], -1))
    # stage 2: one guided DDIM step (50-step schedule, first and a late step) of the conditional model fed with the ORACLE's
    # condition maps, exactly the call of sample.py:104-119
    cfg_c, sd_c, fw_c = _real_fw(golden, "rgbd_imagenet_adm_128_large_cond", 4321, frameworks.InpaintCFG)
    sc = samplers.DdimSampler(fw_c)
    cr = torch.from_numpy(np.stack(conds_ref).transpose(0, 3, 1, 2)).float()          # [2,7,128,128] in [0,1]
    y = cr[:, 0:4] * 2 - 1; mask = cr[:, 4:5]; mask_rgb = cr[:, 5:6]; convex = cr[:, 6:7] * 2 - 1
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", 1000))
    model = lambda xx, tt, c: unet_ref.unet_forward(cfg_c, sd_c, xx, tt, c)
    rng = np.random.default_rng(5)
    classes = torch.tensor([17, 901])
    for (tt, tp) in [(1000, 980), (60, 40)]:
        x_t = torch.from_numpy(rng.standard_normal((2, 4, 128, 128)).astype(np.float32))
        zn = torch.from_numpy(rng.standard_normal((2, 4, 128, 128)).astype(np.float32))
        t = torch.tensor([tt] * 2); tpv = torch.tensor([tp] * 2)
        inp = sampler_ref.make_inpaint_inputs(x_t, y, mask, mask_rgb, zn[:, :3], zn[:, 3:])
        eps = sampler_ref.cond_eps(model, inp, t - 1, classes, 0.5)
        ref, _ = sampler_ref.ddim_step(tb, x_t, t, tpv, eps, torch.zeros_like(x_t), replace_rgb=(0.1, y[:, :3], mask_rgb),
                                       replace_depth=(0.2, y[:, 3:], mask), constrain_depth=(0.5, convex))
        out = sc.sample_once(x_t.cuda(), t.cuda(), tpv.cuda(), classes.cuda(), strength=0.5, y=y.cuda(), mask=mask.cuda(),
                             mask_rgb=mask_rgb.cuda(), replace_rgb=(0.1, y[:, :3].cuda(), mask_rgb.cuda()),
                             replace_depth=(0.2, y[:, 3:].cuda(), mask.cuda()), constrain_depth=(0.5, convex.cuda()),
                             noise=torch.zeros_like(x_t).cuda(), cond_noise=zn.cuda())
        r = G.report(f"chain: large_cond guided DDIM step {tt}->{tp} x_prev", out.pred_x_prev, ref)
        assert r < 1e-3 and r < 4e-4
    # stage 0 on the real unconditional model: one DDPM + CFG step (config 2 / view 0 of configs 3-4)
    cfg_u, sd_u, fw_u = _real_fw(golden, "rgbd_imagenet_adm_128_large_cfg", 1234, frameworks.ClassifierFreeGuidance)
    su = samplers.DdpmSampler(fw_u)
    modelu = lambda xx, tt, c: unet_ref.unet_forward(cfg_u, sd_u, xx, tt, c)
    x_t = torch.from_numpy(rng.standard_normal((1, 4, 128, 128)).astype(np.float32))
    z = torch.from_numpy(rng.standard_normal((1, 4, 128, 128)).astype(np.float32))
    t = torch.tensor([700]); cl = torch.tensor([5])
    ref, _ = sampler_ref.ddpm_step(tb, x_t, t, sampler_ref.cfg_eps(modelu, x_t, t, cl, 0.5), z)
    out = su.sample_once(x_t.cuda(), t.cuda(), cl.cuda(), strength=0.5, noise=z.cuda())
    r = G.report("chain: large_cfg DDPM+CFG step t=700 x_prev", out.pred_x_prev, ref)
    assert r < 1e-3 and r < 5e-5


def test_config1_small_model_ddim10_two_steps(golden):
    """BASELINE config 1 on the GPU path: rgbd_singlecategory_adm_128_small + GaussianDiffusion (no CFG), DDIM-10, batch 1:
    the first two steps teacher-forced against the oracle."""
    import gpu_util as G
    from oracle import sampler_ref
    cfg, sd, fw = _real_fw(golden, "rgbd_singlecategory_adm_128_small", 1234, frameworks.GaussianDiffusion)
    s = samplers.DdimSampler(fw)
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", 1000))
    torch.manual_seed(0)
    xo = torch.randn(1, 4, 128, 128)
    for (tt, tp) in sampler_ref.ddim_schedule(1000, 10)[:2]:
        t = torch.tensor([tt]); tpv = torch.tensor([tp])
        eps = unet_ref.unet_forward(cfg, sd, xo, t - 1, None)
        ref, _ = sampler_ref.ddim_step(tb, xo, t, tpv, eps, torch.zeros_like(xo))
        out = s.sample_once(xo.cuda(), t.cuda(), tpv.cuda(), None, noise=torch.zeros_like(xo).cuda())
        r = G.report(f"config 1: small DDIM-10 step {tt}->{tp} x_prev", out.pred_x_prev, ref)
        # DDIM-10 multiplies the eps error by up to 1.6 (SURVEY Appendix C): x_{t-1} <= 1.6 x eps bar
        assert r < 1.6e-3
        xo = ref


def test_cli_main_writes_reference_outputs(golden, tmp_path):
    """`python -m ivid_b200.inference.sample` end to end on tiny models (configs + checkpoints on disk, as the reference CLI
    consumes them): the directory contract of sample.py:150-176 per view set, scenes loadable by load_scene_views."""
    import argparse
    from PIL import Image
    from ivid_b200.inference import load_scene_views
    from ivid_b200.inference.sample import main
    paths = {}
    for tag, fw_name, seed in (("tiny", "ClassifierFreeGuidance", 1234), ("tiny_cond", "InpaintCFG", 4321)):
        cfg = json.loads(bytes(golden[f"{tag}_cfg"]).decode())
        cj = {"backbone": {"name": "AdmUnet2d", "args": cfg}, "framework": {"name": fw_name, "args": {"timesteps": 1000, "beta_schedule": "linear"}}}
        cp = os.path.join(tmp_path, f"{tag}.json"); json.dump(cj, open(cp, "w"))
        kp = os.path.join(tmp_path, f"{tag}.pt"); torch.save(unet_ref.make_synthetic_state_dict(cfg, seed=seed), kp)
        paths[tag] = (cp, kp)
    for viewset, expect in (("uncond", {"results": 2, "scenes": 2, "grids": 0, "conds": 0}),
                            ("random", {"results": 2, "scenes": 0, "grids": 2, "conds": 2}),
                            ("3x9", {"results": 0, "scenes": 2, "grids": 4, "conds": 4})):
        opt = argparse.Namespace(config_uncond=paths["tiny"][0], ckpt_uncond=paths["tiny"][1], config_cond=paths["tiny_cond"][0],
                                 ckpt_cond=paths["tiny_cond"][1], output_dir=os.path.join(tmp_path, "out"), seeds="3-4", num_samples=None,
                                 classes="mod", viewset=viewset, steps_uncond=4, steps_cond=2, guidance=0.5, batchsize=2, fov=45, near=0.6,
                                 far=5, atol=0.03, rtol=0.03, erode_rgb=3, rng="torch")
        main(0, 1, opt)
        out = os.path.join(tmp_path, "out", f"viewset_{viewset}_steps_u4_c2_guidance0.5")
        for sub, n in expect.items():
            files = sorted(os.listdir(os.path.join(out, sub)))
            assert len(files) == n, (viewset, sub, files)
        if viewset == "3x9":
            assert Image.open(os.path.join(out, "grids", "rgb_class003_seed00003.png")).size == (9 * 34 + 2, 3 * 34 + 2)
            assert len(load_scene_views(os.path.join(out, "scenes", "scene_class004_seed00004.npz"))) == 27
        if viewset == "random":
            assert Image.open(os.path.join(out, "results", "rgb_class003_seed00003.png")).size == (32, 32)

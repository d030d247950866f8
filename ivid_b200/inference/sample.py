"""Multiview sampling driver — mirror of the reference's inference/sample.py (sample_all :30-147, per-rank sharding
:199-202, view sets :304-338) with the per-view loop kept on the device:

    view 0:  unconditional sampler  (DDPM 1000 / DDIM), or a given view (SDEdit of it)  -> RGBD on the GPU
    view j:  DeviceWarp.aggregate (CUDA mesh + rasterise + aggregate + post-filters)  -> condition maps on the GPU
             conditional DDIM sampler with replace / constrain guidance               -> RGBD on the GPU
    then, with a super-resolution network, every view again at its size (superres.superresolve_views)

Nothing crosses PCIe inside the loop; samples are copied to the host once per batch for saving.

    python -m ivid_b200.inference.sample --config_uncond ... --ckpt_uncond ... (same flags as the reference CLI)
"""
from __future__ import annotations

import argparse
import json
import os
import threading
from dataclasses import asdict

import numpy as np
import torch

from .. import backbones, frameworks, samplers
from ..rgbd_3d import DeviceWarp, glm_compat as glm
from ..rgbd_3d import utils as rgbd_utils
from ..samplers.options import (SamplerOptions, add_arguments, check_arguments, int_at_least,
                                parse_apg, solver_sampler)  # noqa: F401  (parse_apg: the --apg parser, part of this CLI's surface)
from ..utils import edict
from .superres import check_superres, superresolve_views
from .utils import colorize_depth, parse_int_list, reorder, save_scene


_SR_STREAM = 0x2A5AC0DE5EED0001      # mixed into the reseed of an unseeded super-resolution stage


def shard(items, rank, world_size):
    """seeds / classes / per-sample modelviews of this rank (sample.py:199-202: [rank::world_size])."""
    return items[rank::world_size] if items is not None else None


def preprocess_init_view(image, disparity, image_size, normalize=False, normalize_depth=False, prepocess_depth="none", near=0.5,
                         far=100, **_):
    """[4, S, S] RGBD of a photo and its disparity map, as the reference's datasets make a training x_0 (datasets/base.py:92-126,
    BaseDataset.get_file / process_file, with their `dataset.args`): the disparity / 6250 rescaled so its maximum is at most
    1 / near, floored at 1e-3 and mapped by `prepocess_depth`; the image resized to S on its short side (LANCZOS) and the
    depth (NEAREST), both centre-cropped to S x S; each mapped to [-1, 1] when its normalize flag is set.
    image: a PIL image; disparity: a 2-D array as the datasets store it (the `arr_0` of their .npz files)."""
    from PIL import Image
    assert prepocess_depth in ("none", "to_depth", "disparity_minmax", "depth_minmax", "z_buffer"), \
        f"unknown depth preprocessing {prepocess_depth!r}"
    depth = np.asarray(disparity).astype(np.float32)
    assert depth.ndim == 2, f"the disparity map must be 2-D, got shape {depth.shape}"
    depth /= 6250
    if depth.max() > 1 / near:
        depth /= depth.max() * near
    depth = np.maximum(depth, 1e-3)
    if prepocess_depth == "to_depth":
        depth = 1 / depth
    elif prepocess_depth == "disparity_minmax":
        depth = (depth - depth.min()) / (depth.max() - depth.min())
    elif prepocess_depth == "depth_minmax":
        depth = 1 / depth
        depth = (depth - depth.min()) / (depth.max() - depth.min())
    elif prepocess_depth == "z_buffer":
        depth = (depth - 1 / near) / (1 / far - 1 / near)
        depth = np.clip(depth, 0, 1)

    def resize_crop(img, resample):
        # torchvision Resize(S) (short side to S, the long side truncated) then CenterCrop(S)
        w, h = img.size
        short, long = (w, h) if w <= h else (h, w)
        new_long = int(image_size * long / short)
        size = (image_size, new_long) if w <= h else (new_long, image_size)
        if size != (w, h):
            img = img.resize(size, resample)
        w, h = img.size
        top, left = int(round((h - image_size) / 2.0)), int(round((w - image_size) / 2.0))
        return img.crop((left, top, left + image_size, top + image_size))

    rgb = np.array(resize_crop(image, Image.LANCZOS))
    rgb = torch.from_numpy(rgb if rgb.ndim == 3 else rgb[:, :, None]).permute(2, 0, 1).contiguous()
    rgb = rgb.to(torch.float32).div(255) if rgb.dtype == torch.uint8 else rgb.to(torch.float32)
    if rgb.shape[0] == 1:
        rgb = rgb.repeat(3, 1, 1)
    if rgb.shape[0] == 4:
        rgb = rgb[:3]
    if normalize:
        rgb = rgb * 2 - 1
    d = torch.from_numpy(np.array(resize_crop(Image.fromarray(depth), Image.NEAREST)).astype(np.float32))[None]
    if normalize_depth:
        d = d * 2 - 1
    return torch.cat([rgb, d])


def load_init_view(image_path, depth_path, dataset_args, image_size):
    """preprocess_init_view of an image file and a disparity file (.npz with arr_0, or .npy)."""
    from PIL import Image
    disparity = np.load(depth_path)
    if isinstance(disparity, np.lib.npyio.NpzFile):
        disparity = disparity["arr_0"]
    return preprocess_init_view(Image.open(image_path), disparity, image_size, **dataset_args)


def build_modelviews(viewset, num_samples, rng=None):
    """View sets of sample.py:304-338.  'random' draws yaw ~ N(0, 0.3^2), pitch ~ N(0, 0.15^2) per sample; the reference
    uses the unseeded global numpy RNG (sample.py:317-318) — pass `rng` for reproducible runs."""
    origin = lambda: glm.lookAt(glm.vec3(0, 0, 1), glm.vec3(0, 0, 0), glm.vec3(0, 1, 0))
    on_sphere = lambda yaw, pitch: glm.lookAt(glm.vec3(np.sin(yaw) * np.cos(pitch), np.sin(pitch), np.cos(yaw) * np.cos(pitch)),
                                              glm.vec3(0, 0, 0), glm.vec3(0, 1, 0))
    if viewset == "uncond":
        return [origin()]
    if viewset == "random":
        normal = (rng.normal if rng is not None else np.random.normal)
        mvs = []
        for _ in range(num_samples):
            yaw = 0.3 * normal()
            pitch = 0.15 * normal()
            mvs.append([origin(), on_sphere(yaw, pitch)])
        return mvs
    if viewset == "3x9":
        yaws, pitches = [0.0], [0.0]
        for i in range(4):
            yaws += [(i + 1) * 0.15, -(i + 1) * 0.15]
        for i in range(1):
            pitches += [(i + 1) * 0.15, -(i + 1) * 0.15]
        return [on_sphere(y, p) for y in yaws for p in pitches]
    raise NotImplementedError


@torch.no_grad()
def sample_all(framework_uncond, framework_cond, seeds_or_num_samples, steps_uncond, steps_cond, modelviews, fov=45, near=0.6,
               far=5, atol=0.03, rtol=0.03, erode_rgb=2, classes=None, guidance=3.0, batchsize=10, rng="philox", solver="ddim",
               precision="fp16", guidance_interval=None, cache_interval=None, cache_branch=0, dynamic_threshold=None, init_views=None,
               init_strength=None, pag_scale=None, pag_layers=None, apg=None, framework_sr=None, steps_sr=50, sr_size=None,
               sr_guidance=None, sr_replace=(0.1, 0.2)):
    """Generator over finished samples: (meshes, colors, samples [V,4,H,W], conds) — signature of sample.py:30-46.
    `meshes[v]` carries what save_scene needs (linear depth, fov, modelview).  solver="dpmpp" runs DpmSolverSampler
    (DPM-Solver++(2M)) wherever the reference runs DdimSampler, solver="dpmpp_sde" its stochastic variant
    (SDE-DPM-Solver++(2M)) and solver="unipc" UniPcSampler at order 2; DDPM at steps_uncond >= 1000 is kept.  precision="fp8"
    runs the ResBlock convs of both networks with e4m3 operands (AdmUnet2d.set_precision).  guidance_interval=(t_lo, t_hi)
    guides only the steps of both networks whose model time lies in [t_lo, t_hi] (the samplers' `guidance_interval`);
    the other steps run at strength 0 with one batch-N forward.  cache_interval=N, cache_branch=b reuse the deep features of
    both networks between full forwards every N steps (the samplers' `cache_interval` / `cache_branch`; None: no reuse).
    dynamic_threshold=p or (p, s_max) thresholds x_0 dynamically at every step of both networks (the samplers'
    `dynamic_threshold`).
    init_views [num_samples, 4, S, S] (RGBD in [-1, 1], one per sample of this rank, sharded like the seeds) starts every
    scene from a given first view: without init_strength view 0 IS that view and the unconditional model does not run
    (framework_uncond may be None); with init_strength view 0 is its SDEdit by the unconditional sampler (the samplers'
    `init` / `init_strength`) with the sample's class, guidance, solver and options.  Views 1... grow from view 0 as always.
    pag_scale=w, pag_layers=names add perturbed-attention guidance to every step of both networks (the samplers'
    `pag_scale` / `pag_layers`), the class-free unconditional network included; the guidance interval gates it there too.
    apg=eta, (eta, r) or (eta, r, beta) runs the classifier-free mix of both networks as adaptive projected guidance (the
    samplers' `apg`); both frameworks must have classifier-free guidance, and classes are needed.
    framework_sr (a SuperResCFG) super-resolves every batch once all its views exist (superres.superresolve_views, with
    steps_sr steps, output size sr_size or its backbone's image_size, guidance sr_guidance or `guidance`, replace weights
    sr_replace, the batch's seeds and every option above).  The stage draws from a fork of the torch RNG, so the views at S
    are bit for bit those of the call without it, seeded or not (unseeded, the fork is reseeded from one draw of the RNG,
    so the stage's draws do not repeat the next batch's); the generator yields the S' views as
    `samples`, their meshes and colours at S', and the S views as conds["lowres"] [V,4,S,S] (conds is created for it when
    the view set has no conditional views)."""
    if init_views is None:
        assert init_strength is None, "init_strength needs init_views"
    else:
        assert init_views.dim() == 4 and init_views.shape[1] == 4, f"init_views must be [num_samples,4,S,S], got {tuple(init_views.shape)}"
    assert framework_uncond is not None or (init_views is not None and init_strength is None), \
        "framework_uncond is needed unless every view 0 is given (init_views without init_strength)"
    opts = SamplerOptions(guidance_interval, cache_interval, cache_branch, dynamic_threshold, pag_scale, pag_layers, apg)
    for fw in (framework_uncond, framework_cond):          # before any device work
        if fw is not None:
            opts.resolve(fw, classes, guidance)
    ode, sde = solver_sampler(solver)
    net = (framework_uncond if framework_uncond is not None else framework_cond).backbone
    S = net.image_size
    dev = net.device
    if framework_sr is not None:
        check_superres(framework_sr, S, sr_size, sr_replace)
        opts.resolve(framework_sr, classes, guidance if sr_guidance is None else sr_guidance)
        assert isinstance(steps_sr, int) and steps_sr >= 1, f"steps_sr must be an integer >= 1, got {steps_sr!r}"
    for fw in (framework_uncond, framework_cond):
        if fw is not None and fw.backbone.precision != precision:
            fw.backbone.set_precision(precision)
    sampler_uncond = None
    if framework_uncond is not None:
        sampler_uncond = ode(framework_uncond) if steps_uncond < 1000 else samplers.DdpmSampler(framework_uncond)
    sampler_cond = ode(framework_cond) if framework_cond is not None else None
    sde_kw = dict(sde=True) if sde else {}
    # as in the reference, the unconditional model decides whether both networks take the guidance strength (without
    # one, the conditional model decides)
    kw = opts.sampler_kwargs(framework_uncond if framework_uncond is not None else framework_cond, guidance)
    num_samples = seeds_or_num_samples if not isinstance(seeds_or_num_samples, list) else len(seeds_or_num_samples)
    seeds = seeds_or_num_samples if isinstance(seeds_or_num_samples, list) else None
    if init_views is not None:
        assert tuple(init_views.shape) == (num_samples, 4, S, S), \
            f"init_views must be [{num_samples},4,{S},{S}] (one view per sample, at the backbone's size), got {tuple(init_views.shape)}"
    per_sample_views = isinstance(modelviews[0], list)
    wparams = dict(fov=fov, near=near, far=far, atol=atol, rtol=rtol, erode_rgb=erode_rgb)
    warps = {}
    sr_cache = {}

    for i in range(0, num_samples, batchsize):
        bs = min(batchsize, num_samples - i)
        if seeds is not None:
            noise = []
            for j in range(bs):
                torch.manual_seed(seeds[i + j])
                noise.append(torch.randn(1, 4, S, S, device=dev))       # sample.py:66-69
            noise = torch.cat(noise, dim=0)
        else:
            noise = None
        b_classes = torch.tensor(classes[i: i + bs]).long().to(dev) if classes is not None else None
        views_of = (lambda k: modelviews[i + k]) if per_sample_views else (lambda k: modelviews)
        n_views = len(views_of(0))
        warp = None
        if framework_cond is not None and n_views > 1:
            if bs not in warps:
                warps[bs] = DeviceWarp(bs, image_size=S, ssaa=3, max_views=max(n_views, 2), device=dev.index)
            warp = warps[bs]
            warp.reset()
        samples, cond_color, cond_depth = [], [], []
        for j in range(n_views):
            mv_j = [views_of(k)[j] for k in range(bs)] if per_sample_views else views_of(0)[j]
            if j == 0 and init_views is not None and init_strength is None:
                res = edict(samples=init_views[i: i + bs].to(device=dev, dtype=torch.float32).contiguous())
            elif j == 0:
                kw_u = dict(kw, **sde_kw) if steps_uncond < 1000 else dict(kw)
                if init_views is not None:     # SDEdit of the given view; the seeds' noise is the forward diffusion's z
                    kw_u.update(init=init_views[i: i + bs].to(device=dev, dtype=torch.float32), init_strength=init_strength)
                res = sampler_uncond.sample(bs, noise=noise, classes=b_classes, steps=steps_uncond, verbose=False, rng=rng, **kw_u)
            else:
                cond = warp.aggregate(mv_j, **wparams)                   # [bs,7,S,S] in [0,1]
                y = cond[:, 0:4] * 2 - 1                                 # sample.py:103
                mask, mask_rgb = cond[:, 4:5], cond[:, 5:6]
                cond_color.append(cond[:, 0:3] * 2 - 1)
                cond_depth.append(cond[:, 3:4] * 2 - 1)
                args = dict(y=y, mask=mask, mask_rgb=mask_rgb, replace_rgb=(0.1, y[:, :3], mask_rgb),
                            replace_depth=(0.2, y[:, 3:], mask), constrain_depth=(0.5, cond[:, 6:7] * 2 - 1))   # sample.py:104-119
                res = sampler_cond.sample(bs, classes=b_classes, steps=steps_cond, verbose=False, rng=rng, **args, **kw, **sde_kw)
            samples.append(res.samples)
            if warp is not None:
                warp.add_view(res.samples, mv_j, **wparams)
        samples = torch.stack(samples, dim=1)                           # [bs, V, 4, S, S]
        conds = {"color": torch.stack(cond_color, dim=1), "depth": torch.stack(cond_depth, dim=1)} if cond_color else None
        if framework_sr is not None:
            conds = dict(conds or {}, lowres=samples)
            # the stage draws from a fork of the torch RNG (CPU and this device), so the batches after it draw what they draw
            # without it; unseeded, the fork is reseeded first, else it would repeat the next batch's draws
            cuda_idx = ([dev.index if dev.index is not None else torch.cuda.current_device()] if dev.type == "cuda" else [])
            with torch.random.fork_rng(devices=cuda_idx):
                if seeds is None:
                    sr_seed = int(torch.randint(0, 2 ** 62, (1,)).item()) ^ _SR_STREAM
                    torch.random.default_generator.manual_seed(sr_seed)
                    for k in cuda_idx:
                        torch.cuda.default_generators[k].manual_seed(sr_seed)
                samples = superresolve_views(
                    framework_sr, samples, [views_of(k) for k in range(bs)] if per_sample_views else views_of(0),
                    steps=steps_sr, size=sr_size, classes=b_classes, guidance=guidance if sr_guidance is None else sr_guidance,
                    seeds=seeds[i: i + bs] if seeds is not None else None, replace=sr_replace, rng=rng, solver=solver,
                    precision=precision, cache=sr_cache, **asdict(opts), **wparams)           # [bs, V, 4, S', S']
        rgbd = samples.permute(0, 1, 3, 4, 2).cpu().numpy() * 0.5 + 0.5   # one D2H per batch
        for k in range(bs):
            meshes = [edict(depth=rgbd_utils.linearize_depth(rgbd[k, v, :, :, 3:], near, far), fov=fov,
                            modelview=(views_of(k)[v])) for v in range(n_views)]
            colors = [rgbd[k, v, :, :, :3] for v in range(n_views)]
            yield meshes, colors, samples[k], ({n: t[k] for n, t in conds.items()} if conds is not None else None)


def image_grid_u8(images, nrow, value_range=(-1, 1), padding=2):
    """uint8 [H', W', 3] grid of `images` [K,3,H,W] — the arithmetic of torchvision.utils.save_image(make_grid(images, nrow,
    normalize=True, value_range=value_range)) that the reference calls (sample.py:160-166): clamp to the range, scale to
    [0,1] with the 1e-5 guard, tiles separated by `padding` black pixels, then *255 + 0.5 and truncation.  Runs on the
    tensor's device (the GPU in the sampling loop), so only the packed uint8 image crosses PCIe."""
    lo, hi = value_range
    t = images.detach().to(torch.float32).clamp(lo, hi).sub(lo).div(max(hi - lo, 1e-5))
    K, C, H, W = t.shape
    if K == 1:                                  # make_grid returns a single image unpadded
        grid = t[0]
    else:
        xm = min(nrow, K)
        ym = -(-K // xm)
        hh, ww = H + padding, W + padding
        grid = t.new_zeros((C, hh * ym + padding, ww * xm + padding))
        for k in range(K):
            y, x = divmod(k, xm)
            grid[:, y * hh + padding: y * hh + padding + H, x * ww + padding: x * ww + padding + W] = t[k]
    return grid.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)


def to_u8(rgb):
    """(np.clip(x*0.5+0.5, 0, 1) * 255).astype(uint8) of a [3,H,W] model-space image (sample.py:156,161-162)."""
    return (rgb.detach().to(torch.float32).mul(0.5).add(0.5).clamp(0, 1).mul(255)).to(torch.uint8).permute(1, 2, 0)


def async_save(meshes, colors, samples, conds, suffix, cfg):
    """Writes the outputs of the reference's async_save (sample.py:150-176) for one finished sample:
         viewset uncond: results/rgb_*.png + scenes/scene_*.npz
         viewset random: grids/rgb_*.png (both views), conds/rgb_*.png (view 0), results/rgb_*.png (view 1)
         viewset 3x9   : grids/{rgb,depth}_*.png, conds/{rgb_cond,depth_cond}_*.png (3x9 mosaics, `reorder`), scenes/scene_*.npz
    After the super-resolution stage (conds["lowres"] holds the views before it) the results, grids and scene are at the
    super-resolved size, conds/ keeps the conditions the conditional model saw, and random / 3x9 add grids/rgb_lowres_*.png.
    The 8-bit images are packed on the device on the caller's stream and copied to pinned host memory asynchronously; a
    worker thread waits for that copy, encodes the PNGs and writes the scene, while the main thread goes on sampling."""
    from PIL import Image
    out = cfg.output_dir
    jobs = []       # (relative path, device uint8 HWC tensor)
    vs = cfg.viewset
    lowres = conds.get("lowres") if conds is not None else None
    if vs == "uncond":
        jobs.append((os.path.join("results", f"rgb_{suffix}.png"), to_u8(samples[0, :3])))
    elif vs == "random":
        jobs.append((os.path.join("grids", f"rgb_{suffix}.png"), image_grid_u8(samples[:, :3], 2)))
        jobs.append((os.path.join("conds", f"rgb_{suffix}.png"), to_u8((samples if lowres is None else lowres)[0, :3])))
        jobs.append((os.path.join("results", f"rgb_{suffix}.png"), to_u8(samples[1, :3])))
        if lowres is not None:
            jobs.append((os.path.join("grids", f"rgb_lowres_{suffix}.png"), image_grid_u8(lowres[:, :3], 2)))
    elif vs == "3x9":
        dev = samples.device
        jobs.append((os.path.join("grids", f"rgb_{suffix}.png"), image_grid_u8(reorder(samples[:, :3], vs), 9)))
        jobs.append((os.path.join("grids", f"depth_{suffix}.png"), image_grid_u8(reorder(colorize_depth(samples[:, 3:]).to(dev), vs), 9)))
        jobs.append((os.path.join("conds", f"rgb_cond_{suffix}.png"), image_grid_u8(reorder(conds["color"][:, :3], vs), 9)))
        jobs.append((os.path.join("conds", f"depth_cond_{suffix}.png"), image_grid_u8(reorder(colorize_depth(conds["depth"]).to(dev), vs), 9)))
        if lowres is not None:
            jobs.append((os.path.join("grids", f"rgb_lowres_{suffix}.png"), image_grid_u8(reorder(lowres[:, :3], vs), 9)))
    else:
        raise NotImplementedError
    host = []
    for rel, t in jobs:
        h = torch.empty(t.shape, dtype=torch.uint8, pin_memory=t.is_cuda)
        h.copy_(t, non_blocking=True)
        host.append((rel, h))
    done = torch.cuda.Event() if samples.is_cuda else None
    if done is not None:
        done.record()

    def worker():
        if done is not None:
            done.synchronize()
        for rel, h in host:
            Image.fromarray(h.numpy()).save(os.path.join(out, rel))
        if vs in ("uncond", "3x9"):
            save_scene(os.path.join(out, "scenes", f"scene_{suffix}.npz"), meshes, colors)

    th = threading.Thread(target=worker)
    th.start()
    return th


def _load_model(cfg, ckpt, device):
    net = getattr(backbones, cfg["backbone"]["name"])(**cfg["backbone"]["args"])
    if ckpt is not None:
        net.load_state_dict(torch.load(ckpt, map_location="cpu"))
    net = net.to(device)
    fw = getattr(frameworks, cfg["framework"]["name"])(net, **cfg["framework"]["args"])
    return fw


def main(rank, world_size, opt):
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    cfg_u = json.load(open(opt.config_uncond))
    init_image, init_strength = getattr(opt, "init_image", None), getattr(opt, "init_strength", None)
    # a given first view without a strength needs no unconditional model
    fw_u = _load_model(cfg_u, opt.ckpt_uncond, dev) if init_image is None or init_strength is not None else None
    cfg_c = json.load(open(opt.config_cond)) if opt.viewset != "uncond" or init_image is not None else None
    fw_c = _load_model(cfg_c, opt.ckpt_cond, dev) if opt.viewset != "uncond" else None
    config_sr = getattr(opt, "config_sr", None)
    fw_sr = _load_model(json.load(open(config_sr)), getattr(opt, "ckpt_sr", None), dev) if config_sr is not None else None
    seeds = parse_int_list(opt.seeds) if opt.num_samples is None else None
    num = len(seeds) if seeds is not None else opt.num_samples
    ncls = cfg_u["backbone"]["args"].get("num_classes")
    classes = None
    if ncls is not None:
        if opt.classes == "mod":
            classes = [seeds[i] % ncls for i in range(num)]
        elif opt.classes == "uniform":
            classes = [i % ncls for i in range(num)]
        elif opt.classes == "random":
            classes = [int(np.random.randint(ncls)) for _ in range(num)]
        else:
            classes = parse_int_list(opt.classes)
    mvs = build_modelviews(opt.viewset, num)
    seeds_r, classes_r = shard(seeds, rank, world_size), shard(classes, rank, world_size)
    idx = list(range(num))[rank::world_size]
    mvs_r = shard(mvs, rank, world_size) if isinstance(mvs[0], list) else mvs
    init_views = None
    if init_image is not None:
        # one view for every sample: the seeds vary the continuation (and, with a strength, the noising)
        size = cfg_u["backbone"]["args"]["image_size"]
        view = load_init_view(init_image, opt.init_depth, cfg_c["dataset"]["args"], size)
        init_views = view[None].expand(len(idx), -1, -1, -1)
    out_dir = output_dir_name(opt)
    for sub in ("results", "grids", "conds", "scenes"):                 # sample.py:283-286
        os.makedirs(os.path.join(out_dir, sub), exist_ok=True)
    save_cfg = edict(output_dir=out_dir, viewset=opt.viewset)
    gen = sample_all(fw_u, fw_c, seeds_r if seeds_r is not None else len(idx), opt.steps_uncond, opt.steps_cond, mvs_r, classes=classes_r,
                     guidance=opt.guidance, batchsize=opt.batchsize, fov=opt.fov, near=opt.near, far=opt.far, atol=opt.atol,
                     rtol=opt.rtol, erode_rgb=opt.erode_rgb, rng=opt.rng, solver=getattr(opt, "solver", "ddim"),
                     precision=getattr(opt, "precision", "fp16"), init_views=init_views, init_strength=init_strength,
                     framework_sr=fw_sr, steps_sr=getattr(opt, "steps_sr", 50),
                     sr_replace=getattr(opt, "sr_replace", SR_REPLACE_DEFAULT), **asdict(SamplerOptions.from_args(opt)))
    threads = []
    for i, (meshes, colors, samples, conds) in enumerate(gen):
        tag = (f"class{classes_r[i]:03d}_" if classes_r is not None else "") + (f"seed{seeds_r[i]:05d}" if seeds_r is not None else f"{idx[i]:05d}")
        threads.append(async_save(meshes, colors, samples, conds, tag, save_cfg))
    for th in threads:
        th.join()


def output_dir_name(opt):
    """Output directory of a run: the reference's name, with a suffix for every extension that changes the samples."""
    solver = getattr(opt, "solver", "ddim")
    precision = getattr(opt, "precision", "fp16")
    init_image, init_strength = getattr(opt, "init_image", None), getattr(opt, "init_strength", None)
    head, tail = SamplerOptions.from_args(opt).dir_suffixes()
    return os.path.join(opt.output_dir, f"viewset_{opt.viewset}_steps_u{opt.steps_uncond}_c{opt.steps_cond}_guidance{opt.guidance}"
                        + ("" if solver == "ddim" else f"_{solver}") + ("" if precision == "fp16" else f"_{precision}") + head
                        + ("" if init_image is None else f"_init-{os.path.splitext(os.path.basename(init_image))[0]}")
                        + ("" if init_strength is None else f"_strength{init_strength}")
                        + tail + _sr_suffix(opt))


SR_REPLACE_DEFAULT = (0.1, 0.2)


def _sr_suffix(opt):
    """_sr{STEPS} with --config_sr, then -replace{RGB}-{DEPTH} or -noreplace when the replace weights are not the default."""
    if getattr(opt, "config_sr", None) is None:
        return ""
    rep = getattr(opt, "sr_replace", SR_REPLACE_DEFAULT)
    tail = "" if rep == SR_REPLACE_DEFAULT else ("-noreplace" if rep is None else f"-replace{rep[0]}-{rep[1]}")
    return f"_sr{getattr(opt, 'steps_sr', 50)}" + tail


def parse_sr_replace(s):
    """'RGB,DEPTH' -> (RGB, DEPTH) of --sr_replace, both in [0, 1]; 'none' -> None (views super-resolved independently)."""
    if s.strip().lower() == "none":
        return None
    parts = s.split(",")
    if len(parts) != 2:
        raise argparse.ArgumentTypeError(f"expected RGB,DEPTH or none, got {s!r}")
    try:
        vals = tuple(float(v) for v in parts)
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected two numbers RGB,DEPTH, got {s!r}") from None
    if not all(0.0 <= v <= 1.0 for v in vals):
        raise argparse.ArgumentTypeError(f"expected weights in [0, 1], got {s!r}")
    return vals


def parse_strength(s):
    """'S' -> S of --init_strength, 0 < S <= 1."""
    try:
        v = float(s)
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected a number, got {s!r}") from None
    if not 0.0 < v <= 1.0:
        raise argparse.ArgumentTypeError(f"expected 0 < S <= 1, got {s!r}")
    return v


def parse_args(argv=None):
    """build_arg_parser().parse_args with the checks between options: --init_image and --init_depth go together, and
    --init_strength needs them."""
    ap = build_arg_parser()
    o = ap.parse_args(argv)
    if (o.init_image is None) != (o.init_depth is None):
        ap.error("--init_image and --init_depth go together")
    if o.init_strength is not None and o.init_image is None:
        ap.error("--init_strength needs --init_image and --init_depth")
    check_arguments(ap, o)
    check_sr_flags(ap, o)
    return o


def add_sr_flags(ap, required=False):
    """The super-resolution flags.  --steps_sr and --sr_replace default to argparse.SUPPRESS so that check_sr_flags can
    tell a given flag from its default."""
    ap.add_argument("--config_sr", required=required, default=None, metavar="PATH",
                    help="super-resolve every scene with this SuperResCFG config (e.g. rgbd_imagenet_adm_256_128_small_sr.json) "
                         "once its views exist: results, grids and scenes at the network's image_size (default: off)")
    ap.add_argument("--ckpt_sr", default=None, metavar="PATH", help="checkpoint of --config_sr (default: random weights)")
    ap.add_argument("--steps_sr", type=int_at_least(1), default=argparse.SUPPRESS, metavar="N",
                    help="sampler steps of every super-resolved view (default 50)")
    ap.add_argument("--sr_replace", type=parse_sr_replace, default=argparse.SUPPRESS, metavar="RGB,DEPTH|none",
                    help="replace-guidance weights of the super-resolved views towards the earlier ones, warped at the new size "
                         "(default 0.1,0.2, the conditional stage's, not tuned for super-resolution); 'none' super-resolves "
                         "every view on its own")


def check_sr_flags(ap, o):
    """--ckpt_sr, --steps_sr and --sr_replace need --config_sr; fills the defaults of the last two."""
    if o.config_sr is None:
        for flag, given in (("ckpt_sr", o.ckpt_sr is not None), ("steps_sr", hasattr(o, "steps_sr")),
                            ("sr_replace", hasattr(o, "sr_replace"))):
            if given:
                ap.error(f"--{flag} needs --config_sr")
    if not hasattr(o, "steps_sr"):
        o.steps_sr = 50
    if not hasattr(o, "sr_replace"):
        o.sr_replace = SR_REPLACE_DEFAULT


def build_arg_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config_uncond", default="configs/rgbd_imagenet_adm_128_large_cfg.json")
    ap.add_argument("--config_cond", default="configs/rgbd_imagenet_adm_128_large_cond.json")
    ap.add_argument("--ckpt_uncond", default=None)
    ap.add_argument("--ckpt_cond", default=None)
    ap.add_argument("--output_dir", default="samples/imagenet128")
    ap.add_argument("--seeds", default="0-8")
    ap.add_argument("--num_samples", type=int, default=None)
    ap.add_argument("--classes", default="mod")
    ap.add_argument("--viewset", default="3x9")
    ap.add_argument("--steps_uncond", type=int, default=1000)
    ap.add_argument("--steps_cond", type=int, default=50)
    ap.add_argument("--guidance", type=float, default=3.0)
    ap.add_argument("--batchsize", type=int, default=10)
    ap.add_argument("--fov", type=float, default=45)
    ap.add_argument("--near", type=float, default=0.6)
    ap.add_argument("--far", type=float, default=5)
    ap.add_argument("--atol", type=float, default=0.03)
    ap.add_argument("--rtol", type=float, default=0.03)
    ap.add_argument("--erode_rgb", type=int, default=3)
    ap.add_argument("--rng", choices=["philox", "torch"], default="philox",
                    help="per-step noise: 'philox' draws in-kernel (fast, default); 'torch' draws with the torch generator exactly "
                         "where the reference does (seed-for-seed reproduction of the reference's images needs this)")
    add_arguments(ap)
    ap.add_argument("--init_image", default=None, metavar="PATH",
                    help="grow every scene from this RGB image as its first view (needs --init_depth); preprocessed as the "
                         "dataset of --config_cond prepares its images")
    ap.add_argument("--init_depth", default=None, metavar="PATH",
                    help="the disparity map of --init_image as the reference's datasets store it: .npz with arr_0, or .npy")
    ap.add_argument("--init_strength", type=parse_strength, default=None, metavar="S",
                    help="with --init_image: re-sample the first view from it by SDEdit, running the last S of the unconditional "
                         "schedule, 0 < S <= 1 (default: the given view is the first view as it is)")
    add_sr_flags(ap)
    return ap


if __name__ == "__main__":
    o = parse_args()
    n = torch.cuda.device_count()
    if n <= 1:
        main(0, 1, o)
    else:
        import torch.multiprocessing as mp
        mp.spawn(main, args=(n, o), nprocs=n)

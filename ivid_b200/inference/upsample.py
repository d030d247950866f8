"""Super-resolve saved scenes: every scenes/*.npz of a run of `ivid_b200.inference.sample` goes through the same stage the
pipeline runs with --config_sr (superres.superresolve_views), so existing scenes reach the SR network's size without being
sampled again.

    python -m ivid_b200.inference.upsample --scene_dir samples/.../viewset_3x9_... --config_sr configs/..._sr.json
                                           [--ckpt_sr PATH] [--steps_sr 50] [--sr_replace 0.1,0.2|none] [--near 0.6] [--far 5]
                                           [--guidance 3.0] [--solver ddim] ...

Output: <scene_dir>_sr{steps}/scenes/ under the same file names, and results/rgb_*.png (the super-resolved views' grid).
The class and seed of a scene come from the class### and seed##### tags of its file name, which the pipeline writes;
without them the scene is super-resolved without classes (one null-class forward) and without seeds.
"""
from __future__ import annotations

import argparse
import glob
import json
import os
import re
from dataclasses import asdict

import numpy as np
import torch
from PIL import Image

from ..rgbd_3d import utils as rgbd_utils
from ..samplers.options import SamplerOptions, add_arguments, check_arguments
from ..utils import edict
from . import sample as sample_cli
from .superres import superresolve_views
from .utils import load_scene_views, reorder, save_scene


def scene_tags(name):
    """(class or None, seed or None) from the class### and seed##### tags of a scene file name."""
    cls = re.search(r"class(\d+)", name)
    seed = re.search(r"seed(\d+)", name)
    return (int(cls.group(1)) if cls else None), (int(seed.group(1)) if seed else None)


def scene_to_model_space(views, near=0.6, far=5):
    """Decoded scene views (load_scene_views) -> [V, 4, S, S] float32 in [-1, 1]: colour c * 2 - 1, depth
    project_depth(linear depth, near, far) * 2 - 1, with the planes the pipeline sampled at."""
    rgb = np.stack([v.color for v in views]).astype(np.float32) * 2 - 1
    depth = np.stack([rgbd_utils.project_depth(v.depth, near, far) for v in views]).astype(np.float32) * 2 - 1
    return torch.from_numpy(np.concatenate([rgb, depth], axis=-1)).permute(0, 3, 1, 2).contiguous()


def upsample_scene(framework_sr, path, steps=50, near=0.6, far=5, **stage_kw):
    """-> ([V, 4, S', S'] super-resolved views on the device, decoded views) of one scene file."""
    views = load_scene_views(path)
    fovs = {float(v.fov) for v in views}
    assert len(fovs) == 1, f"{path}: the views have different fields of view {sorted(fovs)}"
    cls, seed = scene_tags(os.path.basename(path))
    x = scene_to_model_space(views, near, far)[None].to(framework_sr.backbone.device)
    out = superresolve_views(framework_sr, x, [v.modelview for v in views], steps=steps, fov=fovs.pop(), near=near, far=far,
                             classes=[cls] if cls is not None else None, seeds=[seed] if seed is not None else None, **stage_kw)
    return out[0], views


def output_dir(scene_dir, steps):
    return os.path.normpath(scene_dir) + f"_sr{steps}"


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene_dir", required=True)
    sample_cli.add_sr_flags(ap, required=True)
    ap.add_argument("--near", type=float, default=0.6)
    ap.add_argument("--far", type=float, default=5)
    ap.add_argument("--atol", type=float, default=0.03)
    ap.add_argument("--rtol", type=float, default=0.03)
    ap.add_argument("--erode_rgb", type=int, default=3)
    ap.add_argument("--guidance", type=float, default=3.0)
    ap.add_argument("--rng", choices=["philox", "torch"], default="philox")
    add_arguments(ap)
    opt = ap.parse_args(argv)
    sample_cli.check_sr_flags(ap, opt)
    check_arguments(ap, opt)
    scenes = sorted(glob.glob(os.path.join(opt.scene_dir, "scenes", "*.npz")))
    print(f"Found {len(scenes)} scenes.")
    dev = torch.device("cuda", torch.cuda.current_device())
    fw = sample_cli._load_model(json.load(open(opt.config_sr)), opt.ckpt_sr, dev)
    out_dir = output_dir(opt.scene_dir, opt.steps_sr)
    for sub in ("scenes", "results"):
        os.makedirs(os.path.join(out_dir, sub), exist_ok=True)
    stage_kw = dict(replace=opt.sr_replace, atol=opt.atol, rtol=opt.rtol, erode_rgb=opt.erode_rgb, guidance=opt.guidance,
                    rng=opt.rng, solver=opt.solver, precision=opt.precision, cache={}, **asdict(SamplerOptions.from_args(opt)))
    for path in scenes:
        name = os.path.basename(path)
        out, views = upsample_scene(fw, path, steps=opt.steps_sr, near=opt.near, far=opt.far, **stage_kw)
        rgbd = out.permute(0, 2, 3, 1).cpu().numpy() * 0.5 + 0.5
        meshes = [edict(depth=rgbd_utils.linearize_depth(rgbd[v, :, :, 3:], opt.near, opt.far), fov=views[v].fov,
                        modelview=views[v].modelview) for v in range(len(views))]
        save_scene(os.path.join(out_dir, "scenes", name), meshes, [rgbd[v, :, :, :3] for v in range(len(views))])
        rgb = reorder(out[:, :3]) if len(views) in (26, 27) else out[:, :3]
        grid = sample_cli.image_grid_u8(rgb, 9 if len(views) in (26, 27) else len(views))
        stem = name[len("scene_"):-4] if name.startswith("scene_") else name[:-4]
        Image.fromarray(grid.cpu().numpy()).save(os.path.join(out_dir, "results", f"rgb_{stem}.png"))


if __name__ == "__main__":
    main()

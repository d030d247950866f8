"""Mesh export of sampled scenes: every stored scene is fused into one coloured triangle mesh on the GPU
(rgbd_3d.fusion.fuse_views: TSDF fusion of its RGBD views, surface-nets extraction) and written as a binary PLY that
MeshLab, Blender or a game engine can open.

    python -m ivid_b200.inference.export --scene_dir samples/... [--output_dir DIR] [--resolution 256] [--trunc 3]
                                         [--max_depth D] [--atol 0.03 --rtol 0.03 --erode_rgb 3]

writes <output_dir>/meshes/<scene>.ply for every <scene_dir>/scenes/<scene>.npz (the layout render.py reads), for the
pipeline's 128x128 scenes and the 256x256 super-resolved ones alike.  World coordinates are the scene's own: y up, the
cameras on the unit sphere looking at the origin.
"""
from __future__ import annotations

import argparse
import glob
import os

import numpy as np

from ..rgbd_3d.glm_compat import as_matrix
from .utils import load_scene_views


def export_scene(scene_path, resolution=256, trunc=3, max_depth=None, atol=0.03, rtol=0.03, erode_rgb=3):
    """The fused mesh of one scene file (rgbd_3d.fusion.fuse_views on its stored views)."""
    from ..rgbd_3d.fusion import fuse_views
    views = load_scene_views(scene_path)
    fovs = {float(v.fov) for v in views}
    if len(fovs) != 1:
        raise ValueError(f"{scene_path}: the views have different fields of view {sorted(fovs)}")
    depths = np.stack([v.depth[..., 0] for v in views])
    colors = np.stack([np.asarray(v.color, np.float32) for v in views])
    return fuse_views(depths, colors, [as_matrix(v.modelview) for v in views], fov=fovs.pop(), resolution=resolution, trunc=trunc,
                      max_depth=max_depth, atol=atol, rtol=rtol, erode_rgb=erode_rgb)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene_dir", type=str, required=True)
    ap.add_argument("--output_dir", type=str, default=None)
    ap.add_argument("--resolution", type=int, default=256, help="voxels along the longest edge of the scene's bounding box")
    ap.add_argument("--trunc", type=float, default=3, help="truncation distance in voxels")
    ap.add_argument("--max_depth", type=float, default=None, help="ignore pixels farther than this from their camera")
    ap.add_argument("--atol", type=float, default=0.03)
    ap.add_argument("--rtol", type=float, default=0.03)
    ap.add_argument("--erode_rgb", type=int, default=3)
    opt = ap.parse_args(argv)
    from ..rgbd_3d.fusion import write_ply
    out_dir = os.path.join(opt.output_dir or opt.scene_dir, "meshes")
    os.makedirs(out_dir, exist_ok=True)
    scenes = sorted(glob.glob(os.path.join(opt.scene_dir, "scenes", "*.npz")))
    print(f"Found {len(scenes)} scenes.")
    for scene in scenes:
        name = os.path.basename(scene)[:-4]
        mesh = export_scene(scene, opt.resolution, opt.trunc, opt.max_depth, opt.atol, opt.rtol, opt.erode_rgb)
        path = os.path.join(out_dir, f"{name}.ply")
        write_ply(path, mesh)
        print(f"{path}: {mesh.vertices.shape[0]} vertices, {mesh.faces.shape[0]} faces")


if __name__ == "__main__":
    main()

"""Free-view fusion rendering of sampled scenes (reference inference/render.py:41-89): every stored view of a scene is
re-meshed (load_scene, numeric padding) and all of them are aggregated by the CUDA AggregationRenderer at 5x
super-sampling from a camera trajectory; frames are LANCZOS-resolved to 128x128 (colour) and point-sampled + inferno
colour-mapped (depth) at the size of the stored views (128x128 for the pipeline's scenes, 256x256 after super-resolution).

    python -m ivid_b200.inference.render --scene_dir samples/... [--traj swing|random] [--frames 60] [--image_size N]

Differences from the reference script: frames are written as PNG sequences + one .npz per scene when `imageio` (mp4
writer) is not installed; the random trajectory takes a seed.
"""
from __future__ import annotations

import argparse
import glob
import os

import numpy as np
from PIL import Image

from ..rgbd_3d import glm_compat as glm
from .utils import colorize_depth, load_scene, load_scene_views

SSAA = 5                      # render.py:64


def _look_at_origin(yaw, pitch):
    eye = (np.sin(yaw) * np.cos(pitch), np.sin(pitch), np.cos(yaw) * np.cos(pitch))
    return glm.lookAt(eye, (0.0, 0.0, 0.0), (0.0, 1.0, 0.0))


def swing_trajectory(frames=60):
    """render.py:43-50: yaw = 0.6 cos t, pitch = 0.15 sin t over one period, camera on the unit sphere looking at the origin."""
    ts = np.linspace(0, 2 * np.pi, frames)
    return [_look_at_origin(0.6 * np.cos(t), 0.15 * np.sin(t)) for t in ts]


def random_views(num, seed=None):
    """render.py:52-61: one view per scene, yaw ~ clip(0.3 N(0,1), +-0.6), pitch ~ clip(0.15 N(0,1), +-0.15)."""
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(num):
        yaw = np.clip(0.3 * rng.normal(), -0.6, 0.6)
        pitch = np.clip(0.15 * rng.normal(), -0.15, 0.15)
        out.append([_look_at_origin(yaw, pitch)])
    return out


def resolve_frame(frame, image_size=128):
    """One raw aggregated frame (color [S,S,3] in [0,1], depth [S,S,1] linear) -> (uint8 [n,n,3] colour, uint8 [n,n,3]
    colour-mapped depth) exactly as render.py:74-84: 8-bit LANCZOS down-sampling, centre point sample + project_depth
    (with project_depth's own default planes 0.5 / 100, as the reference script calls it)."""
    from ..rgbd_3d import utils as r3d
    col = np.array(Image.fromarray((np.asarray(frame["color"]) * 255).astype(np.uint8)).resize((image_size, image_size), Image.Resampling.LANCZOS))
    off = SSAA // 2
    d = r3d.project_depth(np.asarray(frame["depth"])[off::SSAA, off::SSAA])
    dep = (colorize_depth(d, min=0, max=1) * 255).astype(np.uint8)
    return col, dep


_LUT = None


def depth_colour_table():
    """uint8 [256,3]: what `(colorize_depth(d, min=0, max=1) * 255).astype(np.uint8)` yields for each of the 256 quantised
    depths (cv2.COLORMAP_INFERNO -> RGB -> /255 -> *255 -> truncation, the reference's round trip render.py:80-82)."""
    global _LUT
    if _LUT is None:
        import cv2
        rgb = cv2.cvtColor(cv2.applyColorMap(np.arange(256, dtype=np.uint8)[None], cv2.COLORMAP_INFERNO), cv2.COLOR_BGR2RGB)[0]
        _LUT = ((rgb / 255 * (1 - 0) + 0) * 255).astype(np.uint8)
    return _LUT


def render_scene(renderer, scene_path, modelviews, atol=0.03, rtol=0.03, erode_rgb=3, resolve_on_device=True):
    """-> (colors uint8 [F,n,n,3], depths uint8 [F,n,n,3]) for the F target views.  The SSAA resolve (8-bit LANCZOS) and the
    depth colour map run on the device (AggregationRenderer.render_resolved); resolve_on_device=False keeps the reference's
    numpy / PIL / cv2 steps on the host (`resolve_frame`), bit-identical by construction."""
    meshes, colors = load_scene(scene_path, atol=atol, rtol=rtol, erode_rgb=erode_rgb)
    assert all(c.shape[0] == renderer.image_size for c in colors), \
        f"{scene_path}: the views are {colors[0].shape[0]}x{colors[0].shape[0]}, the renderer's image_size is {renderer.image_size}"
    if resolve_on_device:
        return renderer.render_resolved(meshes, colors, list(modelviews), lut=depth_colour_table())
    res = renderer.render(meshes, colors, list(modelviews))
    frames = res if isinstance(res, list) else [res]
    cols, deps = zip(*(resolve_frame(f, renderer.image_size) for f in frames))
    return np.stack(cols, axis=0), np.stack(deps, axis=0)


def scene_image_size(path):
    """The size n of the n x n views stored in a scene file."""
    return int(load_scene_views(path)[0].color.shape[0])


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene_dir", type=str, required=True)
    ap.add_argument("--output_dir", type=str, default=None)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--traj", type=str, default="swing")
    ap.add_argument("--seed", type=int, default=None)
    ap.add_argument("--atol", type=float, default=0.03)
    ap.add_argument("--rtol", type=float, default=0.03)
    ap.add_argument("--erode_rgb", type=int, default=3)
    ap.add_argument("--image_size", type=int, default=None, help="frame size (default: the size of the first scene's views)")
    opt = ap.parse_args(argv)
    out_dir = opt.output_dir or opt.scene_dir
    os.makedirs(os.path.join(out_dir, "results"), exist_ok=True)
    os.makedirs(os.path.join(out_dir, "videos"), exist_ok=True)
    scenes = sorted(glob.glob(os.path.join(opt.scene_dir, "scenes", "*.npz")))
    print(f"Found {len(scenes)} scenes.")
    if opt.traj == "swing":
        per_scene = [swing_trajectory(opt.frames)] * len(scenes)
    elif opt.traj == "random":
        per_scene = random_views(len(scenes), opt.seed)
    else:
        raise NotImplementedError(opt.traj)

    from .. import rgbd_3d
    n = opt.image_size if opt.image_size is not None else (scene_image_size(scenes[0]) if scenes else 128)
    renderer = rgbd_3d.AggregationRenderer(n * SSAA, n, near=0.1, far=200, device=0)
    try:
        import imageio
    except ImportError:
        imageio = None
    for scene, mvs in zip(scenes, per_scene):
        name = os.path.basename(scene)[:-4]
        cols, deps = render_scene(renderer, scene, mvs, opt.atol, opt.rtol, opt.erode_rgb)
        if opt.traj == "random":
            Image.fromarray(cols[0]).save(os.path.join(out_dir, "results", f"{name}.png"))
        elif imageio is not None:
            imageio.mimsave(os.path.join(out_dir, "videos", f"{name}.mp4"), cols, fps=30)
            imageio.mimsave(os.path.join(out_dir, "videos", f"{name}_depth.mp4"), deps, fps=30)
        else:
            np.savez_compressed(os.path.join(out_dir, "videos", f"{name}.npz"), color=cols, depth=deps)
            for i, (c, d) in enumerate(zip(cols, deps)):
                Image.fromarray(c).save(os.path.join(out_dir, "videos", f"{name}_{i:03d}.png"))
                Image.fromarray(d).save(os.path.join(out_dir, "videos", f"{name}_depth_{i:03d}.png"))


if __name__ == "__main__":
    main()

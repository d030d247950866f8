"""ORACLE (test infrastructure only — never imported by the product path).

CPU restatement of the reference's RGBD novel-view warp.
  * numpy part (this file) follows rgbd_3d/utils.py and is PINNED against the reference's own functions, which are
    importable on the build container with stubbed `glm` / `plyfile` / `easydict` (tests/golden/make_warp_golden.py):
        linearize_depth :38-58     project_depth :61-67      image_uv :70-86       unproject :89-110
        triangulate :113-134       mask_discontinuity :137-141   depth_to_mesh :144-260
        cal_depth_normal :263-274  depth_edge :311-332       aggregate_conditions :420-477
        forward_backward_warp :335-417 (training-pair warp; with SoftwareSimpleRenderer for moderngl_renderer.py:11-148)
  * the OpenGL rasteriser + GLSL shaders (moderngl_renderer.py:260-340, shaders/aggregation.*) cannot run here; they are
    restated in oracle/raster_ref.c — PARITY UNPINNED for that part (third-party GL driver arithmetic).
  * PyGLM is absent: lookAt / perspective / inverse are restated from the published GLM formulas (right-handed,
    [-1,1] clip depth, float32 like glm.mat4).  Matrices here are numpy arrays in MATHEMATICAL orientation
    (m[row, col]); world = inverse(modelview) @ camera, the reading that makes a view reproject onto itself.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import os
import subprocess

import cv2
import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class AttrDict(dict):
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


# ----------------------------------------------------------------------------------------------------------------------
# GLM restatement (float32, column vectors, m[row, col])
# ----------------------------------------------------------------------------------------------------------------------
def look_at(eye, center, up) -> np.ndarray:
    eye, center, up = (np.asarray(v, dtype=np.float32) for v in (eye, center, up))
    f = center - eye
    f = f / np.float32(np.sqrt(np.dot(f, f)))
    s = np.cross(f, up)
    s = s / np.float32(np.sqrt(np.dot(s, s)))
    u = np.cross(s, f)
    m = np.eye(4, dtype=np.float32)
    m[0, :3], m[1, :3], m[2, :3] = s, u, -f
    m[0, 3], m[1, 3], m[2, 3] = -np.dot(s, eye), -np.dot(u, eye), np.dot(f, eye)
    return m


def _tanf():
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.tanf.restype, libm.tanf.argtypes = ctypes.c_float, [ctypes.c_float]
    return libm.tanf


_TANF = _tanf()


def perspective(fovy_rad, aspect, near, far) -> np.ndarray:
    # glm::perspective takes tan of the float32 half angle with the C library's tanf; numpy's float32 tan differs from it
    # by one ulp at some angles (30 degrees is one), which moves every snapped vertex of a render at that fov
    t = np.float32(_TANF(float(np.float32(fovy_rad) / np.float32(2))))
    m = np.zeros((4, 4), dtype=np.float32)
    m[0, 0] = np.float32(1) / (np.float32(aspect) * t)
    m[1, 1] = np.float32(1) / t
    m[2, 2] = -(np.float32(far) + np.float32(near)) / (np.float32(far) - np.float32(near))
    m[3, 2] = -np.float32(1)
    m[2, 3] = -(np.float32(2) * np.float32(far) * np.float32(near)) / (np.float32(far) - np.float32(near))
    return m


def inverse(m) -> np.ndarray:
    return np.linalg.inv(np.asarray(m, dtype=np.float64)).astype(np.float32)


def view_on_sphere(yaw, pitch) -> np.ndarray:
    """Cameras of inference/sample.py:305-336: eye on the unit sphere looking at the origin, +Y up."""
    eye = (np.sin(yaw) * np.cos(pitch), np.sin(pitch), np.cos(yaw) * np.cos(pitch))
    return look_at(eye, (0, 0, 0), (0, 1, 0))


# ----------------------------------------------------------------------------------------------------------------------
# depth conventions
# ----------------------------------------------------------------------------------------------------------------------
def linearize_depth(depth, near=0.5, far=100):
    d = np.clip(depth, 1e-6, 1.0 - 1e-6)
    return near * far / (far - (far - near) * d)


def project_depth(depth, near=0.5, far=100):
    d = np.clip(depth, near, far)
    return (1 / near - 1 / d) / (1 / near - 1 / far)


def image_uv(n):
    c = np.linspace(0.5 / n, 1 - 0.5 / n, n)
    return np.stack(np.meshgrid(c, c, indexing="xy"), axis=-1)


def unproject(depth, fov=45):
    n = depth.shape[0]
    uv = image_uv(n)
    focal = 0.5 / np.tan(0.5 * np.deg2rad(fov))
    rays = np.concatenate([(uv - 0.5) / focal, -np.ones((n, n, 1))], axis=-1)
    return rays[::-1] * depth, uv


def triangulate(points):
    h, w = points.shape[:2]
    idx = np.arange(h * w).reshape(h, w)
    tl, tr, bl, br = idx[:-1, :-1], idx[:-1, 1:], idx[1:, :-1], idx[1:, 1:]
    main = np.linalg.norm(points[:-1, :-1] - points[1:, 1:], axis=-1) < np.linalg.norm(points[:-1, 1:] - points[1:, :-1], axis=-1)
    faces = np.stack([tr.ravel(), tl.ravel(), np.where(main, br, bl).ravel(),
                      bl.ravel(), br.ravel(), np.where(main, tl, tr).ravel()], axis=-1)
    return faces.reshape(-1, 3)


def mask_discontinuity(faces, depths, atol, rtol):
    d = depths.reshape(-1)[faces]
    inv = 1 / d
    return np.logical_and(d.max(-1) - d.min(-1) > atol, inv.max(-1) - inv.min(-1) > rtol)


def cal_depth_normal(points):
    p = np.pad(points, ((1, 1), (1, 1), (0, 0)), "edge")
    ex = p[:, 2:] - p[:, :-2]
    ey = p[:-2, :] - p[2:, :]
    ex = (ex[:-2] + 2 * ex[1:-1] + ex[2:]) / 4
    ey = (ey[:, :-2] + 2 * ey[:, 1:-1] + ey[:, 2:]) / 4
    n = np.cross(ex, ey)
    return n / np.linalg.norm(n, axis=-1, keepdims=True)


def depth_to_mesh(depth, fov=45, modelview=None, atol=None, rtol=None, erode_rgb=None, padding="frustum", cal_normal=True):
    """depth_to_mesh (utils.py:144-260).  padding='frustum' + normals is what inference/sample.py uses (:129-138); a number
    (pixels the border ring is pushed out by, ring not pulled to the near plane) is what inference/utils.py:load_scene uses
    for free-view rendering (padding=32); padding=None with cal_normal=False (plain n x n grid, no normals) is what
    forward_backward_warp uses for its second mesh (utils.py:391-398)."""
    n = depth.shape[0]
    plane = 2 * np.tan(0.5 * np.deg2rad(fov))
    points, uv = unproject(depth, fov)
    normal = cal_depth_normal(points) if cal_normal else None
    ret = AttrDict(depth=depth, fov=fov, modelview=modelview)
    if padding is not None:
        pad = ((1, 1), (1, 1), (0, 0))
        points, uv, depth = (np.pad(a, pad, "edge") for a in (points, uv, depth))
        if cal_normal:
            normal = np.pad(normal, pad, "edge")
        frustum = isinstance(padding, str)
        if frustum and padding != "frustum":
            raise NotImplementedError(padding)
        step = plane / n if frustum else padding * plane / n
        points[0, :, 1] += step * depth[0, :, 0]
        points[-1, :, 1] -= step * depth[-1, :, 0]
        points[:, 0, 0] -= step * depth[:, 0, 0]
        points[:, -1, 0] += step * depth[:, -1, 0]
        if frustum:
            points[0, :] *= -0.1 / points[0, :, 2:]
            points[-1, :] *= -0.1 / points[-1, :, 2:]
            points[:, 0] *= -0.1 / points[:, 0, 2:]
            points[:, -1] *= -0.1 / points[:, -1, 2:]
        ring = np.zeros_like(depth, dtype=bool)
        ring[0, :] = ring[-1, :] = ring[:, 0] = ring[:, -1] = True
        n += 2
    else:
        ring = np.zeros_like(depth, dtype=bool)
    faces = triangulate(points)
    points = points.reshape(-1, 3); uv = uv.reshape(-1, 2)
    if cal_normal:
        normal = normal.reshape(-1, 3)
    depth = depth.reshape(-1, 1); ring = ring.reshape(-1, 1)
    disc = np.zeros_like(depth, dtype=bool)
    if atol is not None or rtol is not None:
        m = mask_discontinuity(faces, depth, 0 if atol is None else atol, 0 if rtol is None else rtol)
        disc[faces[m, :]] = True
    if modelview is not None:
        inv = inverse(modelview)
        points = (inv @ np.concatenate([points, np.ones((points.shape[0], 1))], axis=-1).T).T[:, :3]
        if cal_normal:
            normal = (inv[:3, :3] @ normal.T).T
    ero = np.zeros_like(depth, dtype=bool)
    if erode_rgb is not None and erode_rgb > 0:
        keep = np.ones_like(disc, dtype=np.float32)
        keep[disc] = 0
        k = 2 * erode_rgb + 1
        keep = cv2.erode(keep.reshape(n, n), np.ones((k, k))).reshape(-1, 1)
        ero[keep == 0] = True
    ret["faces"] = faces
    ret["vertices"] = AttrDict(position=points, uv=uv, flag=1 * disc + 2 * ring + 4 * ero)
    if cal_normal:
        ret["vertices"]["normal"] = normal
    return ret


def depth_edge(depth, atol=0.02, rtol=0.02):
    def differs(a, b):
        a = np.maximum(a, 1e-6); b = np.maximum(b, 1e-6)
        return np.logical_and(np.abs(a - b) > atol, np.abs(1 / a - 1 / b) > rtol)
    hits = np.zeros((depth.shape[0], depth.shape[1], 1), dtype=np.uint8)
    for (sa, sb) in [((slice(None), slice(1, None)), (slice(None), slice(None, -1))),
                     ((slice(1, None), slice(None)), (slice(None, -1), slice(None))),
                     ((slice(1, None), slice(1, None)), (slice(None, -1), slice(None, -1))),
                     ((slice(1, None), slice(None, -1)), (slice(None, -1), slice(1, None)))]:
        m = differs(depth[sa], depth[sb])
        hits[sa] += m
        hits[sb] += m
    return hits < 3


def mesh_vertex_buffer(mesh) -> np.ndarray:
    """float32 [V, 9]: position, normal, uv, flag — the VBO layout of moderngl_renderer.py:284-289."""
    v = mesh["vertices"]
    return np.ascontiguousarray(np.concatenate([v["position"], v["normal"], v["uv"], v["flag"]], axis=-1).astype(np.float32))


# ----------------------------------------------------------------------------------------------------------------------
# software AggregationRenderer (C restatement of the GL pipeline)
# ----------------------------------------------------------------------------------------------------------------------
def build_lib(force=False) -> str:
    out_dir = os.path.join(HERE, "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libraster_ref.so")
    src = os.path.join(HERE, "raster_ref.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-std=c99", src, "-o", so, "-lm"])
    return so


def _lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build_lib())
    return _LIB


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class SoftwareAggregationRenderer:
    """AggregationRenderer (moderngl_renderer.py:151-340) on the CPU; same constructor and .render() contract."""

    def __init__(self, render_size=128, image_size=128, near=0.01, far=200.0, device=0, max_views=27):
        self.render_size, self.image_size, self.near, self.far, self.max_views = render_size, image_size, near, far, max_views

    def render(self, meshes, colors, modelview, fov=45.0, is_autoregressive=False, **_):
        S, T = self.render_size, self.image_size
        L = _lib()
        proj = perspective(np.deg2rad(fov), 1, self.near, self.far)
        mvp = np.ascontiguousarray((proj.astype(np.float64) @ np.asarray(modelview, dtype=np.float64)).astype(np.float32))
        agg_c = np.zeros((S * S, 4), np.float32); agg_d = np.zeros((S * S, 2), np.float32); agg_m = np.zeros((S * S, 2), np.float32)
        cfb = np.zeros((S * S, 4), np.float32); dfb = np.zeros((S * S,), np.float32)
        for mesh, col in zip(meshes, colors):
            vb = mesh_vertex_buffer(mesh)
            faces = np.ascontiguousarray(mesh["faces"].astype(np.uint32))
            tex = np.ascontiguousarray(col.astype(np.float32))
            cam = np.ascontiguousarray(inverse(mesh["modelview"])[:3, 3].astype(np.float32))
            L.raster_draw_mesh(_fp(vb), vb.shape[0], _fp(faces), faces.shape[0], _fp(tex), T, _fp(mvp), _fp(cam), S, _fp(cfb), _fp(dfb))
            L.raster_aggregate(_fp(cfb), _fp(dfb), S, _fp(agg_c), _fp(agg_d), _fp(agg_m))
        # read-back / resolve (moderngl_renderer.py:318-331); framebuffer row 0 is the bottom row
        pix = np.flip(agg_c.reshape(S, S, 4), axis=0)
        color = np.where(pix[:, :, 3:] > 0.0, pix[:, :, :3] / np.maximum(pix[:, :, 3:], 1e-24), 0.0)
        d = np.flip(agg_d.reshape(S, S, 2), axis=0)
        depth = np.where(d[:, :, 1:] > 0.0, d[:, :, :1] / np.maximum(d[:, :, 1:], 1e-24), 0.0)
        depth = (self.near * self.far / (self.far - depth * (self.far - self.near))).astype(np.float32)
        m = np.flip(agg_m.reshape(S, S, 2), axis=0)
        return AttrDict(color=color, depth=depth, mask_color=m[:, :, 1:] > 0.5, mask_depth=m[:, :, :1] > 0.5)


class SoftwareSimpleRenderer:
    """SimpleRenderer (moderngl_renderer.py:11-148, shaders/simple.{vsh,fsh}) on the CPU: one mesh, raw texture colours,
    alpha = 0 on discontinuity edges and back faces; single modelview per call."""

    def __init__(self, render_size=128, image_size=128, near=0.01, far=200.0, device=0):
        self.render_size, self.image_size, self.near, self.far = render_size, image_size, near, far

    def render(self, mesh, color, modelview, fov=45.0):
        S, T = self.render_size, self.image_size
        proj = perspective(np.deg2rad(fov), 1, self.near, self.far)
        mvp = np.ascontiguousarray((proj.astype(np.float64) @ np.asarray(modelview, dtype=np.float64)).astype(np.float32))
        v = mesh["vertices"]
        vb = np.ascontiguousarray(np.concatenate([v["position"], v["uv"], v["flag"]], axis=-1).astype(np.float32))
        faces = np.ascontiguousarray(mesh["faces"].astype(np.uint32))
        tex = np.ascontiguousarray(np.asarray(color).astype(np.float32))
        cfb = np.zeros((S * S, 4), np.float32); dfb = np.zeros((S * S,), np.float32)
        _lib().raster_draw_simple(_fp(vb), vb.shape[0], _fp(faces), faces.shape[0], _fp(tex), T, _fp(mvp), S, _fp(cfb), _fp(dfb))
        pix = np.flip(cfb.reshape(S, S, 4), axis=0)
        depth = dfb.reshape(S, S, 1)
        depth = self.near * self.far / (self.far - depth * (self.far - self.near))
        depth = np.flip(depth, axis=0).astype(np.float32)
        return AttrDict(color=pix[:, :, :3], depth=depth, mask=pix[:, :, 3:] > 0.5)


def forward_backward_warp(renderer, rgbd, modelview1, modelview0=None, padding=None, fov=45, near=0.5, far=100, atol=0.02, rtol=0.02):
    """forward_backward_warp (utils.py:335-417): view0 RGBD -> mesh -> rendered at view1 -> re-meshed -> rendered back at
    view0; what survives both trips (and is not a depth edge) is the partial condition of a training pair."""
    n = rgbd.shape[0]
    ssaa = renderer.render_size // n
    off = (ssaa - 1) // 2
    if modelview0 is None:
        modelview0 = view_on_sphere(0.0, 0.0)
    resolve = lambda c: np.array(Image.fromarray(to8b(c)).resize((n, n), Image.Resampling.LANCZOS)) / 255.0
    mesh0 = depth_to_mesh(linearize_depth(rgbd[:, :, 3:], near, far), fov=fov, modelview=modelview0, padding=padding, cal_normal=False)
    res = renderer.render(mesh0, rgbd[:, :, :3], modelview1, fov)
    color1 = resolve(res.color)
    depth1 = res.depth[off::ssaa, off::ssaa, :]
    mesh1 = depth_to_mesh(depth1, fov=fov, modelview=modelview1, atol=atol, rtol=rtol, padding=None, cal_normal=False)
    res = renderer.render(mesh1, color1, modelview0, fov)
    color = resolve(res.color)
    depth = project_depth(res.depth[off::ssaa, off::ssaa, :], near, far)
    mask = res.mask.reshape(n, ssaa, n, ssaa, 1).sum(axis=(1, 3)) > 0.75 * ssaa ** 2
    mask &= depth_edge(depth, atol=atol, rtol=rtol)
    color *= mask
    depth *= mask
    return AttrDict(color=color, depth=depth, mask=mask.astype(np.float32))


def to8b(x):
    return (np.clip(x, 0, 1) * 255).astype(np.uint8)


def aggregate_conditions(renderer, meshes, colors, modelview, fov=45, near=0.5, far=100, atol=0.02, rtol=0.02, erode_rgb=2):
    """aggregate_conditions (utils.py:420-477)."""
    n = colors[0].shape[0]
    ssaa = renderer.render_size // n
    off = (ssaa - 1) // 2
    res = renderer.render(meshes, colors, modelview, fov, is_autoregressive=True)
    color = np.array(Image.fromarray(to8b(res.color)).resize((n, n), Image.Resampling.LANCZOS)) / 255.0
    depth = project_depth(res.depth[off::ssaa, off::ssaa, :], near, far)
    vote = lambda m: m.reshape(n, ssaa, n, ssaa, 1).sum(axis=(1, 3)) > 0.75 * ssaa ** 2
    mask, mask_rgb = vote(res.mask_depth), vote(res.mask_color)
    convex = depth.copy()
    mask &= depth_edge(depth, atol=atol, rtol=rtol)
    k = 2 * erode_rgb - 1
    mask_rgb &= cv2.erode(mask.astype(np.uint8)[..., 0], np.ones((k, k), np.uint8), iterations=1)[..., None] > 0
    color *= mask_rgb
    depth *= mask
    return AttrDict(color=color, depth=depth, mask=mask.astype(np.float32), mask_rgb=mask_rgb.astype(np.float32), depth_convex=convex)

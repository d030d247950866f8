"""Mesh export of generated scenes: TSDF fusion of the RGBD views into a voxel grid and surface-nets extraction of a
coloured triangle mesh, both on the device (csrc/fusion.cu behind ivid_fusion_integrate / ivid_fusion_extract).

The rule is defined once in oracle/fusion_ref.py and the kernels follow it bit for bit:
  * a pixel is valid when depth_to_mesh(depth, padding=None, ...) flags it neither a discontinuity nor eroded (the device
    mesh build), its depth is > 0 and, when max_depth is given, <= max_depth;
  * the default grid spans the world points of the valid pixels: the longest bounding-box edge is `resolution` voxels and
    every side gets trunc + 1 voxels of margin;
  * each voxel takes min(1, sdf / (trunc * voxel)) from every view whose nearest pixel is valid and not more than
    trunc voxels in front of it, sdf = pixel depth - voxel depth; colour only within |sdf| <= trunc * voxel;
  * surface nets: one vertex per cell whose 8 corners were all seen and straddle the surface, one quad per sign-changing
    grid edge whose four cells have vertices, wound so that the normals point out of the surface, towards the cameras.
World coordinates are the scene's own (y up, cameras on the unit sphere looking at the origin).
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from .. import _lib
from ..utils import edict
from .glm_compat import as_matrix

__all__ = ["tsdf_integrate", "extract_surface", "fuse_views", "write_ply", "view_validity", "default_grid", "focal_length"]

_MAX_VOXELS = 2**31 - 2        # linear voxel indices are int32 on the device, one past the end included


def focal_length(fov) -> np.float32:
    """0.5 / tan(fov / 2) in float32: the focal length of csrc/warp.cu:cam_point in image widths."""
    return np.float32(0.5 / np.tan(0.5 * np.deg2rad(float(fov))))


def _grid(grid):
    origin = np.asarray(grid["origin"], np.float32).reshape(3)
    voxel = np.float32(grid["voxel"])
    dims = [int(d) for d in grid["dims"]]
    if len(dims) != 3 or min(dims) < 2:
        raise ValueError(f"grid dims must be three integers >= 2, got {dims}")
    if not (np.isfinite(voxel) and voxel > 0):
        raise ValueError(f"grid voxel size must be positive, got {voxel}")
    if not np.isfinite(origin).all():
        raise ValueError("grid origin must be finite")
    if dims[0] * dims[1] * dims[2] > _MAX_VOXELS:
        raise ValueError(f"a {dims[0]}x{dims[1]}x{dims[2]} grid has more voxels than a 32-bit index can address")
    g = _lib.FusionGridT()
    g.origin[:] = [float(o) for o in origin]
    g.voxel = float(voxel)
    g.dims[:] = dims
    return g, dims


def _check_trunc(trunc):
    if not (np.isfinite(trunc) and trunc > 0):
        raise ValueError(f"trunc must be positive, got {trunc}")


def default_grid(points, resolution=256, trunc=3):
    """edict(origin float32 [3], voxel float32, dims [3]) around float64 world points [P, 3], computed in float64: the
    longest bounding-box edge L gives voxel = L / resolution, origin = min - (trunc + 1) * voxel and
    dims = ceil(extent / voxel) + 2 (trunc + 1) on each axis.  Without points the grid covers the cube [-1, 1]^3 that
    holds the scene's cameras."""
    if int(resolution) != resolution or resolution < 1:
        raise ValueError(f"resolution must be a positive integer, got {resolution}")
    _check_trunc(trunc)
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    if pts.shape[0] == 0:
        pts = np.array([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]])
    lo, hi = pts.min(0), pts.max(0)
    extent = hi - lo
    voxel = extent.max() / resolution
    if not voxel > 0:
        raise ValueError("the valid pixels span no volume: all world points coincide")
    pad = trunc + 1
    dims = np.ceil(extent / voxel).astype(np.int64) + 2 * int(np.ceil(pad))
    return edict(origin=(lo - pad * voxel).astype(np.float32), voxel=np.float32(voxel), dims=[int(d) for d in dims])


def view_validity(depth, fov, modelview, max_depth=None, atol=0.03, rtol=0.03, erode_rgb=3):
    """bool [n, n]: the pixels fusion integrates (vertex flag 0 of the device depth_to_mesh with padding=None, depth > 0,
    depth <= max_depth when given)."""
    from .utils import depth_to_mesh
    d = np.asarray(depth, np.float32)
    n = d.shape[0]
    d = d.reshape(n, n)
    m = depth_to_mesh(d[..., None], padding=None, fov=fov, modelview=modelview, atol=atol, rtol=rtol, erode_rgb=erode_rgb)
    ok = (m.vertices.flag.reshape(n, n) == 0) & (d > 0)
    if max_depth is not None:
        ok &= d <= np.float32(max_depth)
    return ok


def world_points(depth, valid, fov, modelview):
    """float64 world points [P, 3] of the valid pixels of one view (the camera model of csrc/warp.cu:cam_point)."""
    n = depth.shape[0]
    c = (np.arange(n) + 0.5) / n
    focal = 0.5 / np.tan(0.5 * np.deg2rad(float(fov)))
    d = np.asarray(depth, np.float64).reshape(n, n)
    cam = np.stack([(c[None, :] - 0.5) / focal * d, (c[::-1][:, None] - 0.5) / focal * d, -d], axis=-1)[np.asarray(valid, bool)]
    inv = np.linalg.inv(as_matrix(modelview).astype(np.float64))
    return cam @ inv[:3, :3].T + inv[:3, 3]


def _device_plane(a, dtype, np_dtype, device):
    if torch.is_tensor(a):
        return a.to(device=device, dtype=dtype).contiguous()
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a).astype(np_dtype))).to(device)


def tsdf_integrate(depths, colors, valid, modelviews, fov, grid, trunc=3, device=None):
    """Fuse V views into the volumes of `grid` (see default_grid).  depths [V,n,n] (or [V,n,n,1]) linear, colors [V,n,n,3] in
    [0,1], valid bool [V,n,n], modelviews: V world -> camera matrices.  Returns edict of cuda float32 tensors
    tsdf_sum [dz,dy,dx], weight [dz,dy,dx], color_sum [dz,dy,dx,3], color_weight [dz,dy,dx] (the tsdf is
    tsdf_sum / weight where weight > 0)."""
    g, dims = _grid(grid)
    _check_trunc(trunc)
    if len(modelviews) < 1:
        raise ValueError("tsdf_integrate needs at least one view")
    mvs = np.ascontiguousarray(np.stack([as_matrix(m) for m in modelviews]).astype(np.float32))
    V = mvs.shape[0]
    dshape = tuple(depths.shape)
    n = dshape[1]
    if not (dshape[0] == V and len(dshape) in (3, 4) and dshape[2] == n and (len(dshape) == 3 or dshape[3] == 1)):
        raise ValueError(f"depths must be [V,n,n] or [V,n,n,1] with V = {V} views, got {dshape}")
    if tuple(colors.shape) != (V, n, n, 3):
        raise ValueError(f"colors must be [{V},{n},{n},3], got {tuple(colors.shape)}")
    if tuple(valid.shape) != (V, n, n):
        raise ValueError(f"valid must be [{V},{n},{n}], got {tuple(valid.shape)}")
    dev = torch.device("cuda", torch.cuda.current_device() if device is None else device)
    d = _device_plane(depths, torch.float32, np.float32, dev).reshape(V, n, n)
    c = _device_plane(colors, torch.float32, np.float32, dev)
    m = _device_plane(valid, torch.uint8, np.uint8, dev)
    dx, dy, dz = dims
    out = edict(tsdf_sum=torch.empty((dz, dy, dx), dtype=torch.float32, device=dev),
                weight=torch.empty((dz, dy, dx), dtype=torch.float32, device=dev),
                color_sum=torch.empty((dz, dy, dx, 3), dtype=torch.float32, device=dev),
                color_weight=torch.empty((dz, dy, dx), dtype=torch.float32, device=dev))
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ivid_fusion_integrate(_lib.ptr(d), _lib.ptr(m), _lib.ptr(c), mvs.ctypes.data, V, n,
                                                    float(focal_length(fov)), ctypes.byref(g), float(trunc), _lib.ptr(out.tsdf_sum),
                                                    _lib.ptr(out.weight), _lib.ptr(out.color_sum), _lib.ptr(out.color_weight),
                                                    _lib.cur_stream(dev)))
    return out


def extract_surface(volume, grid):
    """Surface nets over the volumes of tsdf_integrate -> edict(vertices float32 [N,3], colors uint8 [N,3], faces int64 [F,3]),
    cuda tensors.  Vertices are numbered in cell order and faces in edge order, so the mesh is a deterministic function of
    the volume."""
    g, dims = _grid(grid)
    dx, dy, dz = dims
    shapes = dict(tsdf_sum=(dz, dy, dx), weight=(dz, dy, dx), color_sum=(dz, dy, dx, 3), color_weight=(dz, dy, dx))
    for k, s in shapes.items():
        t = volume[k]
        if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == s):
            raise ValueError(f"volume.{k} must be a contiguous cuda float32 tensor of shape {s}")
    dev = volume["weight"].device
    vols = [volume[k] for k in shapes]
    nv, nf = ctypes.c_int64(), ctypes.c_int64()
    L = _lib.lib()
    with torch.cuda.device(dev):
        st = _lib.cur_stream(dev)
        _lib.check(L.ivid_fusion_extract(ctypes.byref(g), *[_lib.ptr(t) for t in vols], 0, 0, None, None, None, ctypes.byref(nv),
                                         ctypes.byref(nf), st))
        verts = torch.empty((nv.value, 3), dtype=torch.float32, device=dev)
        cols = torch.empty((nv.value, 3), dtype=torch.uint8, device=dev)
        faces = torch.empty((nf.value, 3), dtype=torch.int64, device=dev)
        if nv.value > 0:
            _lib.check(L.ivid_fusion_extract(ctypes.byref(g), *[_lib.ptr(t) for t in vols], nv.value, nf.value, _lib.ptr(verts),
                                             _lib.ptr(cols), _lib.ptr(faces), ctypes.byref(nv), ctypes.byref(nf), st))
    return edict(vertices=verts, colors=cols, faces=faces)


def fuse_views(depths, colors, modelviews, fov=45, resolution=256, trunc=3, max_depth=None, atol=0.03, rtol=0.03, erode_rgb=3,
               grid=None):
    """Fuse a scene's RGBD views into one coloured mesh.  depths [V,n,n] (or [V,n,n,1]) linear, colors [V,n,n,3] in [0,1],
    modelviews: V world -> camera matrices; the defaults of atol / rtol / erode_rgb are load_scene's.  `grid` (an edict
    like default_grid's) replaces the default grid over the valid pixels.
    Returns edict(vertices float32 [N,3], colors uint8 [N,3], faces int64 [F,3], origin, voxel, dims) on the host."""
    _check_trunc(trunc)
    if max_depth is not None and not max_depth > 0:
        raise ValueError(f"max_depth must be positive, got {max_depth}")
    depths = np.asarray(depths, np.float32)
    V, n = depths.shape[0], depths.shape[1]
    depths = depths.reshape(V, n, n)
    if len(modelviews) != V:
        raise ValueError(f"{V} depth maps but {len(modelviews)} modelviews")
    if grid is None and (int(resolution) != resolution or resolution < 1):
        raise ValueError(f"resolution must be a positive integer, got {resolution}")
    valid = np.stack([view_validity(depths[v], fov, modelviews[v], max_depth, atol, rtol, erode_rgb) for v in range(V)])
    if grid is None:
        pts = [world_points(depths[v], valid[v], fov, modelviews[v]) for v in range(V)]
        grid = default_grid(np.concatenate(pts, 0), resolution, trunc)
    vol = tsdf_integrate(depths, np.asarray(colors, np.float32), valid, modelviews, fov, grid, trunc)
    mesh = extract_surface(vol, grid)
    return edict(vertices=mesh.vertices.cpu().numpy(), colors=mesh.colors.cpu().numpy(), faces=mesh.faces.cpu().numpy(),
                 origin=np.asarray(grid["origin"], np.float32), voxel=np.float32(grid["voxel"]), dims=[int(d) for d in grid["dims"]])


def write_ply(path, mesh):
    """Binary little-endian PLY: float x, y, z and uchar red, green, blue per vertex; a uchar-counted int list per face."""
    v = np.asarray(mesh["vertices"], np.float32).reshape(-1, 3)
    c = np.asarray(mesh["colors"], np.uint8).reshape(-1, 3)
    f = np.asarray(mesh["faces"]).reshape(-1, 3)
    if c.shape[0] != v.shape[0]:
        raise ValueError(f"{v.shape[0]} vertices but {c.shape[0]} colours")
    if f.size and (f.min() < 0 or f.max() >= v.shape[0]):
        raise ValueError("face indices out of range")
    vrec = np.empty(v.shape[0], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    vrec["x"], vrec["y"], vrec["z"] = v[:, 0], v[:, 1], v[:, 2]
    vrec["red"], vrec["green"], vrec["blue"] = c[:, 0], c[:, 1], c[:, 2]
    frec = np.empty(f.shape[0], dtype=[("n", "u1"), ("i", "<i4", (3,))])
    frec["n"] = 3
    frec["i"] = f.astype(np.int32)
    header = (f"ply\nformat binary_little_endian 1.0\nelement vertex {v.shape[0]}\n"
              "property float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              f"element face {f.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vrec.tobytes())
        fh.write(frec.tobytes())

"""Analytic test scene of the mesh export: a sphere of radius 0.3 at the origin in front of the plane z = -1.5, seen by the
27 cameras of the 3x9 view set, with depth maps ray-traced in float64.  The sphere's silhouettes against the plane are
depth discontinuities, so every view has invalid pixels along them."""
import numpy as np

from ivid_b200.inference import build_modelviews
from ivid_b200.utils import edict
from oracle import warp_ref

RADIUS = 0.3
PLANE_Z = -1.5
FOV = 45


def ray_trace(modelview, n, fov=FOV, sphere=True):
    """(linear depth float32 [n,n], colour float32 [n,n,3], hit id [n,n]: 0 none, 1 sphere, 2 plane) of one camera."""
    inv = np.linalg.inv(np.asarray(modelview, np.float64))
    c = (np.arange(n) + 0.5) / n
    focal = 0.5 / np.tan(0.5 * np.deg2rad(fov))
    u = np.broadcast_to(c[None, :], (n, n)); v = np.broadcast_to(c[::-1][:, None], (n, n))
    dcam = np.stack([(u - 0.5) / focal, (v - 0.5) / focal, -np.ones((n, n))], axis=-1)
    D = dcam @ inv[:3, :3].T                   # world direction per unit of linear depth
    C = inv[:3, 3]
    a = (D * D).sum(-1); b = 2 * (D @ C); cc = C @ C - RADIUS ** 2
    disc = b * b - 4 * a * cc
    with np.errstate(invalid="ignore"):
        t_s = (-b - np.sqrt(disc)) / (2 * a)
    t_s = np.where(sphere & (disc >= 0) & (t_s > 0), t_s, np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        t_p = (PLANE_Z - C[2]) / D[..., 2]
    t_p = np.where(t_p > 0, t_p, np.inf)
    t = np.minimum(t_s, t_p)
    hit = np.where(np.isinf(t), 0, np.where(t_s <= t_p, 1, 2))
    depth = np.where(np.isinf(t), 0.0, t)
    P = C + D * depth[..., None]
    sphere_col = 0.5 + 0.5 * P / RADIUS
    checker = ((np.floor(P[..., 0] * 4) + np.floor(P[..., 1] * 4)) % 2)[..., None]
    plane_col = np.where(checker > 0, [0.9, 0.8, 0.3], [0.2, 0.3, 0.7])
    col = np.where((hit == 1)[..., None], sphere_col, np.where((hit == 2)[..., None], plane_col, 0.0))
    return depth.astype(np.float32), np.clip(col, 0, 1).astype(np.float32), hit


def scene(n=64, views=None, sphere=True):
    mvs = build_modelviews("3x9", 1) if views is None else views
    traced = [ray_trace(m, n, sphere=sphere) for m in mvs]
    return edict(depths=np.stack([t[0] for t in traced]), colors=np.stack([t[1] for t in traced]), hits=np.stack([t[2] for t in traced]),
                 modelviews=[np.asarray(m, np.float32) for m in mvs], fov=FOV)


def oracle_validity(depth, modelview, fov=FOV, atol=0.03, rtol=0.03, erode_rgb=3, max_depth=None):
    """The validity rule on the numpy depth_to_mesh of oracle/warp_ref.py (the device mesh build matches its flags exactly)."""
    n = depth.shape[0]
    m = warp_ref.depth_to_mesh(np.asarray(depth, np.float32).reshape(n, n, 1), fov=fov, modelview=modelview, atol=atol, rtol=rtol,
                               erode_rgb=erode_rgb, padding=None, cal_normal=False)
    ok = (m.vertices.flag.reshape(n, n) == 0) & (depth > 0)
    if max_depth is not None:
        ok &= depth <= np.float32(max_depth)
    return ok


def surface_distance(p):
    """Distance of world points [N,3] to the nearer of the two surfaces, and which one (1 sphere, 2 plane)."""
    ds = np.abs(np.linalg.norm(p, axis=-1) - RADIUS)
    dp = np.abs(p[:, 2] - PLANE_Z)
    return np.minimum(ds, dp), np.where(ds <= dp, 1, 2)


def read_ply(path):
    """(vertices float32 [N,3], colours uint8 [N,3], faces int64 [F,3]) of a PLY written by rgbd_3d.fusion.write_ply."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").splitlines()
    assert lines[:2] == ["ply", "format binary_little_endian 1.0"]
    nv = int(lines[2].split()[-1]); nf = int([ln for ln in lines if ln.startswith("element face")][0].split()[-1])
    assert lines[3:9] == ["property float x", "property float y", "property float z", "property uchar red", "property uchar green",
                          "property uchar blue"]
    assert lines[10] == "property list uchar int vertex_indices" and lines[-1] == "end_header"
    vt = np.dtype([("p", "<f4", (3,)), ("c", "u1", (3,))])
    v = np.frombuffer(data, vt, nv, end)
    ft = np.dtype([("n", "u1"), ("i", "<i4", (3,))])
    f = np.frombuffer(data, ft, nf, end + nv * vt.itemsize)
    assert (f["n"] == 3).all() and end + nv * vt.itemsize + nf * ft.itemsize == len(data)
    return v["p"], v["c"], f["i"].astype(np.int64)

"""ORACLE (test infrastructure only — never imported by the product path).

The definition of mesh export by TSDF fusion, in numpy float32.  The reference has no fusion, so this is not a
restatement of it: it is the rule that csrc/fusion.cu follows operation for operation (compiled with -fmad=false), so
the device volumes and meshes equal what these functions return, bit for bit.

  grid      an input (origin float32 [3], voxel float32, dims [3]); the product derives its default from the valid
            pixels (ivid_b200/rgbd_3d/fusion.py:default_grid), so the two never have to agree on computing it
  integrate one pass per voxel over the views in index order; fp32 sums, divided only at extraction (`integrate`)
  extract   surface nets: a vertex per active cell (mean of the edge zero crossings in the order of EDGES), one quad per
            sign-changing grid edge whose four cells are active; vertices in cell order, faces in edge order (`extract`)

Camera model (csrc/warp.cu:cam_point): pixel (r, c) of an n x n view looks along u = (c + 0.5) / n,
v = (n - 1 - r + 0.5) / n with focal = 0.5 / tan(fov / 2), the camera looking down -z; depth is the linear depth -z.
Volumes are indexed [k, j, i] (x fastest); voxel (i, j, k) is centred at origin + ((i, j, k) + 0.5) * voxel.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32

# the 12 edges of a cell as (corner a, corner b); corner q sits at offset (q & 1, q >> 1 & 1, q >> 2); x edges, y edges,
# z edges, and corner a is always the lower end
EDGES = [(0, 1), (2, 3), (4, 5), (6, 7), (0, 2), (1, 3), (4, 6), (5, 7), (0, 4), (1, 5), (2, 6), (3, 7)]


def focal_length(fov) -> np.float32:
    return f32(0.5 / np.tan(0.5 * np.deg2rad(float(fov))))


def integrate(depths, colors, valid, modelviews, fov, origin, voxel, dims, trunc):
    """-> (tsdf_sum [dz,dy,dx], weight [dz,dy,dx], color_sum [dz,dy,dx,3], color_weight [dz,dy,dx]), all float32.
    depths [V,n,n] linear, colors [V,n,n,3], valid bool [V,n,n], modelviews [V,4,4] row-major world -> camera."""
    depths = np.asarray(depths, f32); colors = np.asarray(colors, f32); valid = np.asarray(valid, bool)
    V, n = depths.shape[0], depths.shape[1]
    depths = depths.reshape(V, n, n); colors = colors.reshape(V, n, n, 3); valid = valid.reshape(V, n, n)
    dx, dy, dz = (int(d) for d in dims)
    origin = np.asarray(origin, f32); voxel = f32(voxel)
    focal, nf, tv = focal_length(fov), f32(n), f32(trunc) * voxel
    x = (origin[0] + (np.arange(dx, dtype=f32) + f32(0.5)) * voxel)[None, None, :]
    y = (origin[1] + (np.arange(dy, dtype=f32) + f32(0.5)) * voxel)[None, :, None]
    z = (origin[2] + (np.arange(dz, dtype=f32) + f32(0.5)) * voxel)[:, None, None]
    shape = (dz, dy, dx)
    tsum = np.zeros(shape, f32); w = np.zeros(shape, f32); csum = np.zeros(shape + (3,), f32); cw = np.zeros(shape, f32)
    for v in range(V):
        M = np.asarray(modelviews[v], f32)
        cz = ((M[2, 0] * x + M[2, 1] * y) + M[2, 2] * z) + M[2, 3]
        sel = np.nonzero((cz < 0).ravel())[0]
        if sel.size == 0:
            continue
        X = np.broadcast_to(x, shape).ravel()[sel]; Y = np.broadcast_to(y, shape).ravel()[sel]; Z = np.broadcast_to(z, shape).ravel()[sel]
        dist = -cz.ravel()[sel]
        cx = ((M[0, 0] * X + M[0, 1] * Y) + M[0, 2] * Z) + M[0, 3]
        cy = ((M[1, 0] * X + M[1, 1] * Y) + M[1, 2] * Z) + M[1, 3]
        with np.errstate(over="ignore", invalid="ignore"):
            col = np.floor(((cx / dist) * focal + f32(0.5)) * nf)
            rowv = np.floor(((cy / dist) * focal + f32(0.5)) * nf)
        inside = (col >= 0) & (col < nf) & (rowv >= 0) & (rowv < nf)
        sel, dist, col, rowv = sel[inside], dist[inside], col[inside].astype(np.int64), rowv[inside].astype(np.int64)
        r = n - 1 - rowv
        ok = valid[v, r, col]
        sel, dist, r, col = sel[ok], dist[ok], r[ok], col[ok]
        sdf = depths[v, r, col] - dist
        ok = ~(sdf < -tv)
        sel, sdf, r, col = sel[ok], sdf[ok], r[ok], col[ok]
        # each voxel appears once in `sel`, so the fancy-index updates are plain per-voxel adds
        tsum.ravel()[sel] += np.minimum(f32(1), sdf / tv)
        w.ravel()[sel] += f32(1)
        near = np.abs(sdf) <= tv
        cw.ravel()[sel[near]] += f32(1)
        csum.reshape(-1, 3)[sel[near]] += colors[v, r[near], col[near]]
    return tsum, w, csum, cw


def tsdf(tsum, w):
    """The fused tsdf (float32, NaN where no view wrote)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(w > 0, tsum / np.where(w > 0, w, f32(1)), f32(np.nan)).astype(f32)


def _corner(a, q):
    """corner q of every cell of a voxel array [dz,dy,dx,...] -> [dz-1,dy-1,dx-1,...]"""
    i, j, k = q & 1, (q >> 1) & 1, q >> 2
    dz, dy, dx = a.shape[:3]
    return a[k:k + dz - 1, j:j + dy - 1, i:i + dx - 1]


def extract(tsum, w, csum, cw, origin, voxel):
    """Surface nets -> (vertices float32 [N,3], colors uint8 [N,3], faces int64 [F,3])."""
    tsum, w, csum, cw = (np.asarray(a, f32) for a in (tsum, w, csum, cw))
    origin = np.asarray(origin, f32); voxel = f32(voxel)
    dz, dy, dx = w.shape
    T = tsdf(tsum, w)
    has = w > 0
    inside = T < 0
    corners_ok = np.ones((dz - 1, dy - 1, dx - 1), bool)
    nin = np.zeros((dz - 1, dy - 1, dx - 1), np.int64)
    for q in range(8):
        corners_ok &= _corner(has, q)
        nin += _corner(inside, q)
    active = corners_ok & (nin != 0) & (nin != 8)
    ck, cj, ci = np.nonzero(active)                      # C order: cell linear order, x fastest
    Tc = [_corner(T, q)[active] for q in range(8)]
    s = [np.zeros(ck.size, f32) for _ in range(3)]
    cnt = np.zeros(ck.size, f32)
    for e, (qa, qb) in enumerate(EDGES):
        axis = e // 4
        cross = (Tc[qa] < 0) != (Tc[qb] < 0)
        with np.errstate(invalid="ignore", divide="ignore"):
            t = Tc[qa] / (Tc[qa] - Tc[qb])
        for d in range(3):
            val = t if d == axis else f32((qa >> d) & 1)
            s[d] = np.where(cross, s[d] + val, s[d])
        cnt = np.where(cross, cnt + f32(1), cnt)
    idx = (ci, cj, ck)
    verts = np.stack([origin[d] + ((idx[d].astype(f32) + f32(0.5)) + s[d] / cnt) * voxel for d in range(3)], axis=-1).astype(f32)
    rgb = np.zeros((ck.size, 3), f32)
    nc = np.zeros(ck.size, f32)
    for q in range(8):
        cwq = _corner(cw, q)[active]
        hasc = cwq > 0
        with np.errstate(invalid="ignore", divide="ignore"):
            cq = _corner(csum, q)[active] / np.where(hasc, cwq, f32(1))[:, None]
        rgb = np.where(hasc[:, None], rgb + cq, rgb)
        nc = np.where(hasc, nc + f32(1), nc)
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = np.where(nc[:, None] > 0, rgb / np.where(nc > 0, nc, f32(1))[:, None], f32(0))
    colors = np.floor(np.clip(mean, f32(0), f32(1)) * f32(255) + f32(0.5)).astype(np.uint8)

    # vertex id of every cell, padded by one inactive (-1) cell on each side so cell (k+dk, j+dj, i+di) of voxel (k, j, i)
    # is P[1+dk : 1+dk+dz, 1+dj : 1+dj+dy, 1+di : 1+di+dx]
    P = np.full((dz + 1, dy + 1, dx + 1), -1, np.int64)
    P[1:dz, 1:dy, 1:dx] = np.where(active, np.cumsum(active.ravel()).reshape(active.shape) - 1, -1)
    cell = lambda dk, dj, di: P[1 + dk:1 + dk + dz, 1 + dj:1 + dj + dy, 1 + di:1 + di + dx]
    ins_pad = np.zeros((dz + 1, dy + 1, dx + 1), bool)
    ins_pad[:dz, :dy, :dx] = inside & has
    quads = []
    for axis in range(3):
        u, v = (axis + 1) % 3, (axis + 2) % 3
        ids = []
        for du, dv in ((-1, -1), (0, -1), (0, 0), (-1, 0)):           # c00, c10, c11, c01
            off = [0, 0, 0]                                           # (di, dj, dk) by axis x, y, z
            off[u] += du; off[v] += dv
            ids.append(cell(off[2], off[1], off[0]))
        step = [0, 0, 0]; step[axis] = 1
        ia = ins_pad[:dz, :dy, :dx]
        ib = ins_pad[step[2]:step[2] + dz, step[1]:step[1] + dy, step[0]:step[0] + dx]
        q = (ids[0] >= 0) & (ids[1] >= 0) & (ids[2] >= 0) & (ids[3] >= 0) & (ia != ib)
        quads.append((q, ia, ids))
    emit = np.stack([q for q, _, _ in quads], axis=-1)                # [dz,dy,dx,3]: edge linear order
    vk, vj, vi, va = np.nonzero(emit)
    faces = np.zeros((vk.size * 2, 3), np.int64)
    for axis in range(3):
        q, ia, ids = quads[axis]
        m = va == axis
        sel = (vk[m], vj[m], vi[m])
        c00, c10, c11, c01 = (a[sel] for a in ids)
        out = ia[sel]
        rows = np.nonzero(m)[0] * 2
        faces[rows] = np.where(out[:, None], np.stack([c00, c10, c11], -1), np.stack([c00, c11, c10], -1))
        faces[rows + 1] = np.where(out[:, None], np.stack([c00, c11, c01], -1), np.stack([c00, c01, c11], -1))
    return verts, colors, faces

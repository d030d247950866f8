"""A CPU mirror of the warp rasteriser's vertex stage and per-triangle decisions, and the crafted scenes that test it
(test infrastructure, no GPU).

csrc/warp.cu rasterises each face as follows. Its vertex stage is fp32 (`load_vertex`, `clip_near`, `tri_setup`), with
P*MV formed on the host by `upload_mvp`. `rtri_make` sets up each sub-triangle: the snapped window coordinates, the
edge coefficients, the tie bits and the pixel box. `rtri_raster` then sends it down one of three scans:
  * small32: a box of at most 48 pixels whose edge coefficients fit 15 bits and whose first-pixel edge values fit 29 bits.
    The edge values are evaluated once in 64 bits and stepped in int32 (`rtri_scan_small32`);
  * small64: the same small box when they do not fit. Every pixel is evaluated in 64 bits (`rtri_pixel`);
  * big: the warp takes the box over. Its 8x8 tiles are culled by an exact `emax < 0` corner test, and the survivors
    are scanned two pixels per lane.
Thread f of `raster_kernel` draws face (f * 7919) mod F. A face cut by the near plane becomes a 4-vertex polygon; its
second sub-triangle (poly0, poly2, poly3, primitive id 2 fi + 1) waits in shared memory for a second round.

This module restates all of that in numpy float32 and Python integers, in the kernel's operation order, so that a test
can place a vertex exactly on a chosen 1/256-pixel point and can say which scan path, tile and warp a case reaches.
The scenes are packed into the fixed grid layout that `ivid_warp_set_mesh` and `ivid_warp_render_simple` take. A
palette texture, with every uv at a texel centre, makes each face's colour name the face.

It also holds the colour bound of the aggregation renderer (`colour_bound`). Coverage, visibility and depth are
exact on both sides. Colour with several source views is not, because the shading weight calls `acosf` and `expf`.
"""
from __future__ import annotations

import math
from collections import Counter
from dataclasses import dataclass, field

import numpy as np

from oracle.warp_ref import _TANF

F32 = np.float32
PERM = 7919                 # raster_kernel's face permutation
SMALL_BOX = 48              # rtri_raster: boxes of more pixels are big
NEAR, FAR = 0.01, 200.0     # the renderers' default planes
ORIENTS = ("dy>0", "dy<0", "dy=0,dx<0", "dy=0,dx>0")   # the cases the tie rule distinguishes (sign-adjusted edge)
TIE_OK = {"dy>0": True, "dy<0": False, "dy=0,dx<0": True, "dy=0,dx>0": False}
PATHS = ("small32", "small64", "big")


# ----------------------------------------------------------------------------------------------------------------------
# vertex stage
# ----------------------------------------------------------------------------------------------------------------------
def upload_mvp(mv, fov_deg=45.0, near=NEAR, far=FAR) -> np.ndarray:
    """P*MV as Warp::upload_mvp forms it: P in fp32 (tanf of the fp32 half angle), the product in double, rounded to fp32."""
    half = F32(fov_deg * (math.pi / 180.0)) / F32(2)
    t = F32(_TANF(float(half)))
    nf, ff = F32(near), F32(far)
    P = [0.0] * 16
    P[0] = float(F32(1) / (F32(1) * t))
    P[5] = float(F32(1) / t)
    P[10] = float(-(ff + nf) / (ff - nf))
    P[11] = float(-(F32(2) * ff * nf) / (ff - nf))
    P[14] = -1.0
    m = [float(x) for x in np.asarray(mv, dtype=np.float32).reshape(16)]
    out = np.zeros(16, np.float32)
    for r in range(4):
        for c in range(4):
            s = 0.0
            for k in range(4):
                s += P[r * 4 + k] * m[k * 4 + c]
            out[r * 4 + c] = F32(s)
    return out.reshape(4, 4)


def clip_coords(mvp, pos) -> np.ndarray:
    """load_vertex: clip[r] = ((m0 a0 + m1 a1) + m2 a2) + m3 in fp32.  pos [..., 3] -> [..., 4]."""
    a = np.asarray(pos, np.float32)
    m = np.asarray(mvp, np.float32)
    return np.stack([((m[r, 0] * a[..., 0] + m[r, 1] * a[..., 1]) + m[r, 2] * a[..., 2]) + m[r, 3] for r in range(4)], axis=-1)


def window(clip, S):
    """tri_setup: the divide, the viewport and the snap floor(xw * 256 + 0.5).  -> (X, Y) int64, zw, iw (fp32)."""
    c = np.asarray(clip, np.float32)
    w = c[..., 3]
    xn, yn, zn = c[..., 0] / w, c[..., 1] / w, c[..., 2] / w
    xw = (xn * F32(0.5) + F32(0.5)) * F32(S)
    yw = (yn * F32(0.5) + F32(0.5)) * F32(S)
    X = np.floor(xw * F32(256) + F32(0.5)).astype(np.int64)
    Y = np.floor(yw * F32(256) + F32(0.5)).astype(np.int64)
    return X, Y, zn * F32(0.5) + F32(0.5), F32(1) / w


def place(mv, fov, S, X, Y, d, near=NEAR, far=FAR) -> np.ndarray:
    """World position (fp32) of a vertex at view distance d that the vertex stage snaps to (X, Y) in 1/256 pixel.
    The point is solved in float64 and then nudged by ulps until the fp32 stage puts it exactly there."""
    mvp = upload_mvp(mv, fov, near, far)
    p00, p11 = _p(fov)
    xn, yn = 2.0 * (X / 256.0) / S - 1.0, 2.0 * (Y / 256.0) / S - 1.0
    view = np.array([xn * d / p00, yn * d / p11, -d, 1.0])
    world = np.linalg.inv(np.asarray(mv, np.float64)) @ view
    base = world[:3].astype(np.float32)
    steps = [0, 1, -1, 2, -2, 3, -3]
    for dx in steps:
        for dy in steps:
            for dz in (0, 1, -1):
                p = base.copy()
                for k, s in enumerate((dx, dy, dz)):
                    for _ in range(abs(s)):
                        p[k] = np.nextafter(p[k], F32(np.inf) if s > 0 else F32(-np.inf))
                Xg, Yg, _, _ = window(clip_coords(mvp, p), S)
                if int(Xg) == X and int(Yg) == Y:
                    return p
    raise AssertionError(f"cannot place a vertex at ({X}, {Y}) / 256 px, d = {d}")


def _p(fov):
    half = F32(fov * (math.pi / 180.0)) / F32(2)
    t = F32(_TANF(float(half)))
    return float(F32(1) / (F32(1) * t)), float(F32(1) / t)


def centre(p) -> int:
    """1/256-pixel coordinate of the centre of pixel p."""
    return int(p) * 256 + 128


# ----------------------------------------------------------------------------------------------------------------------
# the kernel's decisions
# ----------------------------------------------------------------------------------------------------------------------
def clip_near(clip):
    """clip_near on the clip coordinates of a face ([3, 4] fp32) -> polygon [n, 4] with n in (0, 3, 4)."""
    d = [F32(clip[i, 2] + clip[i, 3]) for i in range(3)]
    if all(x >= 0 for x in d):
        return clip.copy()
    if all(x < 0 for x in d):
        return clip[:0]
    out = []
    for i in range(3):
        j = (i + 1) % 3
        if d[i] >= 0:
            out.append(clip[i])
        if (d[i] >= 0) != (d[j] >= 0):
            t = F32(d[i] / (d[i] - d[j]))
            out.append(clip[i] + (clip[j] - clip[i]) * t)
    return np.stack(out).astype(np.float32)


@dataclass
class SubTri:
    """rtri_make's record of one sub-triangle, plus what rtri_raster does with it."""
    X: list
    Y: list
    zw: np.ndarray
    area: int
    valid: bool
    path: str = ""
    box: tuple = ()
    ea: list = field(default_factory=list)
    eb: list = field(default_factory=list)
    ec: list = field(default_factory=list)
    tie: int = 0

    @property
    def sgn(self):
        return 1 if self.area > 0 else -1


def rtri_make(clip3, S) -> SubTri:
    X, Y, zw, _ = window(clip3, S)
    X, Y = [int(v) for v in X], [int(v) for v in Y]
    area = (X[1] - X[0]) * (Y[2] - Y[0]) - (Y[1] - Y[0]) * (X[2] - X[0])
    r = SubTri(X, Y, zw, area, False)
    if area == 0:
        return r
    sgn = r.sgn
    for i in range(3):
        a, c = (i + 1) % 3, (i + 2) % 3
        dx, dy = (X[c] - X[a]) * sgn, (Y[c] - Y[a]) * sgn
        r.ea.append(-dy)
        r.eb.append(dx)
        r.ec.append(-(-dy * X[a] + dx * Y[a]))
        if dy > 0 or (dy == 0 and dx < 0):
            r.tie |= 1 << i
    minx, maxx, miny, maxy = min(X), max(X), min(Y), max(Y)
    if maxx < 128 or maxy < 128:
        return r
    px0 = 0 if minx <= 128 else (minx - 128 + 255) // 256
    py0 = 0 if miny <= 128 else (miny - 128 + 255) // 256
    px1, py1 = min((maxx - 128) // 256, S - 1), min((maxy - 128) // 256, S - 1)
    if px0 > px1 or py0 > py1:
        return r
    r.box, r.valid = (px0, px1, py0, py1), True
    r.path = path_of(r)
    return r


def path_of(r: SubTri) -> str:
    """rtri_raster's choice of scan."""
    px0, px1, py0, py1 = r.box
    if (px1 - px0 + 1) * (py1 - py0 + 1) > SMALL_BOX:
        return "big"
    fit = all(-32768 < v < 32768 for v in r.ea + r.eb)
    cx0, cy0 = centre(px0), centre(py0)
    fit = fit and all(-(1 << 29) < r.ea[i] * cx0 + r.eb[i] * cy0 + r.ec[i] < (1 << 29) for i in range(3))
    return "small32" if fit else "small64"


def orient(r: SubTri, i) -> str:
    dx, dy = r.eb[i], -r.ea[i]
    if dy > 0:
        return "dy>0"
    if dy < 0:
        return "dy<0"
    return "dy=0,dx<0" if dx < 0 else "dy=0,dx>0"


def edge_values(r: SubTri):
    """(px, py, E [3, h, w]) over the box, exact int64."""
    px0, px1, py0, py1 = r.box
    py, px = np.mgrid[py0:py1 + 1, px0:px1 + 1].astype(np.int64)
    cx, cy = px * 256 + 128, py * 256 + 128
    E = np.stack([r.ea[i] * cx + r.eb[i] * cy + r.ec[i] for i in range(3)])
    return px, py, E


def coverage(r: SubTri):
    """Pixels whose centre the triangle owns: [(px, py)] and the per-edge inside tests."""
    px, py, E = edge_values(r)
    ins = np.stack([(E[i] > 0) | ((E[i] == 0) & bool((r.tie >> i) & 1)) for i in range(3)])
    cov = ins.all(0)
    return px, py, E, ins, cov


def tile_stats(r: SubTri):
    """The big scan's tile cull: (#culled, #kept, #kept tiles whose only covered pixel is a tie pixel at the corner where
    the tie edge's emax == 0)."""
    px0, px1, py0, py1 = r.box
    culled = kept = lone = 0
    px, py, E, ins, cov = coverage(r)
    for ty in range(py0 >> 3, (py1 >> 3) + 1):
        for tx in range(px0 >> 3, (px1 >> 3) + 1):
            x0, x1, y0, y1 = max(tx * 8, px0), min(tx * 8 + 7, px1), max(ty * 8, py0), min(ty * 8 + 7, py1)
            emax = [r.ea[i] * centre(x1 if r.ea[i] > 0 else x0) + r.eb[i] * centre(y1 if r.eb[i] > 0 else y0) + r.ec[i] for i in range(3)]
            if any(e < 0 for e in emax):
                culled += 1
                continue
            kept += 1
            sel = (px >= x0) & (px <= x1) & (py >= y0) & (py <= y1) & cov
            if sel.sum() == 1:
                j = np.argwhere(sel)[0]
                if any(emax[i] == 0 and E[i][tuple(j)] == 0 for i in range(3)):
                    lone += 1
    return culled, kept, lone


def tie_pixels(r: SubTri):
    """Counter of (orientation, sgn) -> pixels whose coverage the tie bit of that edge decides (E_i == 0, the other
    two edges inside)."""
    px, py, E, ins, cov = coverage(r)
    c = Counter()
    for i in range(3):
        others = ins[(i + 1) % 3] & ins[(i + 2) % 3]
        k = int(((E[i] == 0) & others).sum())
        if k:
            c[(orient(r, i), r.sgn)] += k
    return c


def depth_values(r: SubTri):
    """Window depth of every covered pixel, in rtri_cover's fp32 order."""
    px, py, E, ins, cov = coverage(r)
    farea = F32(r.sgn * r.area)
    l = [E[i][cov].astype(np.float32) / farea for i in range(3)]
    return (l[0] * r.zw[0] + l[1] * r.zw[1]) + l[2] * r.zw[2]


def face_plan(clip3, S):
    """raster_kernel for one face: (polygon size, first-round sub-triangle, second-round sub-triangle or None)."""
    poly = clip_near(clip3)
    n = len(poly)
    first = second = None
    if n == 4:
        s = rtri_make(poly[[0, 2, 3]], S)
        second = s if s.valid else None
    if n >= 3:
        first = rtri_make(poly[[0, 1, 2]], S)
    return n, first, second


def face_of_thread(f, F):
    return (f * PERM) % F


def thread_of_face(fi, F):
    return (fi * pow(PERM, -1, F)) % F


# ----------------------------------------------------------------------------------------------------------------------
# scenes
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class Tri:
    pos: np.ndarray             # [3, 3] fp32 world positions
    flag: int = 0               # vertex flag of all three vertices: 1 edge, 2 padding ring, 4 eroded
    nrm: np.ndarray = None      # [3, 3] vertex normals (None: towards +z)
    want: list = None           # [(X, Y)] * 3 the placement aimed at (None: not placed)
    tag: str = ""
    dup_of: int = -1            # index of the triangle it duplicates (same positions), or -1


def palette(n) -> np.ndarray:
    """n x n x 3 texture whose texels are pairwise distinct colours in (0, 1), recoverable by `texel_of`."""
    k = np.arange(n * n)
    rgb = np.stack([(k % 16 + 1) / 17.0, ((k // 16) % 16 + 1) / 17.0, (k // 256 + 1) / 17.0], axis=-1)
    return rgb.reshape(n, n, 3).astype(np.float32)


def texel_of(colour) -> np.ndarray:
    """Palette index of colours within a few ulps of a palette entry ([..., 3] -> [...])."""
    q = np.rint(np.asarray(colour, np.float64) * 17.0).astype(np.int64) - 1
    return q[..., 0] + 16 * q[..., 1] + 256 * q[..., 2]


@dataclass
class Scene:
    S: int
    n: int
    mv: np.ndarray
    fov: float
    tris: list
    threads: list = None        # raster thread of each triangle
    name: str = ""

    @property
    def F(self):
        return 2 * (self.n + 1) ** 2

    @property
    def V(self):
        return (self.n + 2) ** 2

    def faces_index(self):
        return [face_of_thread(t, self.F) for t in self.threads]

    def pack(self, uv_shift=0):
        """-> (vertex buffer [V, 9] fp32, faces [F, 3] uint32, texture [n, n, 3]).  Triangle k uses vertices 3k..3k+2 and
        the texel (k + uv_shift) mod n^2; unused faces are (0, 0, 0), which rtri_make rejects (zero area)."""
        n, V, F = self.n, self.V, self.F
        assert 3 * len(self.tris) <= V, "scene too large for the grid layout"
        vb = np.zeros((V, 9), np.float32)
        vb[:, 5] = 1.0
        faces = np.zeros((F, 3), np.uint32)
        for k, (t, fi) in enumerate(zip(self.tris, self.faces_index())):
            tex = (k + uv_shift) % (n * n)
            uv = np.float32([((tex % n) + 0.5) / n, ((tex // n) + 0.5) / n])
            for j in range(3):
                v = 3 * k + j
                vb[v, :3] = t.pos[j]
                vb[v, 3:6] = (0.0, 0.0, 1.0) if t.nrm is None else t.nrm[j]
                vb[v, 6:8] = uv
                vb[v, 8] = t.flag
            faces[fi] = (3 * k, 3 * k + 1, 3 * k + 2)
        return vb, faces, palette(n)

    def mesh(self, modelview=None, uv_shift=0):
        """The mesh dict both renderers take."""
        vb, faces, tex = self.pack(uv_shift)
        return dict(faces=faces, modelview=self.mv if modelview is None else modelview,
                    vertices=dict(position=vb[:, :3], normal=vb[:, 3:6], uv=vb[:, 6:8], flag=vb[:, 8:9])), tex

    def plans(self):
        mvp = upload_mvp(self.mv, self.fov)
        return [face_plan(clip_coords(mvp, t.pos), self.S) for t in self.tris]

    def check_placement(self):
        mvp = upload_mvp(self.mv, self.fov)
        for t in self.tris:
            if t.want is None:
                continue
            X, Y, _, _ = window(clip_coords(mvp, t.pos), self.S)
            assert [(int(a), int(b)) for a, b in zip(X, Y)] == [tuple(w) for w in t.want], (self.name, t.tag)


def assign_threads(scene: Scene):
    """Raster threads in order, one per triangle.  A duplicate goes to a later thread whose face index is lower than its
    original's: the earlier thread draws the higher face index, and the duplicate must still win, as it does in the
    oracle's sequential draw with a strict '<'."""
    F = scene.F
    threads, used = [], set()
    t = 0
    for k, tri in enumerate(scene.tris):
        if tri.dup_of >= 0:
            orig_fi = face_of_thread(threads[tri.dup_of], F)
            u = threads[tri.dup_of] + 1
            while u < F and (u in used or face_of_thread(u, F) >= orig_fi):
                u += 1
            assert u < F, "no later thread draws a lower face index"
            threads.append(u)
            used.add(u)
            continue
        has_dup = any(o.dup_of == k for o in scene.tris)
        while t in used or (has_dup and face_of_thread(t, F) < F // 2):
            t += 1
        threads.append(t)
        used.add(t)
    scene.threads = threads


# ---- case generators ------------------------------------------------------------------------------------------------
SMALL_SHAPES = [[(0, 0), (5, 0), (0, 5)], [(0, 0), (4, 2), (2, 5)], [(0, 0), (6, 0), (3, 3)]]
BIG_SHAPES = [[(0, 0), (20, 0), (0, 20)], [(0, 0), (24, 10), (6, 22)], [(0, 0), (24, 0), (12, 12)]]
SYMS = [lambda x, y: (x, y), lambda x, y: (-x, y), lambda x, y: (x, -y), lambda x, y: (-x, -y),
        lambda x, y: (y, x), lambda x, y: (-y, x), lambda x, y: (y, -x), lambda x, y: (-y, -x)]


def variants(shape):
    """The shape under the 8 symmetries of the square, both windings and the 3 rotations of its vertex order, so that
    every orientation of every edge lands in every edge slot of rtri_make, on front and back faces."""
    out = []
    for sym in SYMS:
        pts = [sym(x, y) for x, y in shape]
        mx, my = min(p[0] for p in pts), min(p[1] for p in pts)
        pts = [(x - mx, y - my) for x, y in pts]
        for wind in (pts, pts[::-1]):
            for rot in range(3):
                out.append(wind[rot:] + wind[:rot])
    return out


def _tri_px(scene_S, mv, fov, pts_px, depths, flag=0, tag="", nrm=None):
    """A triangle whose vertices sit exactly on the centres of the given pixels (window coordinates, y up)."""
    want = [(centre(x), centre(y)) for x, y in pts_px]
    pos = np.stack([place(mv, fov, scene_S, X, Y, d) for (X, Y), d in zip(want, depths)])
    return Tri(pos=pos, flag=flag, want=want, tag=tag, nrm=nrm)


def _cells(S, cell):
    k = max(1, S // cell)
    return [(i * cell, j * cell) for j in range(k) for i in range(k)]


def case_scenes(S, n, mv=None, fov=45.0, max_tris=None):
    """Every crafted case for render size S (texture / image size n), split into scenes that fit the grid layout."""
    mv = np.eye(4, dtype=np.float32) if mv is None else np.asarray(mv, np.float32)
    cap = (n + 2) ** 2 // 3 if max_tris is None else max_tris
    rng = np.random.default_rng(S)
    scenes = []

    def new(name):
        scenes.append(Scene(S, n, mv, fov, [], name=f"S{S}:{name}"))
        return scenes[-1]

    def add(sc, tri, name):
        if len(sc.tris) >= cap:
            sc = new(name)
        sc.tris.append(tri)
        return sc

    def depth3(k):
        base = 1.0 + 0.37 * (k % 7)
        return [base, base * 1.1, base * 1.23]

    # small32 and big: the shapes on pixel centres, one per cell, the next scene when the cells run out
    for kind, shapes, cell in (("small", SMALL_SHAPES, 8), ("big", BIG_SHAPES, 32)):
        cells = _cells(S, cell)
        sc, used, k = new(kind), 0, 0
        for shape in shapes:
            for v in variants(shape):
                if used == len(cells) or len(sc.tris) >= cap:
                    sc, used = new(kind), 0
                ox, oy = cells[used]
                used += 1
                pts = [(ox + x, oy + y) for x, y in v]
                flag = 2 if (k % 5 == 3) else 0
                sc.tris.append(_tri_px(S, mv, fov, pts, depth3(k), flag=flag, tag=kind))
                k += 1
    # big: a lone tie pixel at the corner of its tile where the tie edge's emax is 0 (both windings)
    sc = new("lone")
    c = 16 if S < 64 else 8 * (S // 16)
    for wind in (1, -1):
        pts = [(c - 8, c + 8), (c + 8, c - 8), (c - 24, c - 24)][::wind]
        sc = add(sc, _tri_px(S, mv, fov, pts, [2.0, 2.0, 2.0], tag="lone"), "lone")
        c2 = c + (8 if S >= 64 else 0)
        pts = [(c2 - 8, c2 + 8), (c2 + 8, c2 - 8), (c2 - 24, c2 - 24)][::wind]
        sc = add(sc, _tri_px(S, mv, fov, pts, [1.5, 1.5, 1.5], tag="lone"), "lone")
        sc = new("lone")
    # small64: giant triangles whose on-screen box is a few pixels at a screen corner (axis-aligned tie edges) or at
    # a border (a wedge whose tip is on a pixel centre); one scene per vertex order so the corners do not hide each other
    far_ = 3000
    L = S - 1
    corners = [((2, 2), (-far_, 2), (2, -far_)), ((L - 2, 2), (L + far_, 2), (L - 2, -far_)),
               ((2, L - 2), (-far_, L - 2), (2, L + far_)), ((L - 2, L - 2), (L + far_, L - 2), (L - 2, L + far_))]
    for wind in (1, -1):
        for rot in range(3):
            sc = new("small64")
            for j, tri in enumerate(corners):
                pts = list(tri[::wind])
                pts = pts[rot:] + pts[:rot]
                sc = add(sc, _tri_px(S, mv, fov, pts, [1.0 + 0.2 * j, 1.3, 1.6], tag="small64"), "small64")
            for j, y0 in enumerate(range(8, S - 8, 11)[:4]):
                tip = (1, y0)
                pts = [tip, (-far_, y0 - far_), (-far_, y0 + far_)][::wind]
                pts = pts[rot:] + pts[:rot]
                sc = add(sc, _tri_px(S, mv, fov, pts, [1.2, 1.4, 1.9], tag="small64"), "small64")
                tip = (L - 1, y0)
                pts = [tip, (L + far_, y0 + far_), (L + far_, y0 - far_)][::wind]
                pts = pts[rot:] + pts[:rot]
                sc = add(sc, _tri_px(S, mv, fov, pts, [1.2, 1.4, 1.9], tag="small64"), "small64")
    # generic triangles at arbitrary sub-pixel positions and depths, some overlapping, front and back, some padded
    sc = new("random")
    for k in range(min(cap, 24)):
        c0 = rng.uniform(0.1, 0.9, 2) * S * 256
        span = rng.choice([3, 12, 40]) * 256
        want = [(int(c0[0] + rng.uniform(-span, span)), int(c0[1] + rng.uniform(-span, span))) for _ in range(3)]
        ds = rng.uniform(0.8, 4.0, 3)
        pos = np.stack([place(mv, fov, S, X, Y, d) for (X, Y), d in zip(want, ds)])
        sc = add(sc, Tri(pos=pos, want=want, flag=int(rng.choice([0, 0, 2, 1, 4])), tag="random",
                         nrm=_normals(rng)), "random")
    # equal depth: duplicated faces (same positions, other uv) whose higher face index is drawn by the earlier thread
    sc = new("dup")
    for k, shape in enumerate([SMALL_SHAPES[0], BIG_SHAPES[1]]):
        o = 2 + 10 * k if S < 64 else 4 + 40 * k
        pts = [(o + x, o + y) for x, y in shape]
        sc.tris.append(_tri_px(S, mv, fov, pts, [1.5, 1.7, 2.1], tag="dup"))
        sc.tris.append(Tri(pos=sc.tris[-1].pos.copy(), want=sc.tris[-1].want, tag="dup", dup_of=len(sc.tris) - 1))
    y0 = S // 2
    orig = _tri_px(S, mv, fov, [(1, y0), (-far_, y0 + far_), (-far_, y0 - far_)], [1.2, 1.4, 1.9], tag="dup")
    sc.tris += [orig, Tri(pos=orig.pos.copy(), want=orig.want, tag="dup", dup_of=len(sc.tris))]
    # near plane: faces crossing it (4-vertex polygons with a small or a big second sub-triangle, duplicated as well),
    # two vertices behind it, all three behind it
    sc = new("near")
    for tri in near_cases(S, mv, fov, rng):
        sc = add(sc, tri, "near")
        if tri.tag == "near4":
            sc = add(sc, Tri(pos=tri.pos.copy(), tag="near4", dup_of=len(sc.tris) - 1), "near")
    # window depth <= 0 and >= 1: one vertex exactly on the near plane, one beyond the far plane
    sc = new("zrange")
    for k in range(3):
        o = 3 + 4 * k if S < 64 else 10 + 30 * k
        # the near vertex is the rightmost one, so the tie rule gives it its own pixel, whose depth is 0
        pts = [(o + 12, o + 6), (o, o + 1), (o + 2, o + 12)]
        ds = [NEAR, 320.0, 5.0] if k == 0 else ([5.0, 320.0, 400.0] if k == 1 else [NEAR, 2.0, 199.99])
        want = [(centre(x), centre(y)) for x, y in pts]
        pos = np.stack([place(mv, fov, S, X, Y, d) for (X, Y), d in zip(want, ds)])
        sc = add(sc, Tri(pos=pos, want=want, tag="zrange"), "zrange")
    out = [s for s in scenes if s.tris]
    for s in out:
        if s.threads is None:
            assign_threads(s)
    return out


def _normals(rng):
    n = rng.normal(size=(3, 3)) * 0.4 + np.float64([0.0, 0.0, 1.0])
    return (n / np.linalg.norm(n, axis=-1, keepdims=True)).astype(np.float32)


def near_cases(S, mv, fov, rng):
    """Faces cut by the near plane, found by search through the mirror: a 4-vertex polygon whose second sub-triangle is
    small, one where it is big, a face with two vertices behind the plane, one with all three behind it."""
    mvp = upload_mvp(mv, fov)
    inv = np.linalg.inv(np.asarray(mv, np.float64))
    need = {"near4:small": None, "near4:big": None, "near3": None, "near0": None}
    for _ in range(20000):
        if all(v is not None for v in need.values()):
            break
        zs = rng.uniform(-0.03, 0.02, 3) if rng.random() < 0.5 else rng.uniform(-2.0, 0.02, 3)
        xy = rng.uniform(-1, 1, (3, 2)) * 10 ** rng.uniform(-4.5, -1.5) * np.maximum(np.abs(zs)[:, None], 0.005) / 0.01
        view = np.concatenate([xy, zs[:, None], np.ones((3, 1))], axis=1)
        pos = (inv @ view.T).T[:, :3].astype(np.float32)
        clip = clip_coords(mvp, pos)
        n, first, second = face_plan(clip, S)
        if n == 4 and second is not None and first is not None and first.valid:
            key = "near4:big" if second.path == "big" else "near4:small"
        elif n == 3 and first is not None and first.valid and int((clip[:, 2] + clip[:, 3] < 0).sum()) == 2:
            key = "near3"
        elif n == 0:
            key = "near0"
        else:
            continue
        if need[key] is None:
            need[key] = Tri(pos=pos, tag=key.split(":")[0], nrm=_normals(rng))
    missing = [k for k, v in need.items() if v is None]
    assert not missing, f"near-plane search found no {missing} at S = {S}"
    return list(need.values())


# ----------------------------------------------------------------------------------------------------------------------
# what the cases reach
# ----------------------------------------------------------------------------------------------------------------------
def reach(scenes):
    """Counter of everything the issue of exact coverage depends on, over a list of scenes."""
    c = Counter()
    for sc in scenes:
        plans = sc.plans()
        warps = {}
        for tri, t, (n, first, second) in zip(sc.tris, sc.threads, plans):
            c[f"poly{n}"] += 1
            w = warps.setdefault(t // 32, {"r1": [], "r2": []})
            for rnd, r in (("r1", first), ("r2", second)):
                if r is None or not r.valid:
                    continue
                w[rnd].append(r.path)
                c[f"path:{r.path}"] += 1
                c[f"path:{r.path}:sgn{r.sgn:+d}"] += 1
                if rnd == "r2":
                    c[f"second:{'big' if r.path == 'big' else 'small'}"] += 1
                for (o, s), k in tie_pixels(r).items():
                    c[f"tie:{r.path}:{o}:sgn{s:+d}"] += k
                if r.path == "big":
                    culled, kept, lone = tile_stats(r)
                    c["big:tiles_culled"] += culled
                    c["big:tiles_kept"] += kept
                    c["big:lone_tie_at_emax_corner"] += lone
                    if culled and kept:
                        c["big:both_culled_and_kept"] += 1
                px0, px1, py0, py1 = r.box
                if px1 == sc.S - 1 or py1 == sc.S - 1:
                    c["box_touches_S-1"] += 1
                    if sc.S % 8 and r.path == "big" and (px1 >> 3 == (sc.S - 1) >> 3 or py1 >> 3 == (sc.S - 1) >> 3):
                        c["big:partial_tile_at_S"] += 1
                z = depth_values(r)
                c["frag:z<=0"] += int((z <= 0).sum())
                c["frag:z>=1"] += int((z >= 1).sum())
        for w in warps.values():
            if w["r1"].count("big") >= 2:
                c["warp:two_big"] += 1
            if "big" in w["r1"] and any(p != "big" for p in w["r1"]):
                c["warp:small_and_big"] += 1
            if w["r2"]:
                c["warp:some_lanes_second"] += 1
        for tri in sc.tris:
            if tri.dup_of >= 0:
                c["dup"] += 1
    return c


# ----------------------------------------------------------------------------------------------------------------------
# colour bound of the aggregation renderer
# ----------------------------------------------------------------------------------------------------------------------
# The shading weight is w = max(exp(max(-20 acos(dt), -50)), 1e-4) [* 1e-8] or 1e-16. dt, every flag test, every mask
# and depth sum is the same IEEE fp32 arithmetic on both sides (-fmad=false against -ffp-contract=off), so masks and
# depth are exact. Only acosf and expf differ. The CUDA Math API documents a maximum error of 2 ulp for each. glibc
# documents 1 ulp for each (libm-test-ulps, x86_64).
#   a = acos(dt): |a_gpu - a_cpu| <= 3 ulp(a) <= 3 * 2^-23 a.
#   u = -20 a: both sides round the product, so |du| <= (3 + 1) * 2^-23 |u|.
#   w = exp(u) is clamped to 1e-4, so only |u| <= ln(1e4) < 9.22 matters (max() is 1-Lipschitz), and
#   |dw| / w <= exp(4 * 2^-23 * 9.22) - 1 + (2 + 1) * 2^-23 < 40 * 2^-23 = DELTA_W. The 1e-8 factor rounds identically.
# The colour C = sum(c_i w_i) / sum(w_i) with c_i in [0, 1] moves by at most DELTA_W / (1 - DELTA_W) in exact arithmetic.
# Each side then rounds k products, k - 1 sums and one quotient (gamma_{2k+1} relative, |C| <= 1), and the two sides'
# roundings are independent: |C_gpu - C_cpu| <= DELTA_W / (1 - DELTA_W) + 2 gamma_{2k+1}.
DELTA_W = 40 * 2.0 ** -23


def colour_bound(views: int) -> float:
    u = 2.0 ** -24
    m = 2 * views + 1
    gamma = m * u / (1 - m * u)
    return DELTA_W / (1 - DELTA_W) + 2 * gamma

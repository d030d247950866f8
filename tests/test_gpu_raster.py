"""The warp rasteriser (csrc/warp.cu) against its oracle (oracle/raster_ref.c) on crafted geometry, bit for bit.

The scenes come from tests/raster_model.py: vertices placed exactly on chosen 1/256-pixel points, so that pixel centres
sit on edges of every orientation in each of the three scan paths (small32, small64, big), tie pixels sit alone in
their 8x8 tile, duplicated faces tie in depth, faces cross the near plane and fragments leave the (0, 1) depth range.
Both renderers get identical meshes. Masks and depth must be equal everywhere, the winning face (named by its palette
texel) must be the same at every pixel, and colour with several source views is held to raster_model.colour_bound.
The mesh build is checked on crafted depth maps where its diagonal and atol comparisons tie exactly."""
import dataclasses
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ivid_b200.rgbd_3d as rgbd_3d
import raster_model as RM
from conftest import ROOT
from ivid_b200 import _lib
from oracle import warp_ref

pytestmark = pytest.mark.gpu

SIZES = [(27, 9), (192, 64), (300, 100), (384, 128), (640, 128), (768, 256)]
SOURCE_CAMS = [warp_ref.look_at((0.3, 0.2, 1.0), (0, 0, -2), (0, 1, 0)), warp_ref.look_at((-0.5, 0.1, 0.8), (0, 0, -2), (0, 1, 0)),
               warp_ref.look_at((0.1, -0.6, 1.2), (0, 0, -2), (0, 1, 0))]


def _ulps_of(got, want):
    return np.abs(got.astype(np.float64) - want) / np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)


def _check_agg(tag, got, ref, views, pal):
    for k in ("mask_color", "mask_depth"):
        assert np.array_equal(got[k], ref[k]), f"{tag}: {k} differs on {int((got[k] != ref[k]).sum())} pixels"
    assert np.array_equal(got["depth"], ref["depth"].astype(np.float32)), f"{tag}: depth differs on " \
        f"{int((got['depth'] != ref['depth']).sum())} pixels"
    rc = np.asarray(ref["color"], np.float32)
    if views == 1:
        lit = rc.sum(-1) > 0
        tg, tr = RM.texel_of(got["color"]), RM.texel_of(rc)
        assert np.array_equal(tg[lit], tr[lit]), f"{tag}: winning face differs"
        assert np.array_equal(got["color"][~lit], rc[~lit])
        flat = pal.reshape(-1, 3)
        assert (_ulps_of(got["color"][lit], flat[tg[lit]]) <= 2).all(), f"{tag}: colour is not (c w) / w"
    err = float(np.abs(got["color"] - rc).max())
    assert err <= RM.colour_bound(views), f"{tag}: colour off by {err:.3e} > {RM.colour_bound(views):.3e}"
    return err


@pytest.mark.parametrize("S,n", SIZES)
def test_crafted_scenes_simple_mode(S, n):
    """SimpleRenderer: coverage, depth and the winning face's texel exactly, back faces drawn but not lit."""
    gpu, ref = rgbd_3d.SimpleRenderer(S, n), warp_ref.SoftwareSimpleRenderer(S, n)
    dups = 0
    for sc in RM.case_scenes(S, n):
        mesh, tex = sc.mesh()
        g, r = gpu.render(mesh, tex, sc.mv, sc.fov), ref.render(mesh, tex, sc.mv, sc.fov)
        assert np.array_equal(g.mask, r.mask), f"{sc.name}: mask differs on {int((g.mask != r.mask).sum())} pixels"
        assert np.array_equal(g.depth, r.depth), f"{sc.name}: depth differs on {int((g.depth != r.depth).sum())} pixels"
        assert np.array_equal(g.color, r.color.astype(np.float32)), f"{sc.name}: winning texel differs"
        win = np.where(g.mask[..., 0], RM.texel_of(g.color), -1)
        for k, t in enumerate(sc.tris):
            if t.dup_of >= 0 and t.tag != "near4":
                # the lower face index (the duplicate, drawn by the later thread) owns every pixel of the pair
                assert (win == k).any() and not (win == t.dup_of).any(), f"{sc.name}: equal depth went to the higher face index"
                dups += 1
    assert dups >= 3


@pytest.mark.parametrize("S,n", SIZES)
def test_crafted_scenes_aggregation_mode(S, n):
    """AggregationRenderer with 1, 2 and 3 source views: the scenes of one size overlap, so later views add fragments at
    other depths; padded back faces are discarded, edge-flagged and eroded faces give the low-confidence weights."""
    gpu, ref = rgbd_3d.AggregationRenderer(S, n), warp_ref.SoftwareAggregationRenderer(S, n)
    scenes = RM.case_scenes(S, n)
    pal = RM.palette(n)
    worst = {1: 0.0, 2: 0.0, 3: 0.0}
    farther = 0
    for i, sc in enumerate(scenes):
        for views in (1, 2, 3):
            if views > 1 and i % 3:
                continue
            meshes, cols = [], []
            for v in range(views):
                m, tex = scenes[(i + v) % len(scenes)].mesh(modelview=SOURCE_CAMS[v])
                meshes.append(m)
                cols.append(tex)
            g = gpu.render(meshes, cols, sc.mv, sc.fov)
            r = ref.render(meshes, cols, sc.mv, sc.fov)
            worst[views] = max(worst[views], _check_agg(f"{sc.name} x{views}", g, r, views, pal))
            if views > 1:
                farther += _low_confidence_overlaps(ref, meshes, cols, sc)
    # the same small triangles in two views at two depths (scaling about the camera keeps their pixels), edge-flagged in
    # one and padded in the other: every covered pixel has only weight-1e-16 fragments, and the farther one must win
    near_, far_ = scenes[0], scenes[0]
    lc = [RM.Scene(S, n, sc0.mv, sc0.fov, [dataclasses.replace(t, pos=t.pos * np.float32(k), flag=f, want=None) for t in sc0.tris],
                   threads=sc0.threads, name=f"S{S}:low-confidence") for sc0, k, f in ((near_, 1.0, 1), (far_, 1.25, 2))]
    meshes, cols = zip(*[x.mesh(modelview=SOURCE_CAMS[v]) for v, x in enumerate(lc)])
    g, r = gpu.render(list(meshes), list(cols), lc[0].mv, lc[0].fov), ref.render(list(meshes), list(cols), lc[0].mv, lc[0].fov)
    _check_agg(lc[0].name, g, r, 2, pal)
    farther += _low_confidence_overlaps(ref, meshes, cols, lc[0])
    print(f"[raster] S={S}: {len(scenes)} scenes, colour max |gpu - oracle| by source views {worst} "
          f"(bounds {[f'{RM.colour_bound(v):.2e}' for v in (1, 2, 3)]}), {farther} pixels decided by 'farther wins'")
    assert farther > 0, "no pixel reached aggregation.csh's low-confidence branch"


def _low_confidence_overlaps(ref, meshes, cols, sc):
    """Pixels where at least two source views have only a weight-1e-16 fragment (padding or edge flag), at different
    depths: aggregation.csh keeps the farther one.  Each view rendered alone by the oracle shows them as drawn (depth
    written) but without a depth vote."""
    empty = np.float32(ref.near * ref.far) / (np.float32(ref.far) - np.float32(0) * np.float32(ref.far - ref.near))
    low, depth = [], []
    for m, c in zip(meshes, cols):
        r = ref.render([m], [c], sc.mv, sc.fov)
        low.append(~r.mask_depth[..., 0] & (r.depth[..., 0] != empty))
        depth.append(r.depth[..., 0])
    n = 0
    for a in range(len(meshes)):
        for b in range(a + 1, len(meshes)):
            n += int((low[a] & low[b] & (depth[a] != depth[b])).sum())
    return n


def test_batch_of_three_samples_and_views():
    """3 samples x 3 source views, each a different mesh, with per-sample target modelviews, through the C API: the
    visibility buffers and view tables are indexed by (sample, view)."""
    S, n = 192, 64
    scenes = RM.case_scenes(S, n)
    targets = [np.eye(4, dtype=np.float32), warp_ref.look_at((0.05, 0.02, 0.0), (0.05, 0.0, -1.0), (0, 1, 0)),
               warp_ref.look_at((-0.04, 0.03, 0.1), (0.0, -0.02, -1.0), (0, 1, 0))]
    dw = rgbd_3d.DeviceWarp(3, image_size=n, ssaa=3, max_views=3)
    meshes = [[None] * 3 for _ in range(3)]
    for b in range(3):
        for v in range(3):
            m, tex = scenes[(3 * b + v) % len(scenes)].mesh(modelview=SOURCE_CAMS[v], uv_shift=b)
            vb = np.ascontiguousarray(np.concatenate([m["vertices"][k] for k in ("position", "normal", "uv", "flag")], -1))
            mv = np.ascontiguousarray(SOURCE_CAMS[v], np.float32)
            _lib.check(_lib.lib().ivid_warp_set_mesh(dw._handle, b, v, vb.ctypes.data, m["faces"].ctypes.data, tex.ctypes.data,
                                                     mv.ctypes.data))
            meshes[b][v] = (m, tex)
    color, depth, mc, md = dw.render_raw(targets, 45.0)
    ref = warp_ref.SoftwareAggregationRenderer(S, n)
    for b in range(3):
        r = ref.render([m for m, _ in meshes[b]], [t for _, t in meshes[b]], targets[b], 45.0)
        got = dict(color=color[b].cpu().numpy(), depth=depth[b].cpu().numpy()[..., None], mask_color=mc[b].cpu().numpy()[..., None] > 0.5,
                   mask_depth=md[b].cpu().numpy()[..., None] > 0.5)
        _check_agg(f"batch sample {b}", got, r, 3, RM.palette(n))
        assert got["mask_depth"].mean() > 0.01


@pytest.fixture(scope="module")
def wg():
    return {k: v for i in (0, 1) for k, v in np.load(os.path.join(ROOT, "tests", "golden", f"warp_golden_part{i}.npz")).items()}


@pytest.mark.parametrize("n", [64, 128, 256])
def test_natural_fixtures_on_identical_meshes(wg, n):
    """The warp_golden views at 192^2, 384^2 and 768^2, rendered from identical meshes on both sides: the oracle's
    meshes, and the GPU's own meshes read back.  Masks and depth exact, colour within the transcendental bound."""
    near, far, fov, atol, rtol, erode = [float(v) for v in wg["params"]]
    p = dict(fov=fov, near=near, far=far, atol=atol, rtol=rtol, erode_rgb=int(erode))
    xs = [torch.from_numpy(wg[f"rgbd{i}"].transpose(2, 0, 1)[None] * 2 - 1).float() for i in range(2)]
    if n != 128:
        xs = [F.interpolate(x, size=(n, n), mode="bilinear", align_corners=False) for x in xs]
    xs = [x.cuda() for x in xs]
    dw = rgbd_3d.DeviceWarp(1, image_size=n, ssaa=3, max_views=3)
    ours, theirs, cs = [], [], []
    for j in range(2):
        r01 = xs[j].cpu().numpy().transpose(0, 2, 3, 1)[0] * 0.5 + 0.5
        theirs.append(warp_ref.depth_to_mesh(warp_ref.linearize_depth(r01[:, :, 3:], near, far), fov=fov, modelview=wg["views"][j],
                                             atol=atol, rtol=rtol, erode_rgb=p["erode_rgb"]))
        cs.append(r01[:, :, :3])
        dw.add_view(xs[j], wg["views"][j], **p)
        vb, faces, col = dw.get_mesh(0, j)
        ours.append(dict(faces=faces, modelview=wg["views"][j], vertices=dict(position=vb[:, :3], normal=vb[:, 3:6], uv=vb[:, 6:8],
                                                                              flag=vb[:, 8:9])))
    gpu, ref = rgbd_3d.AggregationRenderer(3 * n, n), warp_ref.SoftwareAggregationRenderer(3 * n, n)
    for name, ms in (("oracle meshes", theirs), ("device meshes", ours)):
        g = gpu.render(ms, cs, wg["views"][2], fov)
        r = ref.render(ms, cs, wg["views"][2], fov)
        err = _check_agg(f"{name} at {3 * n}^2", g, r, 2, None)
        print(f"[raster] natural views at {3 * n}^2 from {name}: masks and depth exact, colour max {err:.2e}")


# ---- mesh build on crafted depth maps ------------------------------------------------------------------------------
def _crafted_depths(n):
    rng = np.random.default_rng(n)
    plane = np.full((n, n), 2.0, np.float32)
    # fp32 differences exactly on float32(0.03): depths (t, 2t), and inverse depths 1/25 - 1/100
    t = np.float32(0.03)
    assert t * np.float32(2) - t == t
    step_a = np.where(np.arange(n)[None, :] < n // 2, t, t * np.float32(2)).repeat(n, 0).astype(np.float32)
    assert np.float32(1) / np.float32(25) - np.float32(1) / np.float32(100) == t
    step_r = np.where(np.arange(n)[:, None] < n // 3, np.float32(25), np.float32(100)).repeat(n, 1).astype(np.float32)
    corners = np.full((n, n), 1.5, np.float32) + rng.uniform(0, 1e-3, (n, n)).astype(np.float32)
    corners[0, 0] = corners[-1, -1] = 4.0
    corners[0, n // 2] = corners[n // 2, -1] = 0.6
    return dict(plane=plane, atol_step=step_a, rtol_step=step_r, corners=corners)


@pytest.mark.parametrize("n", [9, 100, 128])
def test_mesh_build_on_crafted_depth(n):
    """Diagonal ties (a fronto-parallel plane: every cell's two diagonals have equal length), depth steps exactly at
    float32(atol) and float32(rtol) with the other tolerance None or passing, and discontinuities at the corners and
    borders under every erosion radius."""
    mv = warp_ref.view_on_sphere(0.2, 0.1)
    for name, d in _crafted_depths(n).items():
        cfgs = [(0.03, None, 2), (None, 0.03, 2), (0.03, 0.03, 1), (0.03, 0.03, 3)]
        for pad in ("frustum", None):
            for at, rt, er in cfgs:
                got = rgbd_3d.utils.depth_to_mesh(d[..., None], padding=pad, fov=45, modelview=mv, atol=at, rtol=rt, erode_rgb=er,
                                                  cal_normal=pad is not None)
                want = warp_ref.depth_to_mesh(d[..., None], fov=45, modelview=mv, atol=at, rtol=rt, erode_rgb=er, padding=pad,
                                              cal_normal=pad is not None)
                tag = f"{name} n={n} padding={pad} atol={at} rtol={rt} erode={er}"
                assert np.array_equal(got.faces, want.faces), f"{tag}: triangulation"
                assert np.array_equal(got.vertices.flag, want.vertices.flag.astype(np.float32)), f"{tag}: flags"
                pos = want.vertices.position.astype(np.float32)
                assert (np.abs(got.vertices.position - pos) <= np.spacing(np.abs(pos))).all(), f"{tag}: positions"
        # a step exactly on its tolerance is continuous ('>'), with the other tolerance None or passing
        for at, rt in {"atol_step": ((0.03, None), (0.03, 0.03)), "rtol_step": ((None, 0.03), (0.03, 0.03))}.get(name, ()):
            m = warp_ref.depth_to_mesh(d[..., None], fov=45, modelview=mv, atol=at, rtol=rt, erode_rgb=2)
            assert not (m.vertices.flag & 1).any(), (name, at, rt)


def _raw_depth_maps(n):
    """Model-space depth channels for add_view: a plane, raw depth exactly -1 and +1 (and one ulp inside) next to each
    other, and discontinuities at the corners and borders."""
    rng = np.random.default_rng(n + 1)
    one = np.float32(1)
    clip = np.full((n, n), 0.1, np.float32)
    clip[: n // 2, : n // 2] = -one
    clip[n // 2:, n // 2:] = one
    clip[: n // 2, n // 2:] = np.nextafter(-one, one)
    clip[n // 2:, : n // 2] = np.nextafter(one, -one)
    clip[0, :] = one
    corners = np.float32(-0.2) + rng.uniform(0, 1e-3, (n, n)).astype(np.float32)
    corners[0, 0] = corners[-1, -1] = corners[0, -1] = 0.9
    corners[n // 2, 0] = corners[-1, n // 2] = -0.9
    return dict(plane=np.full((n, n), 0.3, np.float32), clip=clip, corners=corners)


@pytest.mark.parametrize("n", [9, 100, 128])
def test_add_view_on_crafted_depth(n):
    """DeviceWarp.add_view (the sampling loop's mesh build from model-space RGBD) against depth_to_mesh on the oracle's
    reading of the same tensor: raw depth at +-1 hits the 1e-6 clip of linearize_depth; erosion radius 1 to 3 at the
    image corners and borders.  Faces and flags exact, positions and normals within one fp32 ulp of the float64 math."""
    mv = warp_ref.view_on_sphere(-0.3, 0.15)
    rng = np.random.default_rng(n)
    for name, raw in _raw_depth_maps(n).items():
        rgb = rng.uniform(-1, 1, (3, n, n)).astype(np.float32)
        x = torch.from_numpy(np.concatenate([rgb, raw[None]], 0)[None]).cuda()
        r01 = x.cpu().numpy().transpose(0, 2, 3, 1)[0] * 0.5 + 0.5
        for at, rt, er in ((0.03, 0.03, 1), (0.03, None, 2), (None, 0.03, 3)):
            kw = dict(fov=45, near=0.6, far=5, atol=at, rtol=rt, erode_rgb=er)
            dw = rgbd_3d.DeviceWarp(1, image_size=n, ssaa=3, max_views=1)
            dw.add_view(x, mv, **kw)
            vb, faces, col = dw.get_mesh(0, 0)
            m = warp_ref.depth_to_mesh(warp_ref.linearize_depth(r01[:, :, 3:], 0.6, 5), fov=45, modelview=mv, atol=at, rtol=rt,
                                       erode_rgb=er)
            ref = warp_ref.mesh_vertex_buffer(m)
            tag = f"{name} n={n} atol={at} rtol={rt} erode={er}"
            assert np.array_equal(faces, m.faces.astype(np.uint32)), f"{tag}: triangulation"
            assert np.array_equal(vb[:, 8], ref[:, 8]) and np.array_equal(vb[:, 6:8], ref[:, 6:8]), f"{tag}: flags / uv"
            pos = np.asarray(m.vertices.position, np.float64)
            assert (np.abs(vb[:, :3] - pos) <= np.spacing(np.abs(pos).astype(np.float32))).all(), f"{tag}: positions"
            assert np.abs(vb[:, 3:6] - m.vertices.normal).max() <= 2.5e-7, f"{tag}: normals"
            assert np.array_equal(col, r01[:, :, :3]), tag
            if name == "clip":
                assert (m.vertices.flag & 1).any(), tag


# ---- post-filters on crafted raw renders ---------------------------------------------------------------------------
POST_NEAR, POST_FAR = 0.6, 5.0
ATOL_EXACT, RTOL_EXACT = 2.0 ** -5, 2.0 ** -4     # tolerances a pair of projected depths can sit on exactly


def _project(d):
    """project_depth in the fp32 order both sides use."""
    d = np.clip(np.asarray(d, np.float32), POST_NEAR, POST_FAR)
    return (1 / POST_NEAR - 1 / d) / (1 / POST_NEAR - 1 / POST_FAR)


def _raw_pair(t, inverse):
    """Raw depths (da, db) whose projected values differ by exactly fp32 t (or whose fp32 inverses do).  The projected
    values lie in [0, 1], so a difference is a multiple of their ulp: t must be a dyadic value such as 2^-5."""
    for da in np.float32(1.2) + np.arange(400, dtype=np.float32) * np.float32(1e-3):
        pa = _project(da)
        pb0 = 1.0 / (1.0 / float(pa) - t) if inverse else float(pa) + t
        db0 = np.float32(1.0 / (1.0 / POST_NEAR - pb0 * (1.0 / POST_NEAR - 1.0 / POST_FAR)))
        cand = db0 + np.arange(-64, 64, dtype=np.float32) * np.spacing(db0)
        pb = _project(cand)
        diff = (np.float32(1) / pa - np.float32(1) / pb) if inverse else (pb - pa)
        hit = np.flatnonzero(diff == np.float32(t))
        if hit.size:
            return da, cand[hit[0]]
    raise AssertionError("no exact pair")


def _crafted_raw(S, n, seed):
    """A raw render (what AggregationRenderer.render returns) built to sit on the post-filters' boundaries."""
    rng = np.random.default_rng(seed)
    k = S // n
    off = (k - 1) // 2
    # SSAA votes: exactly 6, 7, 8 or 9 of the 9 sub-pixels, or any count
    votes = []
    for _ in range(2):
        want = rng.choice([6, 7, 8, 9, -1], size=(n, n))
        m = np.zeros((n, n, k * k), bool)
        for y in range(n):
            for x in range(n):
                c = want[y, x] if want[y, x] >= 0 else rng.integers(0, k * k + 1)
                m[y, x, rng.permutation(k * k)[:c]] = True
        assert {6, 7, 8} <= set(m.sum(-1).ravel().tolist())
        votes.append(m.reshape(n, n, k, k).transpose(0, 2, 1, 3).reshape(S, S, 1))
    # depth: smooth, a few pixels outside [near, far], and 3x3 spots whose centre differs from three neighbours by exactly
    # ATOL_EXACT (even spots) or whose inverses differ by exactly RTOL_EXACT (odd spots)
    proj = np.float32(1.0) + 0.2 * np.sin(np.arange(n)[:, None] / 3.0) * np.cos(np.arange(n)[None, :] / 4.0)
    d = proj.astype(np.float32)
    d[rng.integers(0, n, 3), rng.integers(0, n, 3)] = 0.2
    d[rng.integers(0, n, 3), rng.integers(0, n, 3)] = 9.0
    spots = [(y, x) for y in range(1, n - 2, 4) for x in range(1, n - 2, 4)]
    for j, (y, x) in enumerate(spots[:8]):
        inverse = j % 2 == 1
        da, db = _raw_pair(RTOL_EXACT if inverse else ATOL_EXACT, inverse)
        d[y - 1:y + 2, x - 1:x + 2] = da
        d[y, x + 1] = d[y + 1, x] = d[y + 1, x + 1] = db
    depth = np.repeat(np.repeat(d, k, 0), k, 1).astype(np.float32)
    depth += np.where((np.arange(S)[:, None] % k == off) & (np.arange(S)[None, :] % k == off), 0, 0.5).astype(np.float32)
    # colour: k/255 and one ulp either side (to8b truncates), 0, 1, out of range, saturated stripes at the borders
    levels = np.arange(256, dtype=np.float32) / np.float32(255)
    pool = np.concatenate([levels, np.nextafter(levels, np.float32(2)), np.nextafter(levels, np.float32(-1)),
                           np.float32([-0.5, 1.5, 0.0, 1.0])])
    color = rng.choice(pool, size=(S, S, 3)).astype(np.float32)
    color[:2] = 1.5
    color[-2:] = -0.25
    color[:, :3] = np.float32([1.0, 0.0, 1.0])[None, None, :] * (np.arange(3)[None, :, None] % 2)
    color[:, -1] = 1.0
    return warp_ref.AttrDict(color=color, depth=depth[..., None], mask_color=votes[0], mask_depth=votes[1])


@pytest.mark.parametrize("S,n", [(27, 9), (300, 100), (384, 128)])
def test_postfilters_on_crafted_raw_renders(S, n):
    """aggregate_conditions' post-filters (ivid_warp_postfilter) on crafted raw renders: votes of exactly 6, 7 and 8 of 9,
    depth_edge pairs exactly on atol and on rtol (2^-5 and 2^-4: differences of projected depths in [0, 1] are multiples
    of their ulp, so only a dyadic tolerance can be met exactly), colours at k/255 and one ulp either side, saturated borders for the 8-bit
    LANCZOS.  Every output bit-identical to the oracle's numpy / PIL / cv2 steps."""
    class Replay:
        render_size = S
        def __init__(self, raw): self.raw = raw
        def render(self, *a, **k): return self.raw

    mv = np.eye(4, dtype=np.float32)
    colors = [np.zeros((n, n, 3), np.float32)]
    for seed, (atol, rtol, erode) in enumerate(((ATOL_EXACT, 0.01, 1), (0.01, RTOL_EXACT, 2), (0.02, 0.02, 3))):
        raw = _crafted_raw(S, n, seed)
        kw = dict(fov=45, near=POST_NEAR, far=POST_FAR, atol=atol, rtol=rtol, erode_rgb=erode)
        ref = warp_ref.aggregate_conditions(Replay(raw), None, colors, mv, **kw)
        gpu_r = rgbd_3d.AggregationRenderer(S, n)
        gpu_r._last_raw = tuple(torch.from_numpy(np.ascontiguousarray(a.astype(np.float32))).cuda() for a in
                                (raw.color, raw.depth[..., 0], raw.mask_color[..., 0], raw.mask_depth[..., 0]))
        gpu_r.render = lambda *a, **k: None
        got = rgbd_3d.utils.aggregate_conditions(gpu_r, None, colors, mv, **kw)
        tag = f"S={S} atol={atol} rtol={rtol} erode={erode}"
        for key in ("mask", "mask_rgb", "depth", "depth_convex"):
            assert np.array_equal(got[key], np.asarray(ref[key], np.float32)), f"{tag}: {key}"
        assert np.array_equal(got["color"], np.asarray(ref["color"]).astype(np.float32)), f"{tag}: colour"
        assert 0 < float(ref["mask"].mean()) < 1, tag
        assert erode > 1 or 0 < float(ref["mask_rgb"].mean()) < 1, tag

"""The crafted rasteriser cases of tests/raster_model.py on the CPU: the mirrored vertex stage agrees with the oracle
renderer, every case lands where it was placed, the case set reaches every scan path, tile rule and tie orientation of
csrc/warp.cu, and the oracle (oracle/raster_ref.c) gives hand-derived coverage on cases whose answer is known."""
import math

import numpy as np
import pytest

import raster_model as RM
from oracle import warp_ref

SIZES = [(27, 9), (192, 64), (300, 100), (384, 128), (640, 128), (768, 256)]
CAMERAS = [np.eye(4, dtype=np.float32), warp_ref.view_on_sphere(0.3, 0.2), warp_ref.view_on_sphere(-0.7, -0.4)]


@pytest.fixture(scope="module")
def scenes():
    return {S: RM.case_scenes(S, n) for S, n in SIZES}


@pytest.mark.parametrize("fov", [45.0, 30.0, 60.0])
@pytest.mark.parametrize("cam", range(len(CAMERAS)))
def test_mirrored_mvp_equals_oracle_mvp(fov, cam):
    """The oracle renderer's P*MV, bit for bit (exact placement means nothing otherwise)."""
    mv = CAMERAS[cam]
    for near, far in ((RM.NEAR, RM.FAR), (0.1, 200.0)):
        proj = warp_ref.perspective(np.deg2rad(fov), 1, near, far)
        want = (proj.astype(np.float64) @ np.asarray(mv, np.float64)).astype(np.float32)
        assert np.array_equal(RM.upload_mvp(mv, fov, near, far), want)


def test_every_case_lands_where_intended(scenes):
    for S, sc in scenes.items():
        for s in sc:
            s.check_placement()
    s = RM.case_scenes(192, 64, mv=CAMERAS[1])
    for x in s:
        x.check_placement()


def test_permutation_is_a_bijection():
    for S, n in SIZES:
        F = 2 * (n + 1) ** 2
        assert math.gcd(RM.PERM, F) == 1, F
        f = np.arange(F)
        fi = RM.face_of_thread(f, F)
        assert np.array_equal(np.sort(fi), f)
        assert all(RM.thread_of_face(int(x), F) == int(t) for t, x in zip(f[:500], fi[:500]))


def test_case_set_reaches_every_path_and_rule(scenes, capsys):
    from collections import Counter
    total = Counter()
    per = {}
    for S, sc in scenes.items():
        per[S] = RM.reach(sc)
        total += per[S]
    lines = []
    for path in RM.PATHS:
        lines.append(f"  {path}: {total['path:' + path]} sub-triangles")
        for o in RM.ORIENTS:
            lines.append(f"    tie {o:10s} front {total[f'tie:{path}:{o}:sgn+1']:5d}   back {total[f'tie:{path}:{o}:sgn-1']:5d}")
    other = ["big:both_culled_and_kept", "big:tiles_culled", "big:tiles_kept", "big:lone_tie_at_emax_corner", "big:partial_tile_at_S",
             "warp:two_big", "warp:small_and_big", "warp:some_lanes_second", "second:small", "second:big", "poly4", "poly3", "poly0",
             "frag:z<=0", "frag:z>=1", "box_touches_S-1", "dup"]
    lines += [f"  {k}: {total[k]}" for k in other]
    with capsys.disabled():       # the reach is part of the result: list it whether or not the test passes
        print("\n[reach] crafted rasteriser cases over S = " + ", ".join(str(S) for S, _ in SIZES) + "\n" + "\n".join(lines))
    for path in RM.PATHS:
        for o in RM.ORIENTS:
            for sg in ("+1", "-1"):
                assert total[f"tie:{path}:{o}:sgn{sg}"] > 0, (path, o, sg)
    for k in other:
        assert total[k] > 0, k
    for S, c in per.items():
        for path in RM.PATHS:
            assert c["path:" + path] > 0, (S, path)
        assert c["big:lone_tie_at_emax_corner"] > 0 and c["second:small"] > 0 and c["second:big"] > 0, S
    # two vertices behind the near plane still leave a triangle; all three behind leave nothing
    assert total["poly0"] >= len(SIZES)


def _oracle_simple(S, n, tris_px, mv=None):
    """SoftwareSimpleRenderer on triangles given by pixel-centre vertices; -> winner texel per pixel (row 0 = bottom)."""
    mv = np.eye(4, dtype=np.float32) if mv is None else mv
    sc = RM.Scene(S, n, mv, 45.0, [RM._tri_px(S, mv, 45.0, t, [2.0, 2.0, 2.0]) for t in tris_px])
    RM.assign_threads(sc)
    sc.check_placement()
    mesh, tex = sc.mesh()
    r = warp_ref.SoftwareSimpleRenderer(S, n).render(mesh, tex, mv)
    win = np.where(r.mask[..., 0], RM.texel_of(r.color), -1)
    return win[::-1]          # framebuffer orientation: row py


def _oracle_depth_cover(S, n, tris_px):
    """Pixels the oracle wrote depth to (back faces in the simple renderer have alpha 0 but still win depth)."""
    mv = np.eye(4, dtype=np.float32)
    sc = RM.Scene(S, n, mv, 45.0, [RM._tri_px(S, mv, 45.0, t, [2.0, 2.0, 2.0]) for t in tris_px])
    RM.assign_threads(sc)
    mesh, tex = sc.mesh()
    r = warp_ref.SoftwareSimpleRenderer(S, n).render(mesh, tex, mv)
    return (r.depth[..., 0] < np.float32(RM.FAR) * 0.999)[::-1]


def test_oracle_gives_hand_derived_coverage():
    """Coverage known by construction: the oracle is the second witness of the rules, not the only one."""
    S, n = 27, 9
    # a rectangle [2, 12] x [3, 9] (pixel centres) as two triangles sharing the diagonal through pixel centres
    a, b, c, d = (2, 3), (12, 3), (12, 9), (2, 9)
    for tris in ([[a, b, c], [a, c, d]], [[a, c, b], [a, d, c]]):       # front faces, back faces
        win = _oracle_simple(S, n, tris)
        py, px = np.mgrid[0:S, 0:S]
        covered = win >= 0 if tris[0][1] == b else _oracle_depth_cover(S, n, tris)
        # left edge x = 2 (interior to the right: dy < 0 after sign adjustment -> excluded), right edge x = 12 (included),
        # bottom y = 3 (interior above: dx > 0 -> excluded), top y = 9 (included)
        want = (px > 2) & (px <= 12) & (py > 3) & (py <= 9)
        assert np.array_equal(covered, want)
        # every centre on the shared diagonal (2,3)-(12,9)... passes through (7,6): covered exactly once, by one face
        assert covered[6, 7] and (win[6, 7] in (0, 1) or tris[0][1] == c)
    # two front faces sharing the edge (15, 9)-(3, 15), which passes through the centres (13, 10), (11, 11) ... (5, 14).
    # In the first face the edge runs (15, 9) -> (3, 15): dy > 0, so its tie pixels belong to it; in the second it runs
    # (3, 15) -> (15, 9): dy < 0, so they do not.  Each face is rendered alone, so the oracle shows both coverages.
    tris = [[(3, 3), (15, 9), (3, 15)], [(15, 9), (21, 21), (3, 15)]]
    alone = [_oracle_depth_cover(S, n, [t]) for t in tris]
    assert not (alone[0] & alone[1]).any(), "a pixel centre owned by both faces"
    shared = [(15 - 2 * k, 9 + k) for k in range(1, 6)]      # the centres strictly between (15, 9) and (3, 15)
    for x, y in shared:
        assert alone[0][y, x] and not alone[1][y, x], (x, y)
    # the pair drawn together: every pixel goes to the face that owns it alone, and the mirror agrees
    win = _oracle_simple(S, n, tris)
    assert np.array_equal(win == 0, alone[0]) and np.array_equal(win == 1, alone[1])
    sc = RM.Scene(S, n, np.eye(4, dtype=np.float32), 45.0, [RM._tri_px(S, np.eye(4), 45.0, t, [2.0] * 3) for t in tris])
    RM.assign_threads(sc)
    for (_, first, _), want in zip(sc.plans(), alone):
        px, py, E, ins, c = RM.coverage(first)
        m = np.zeros((S, S), bool)
        m[py[c], px[c]] = True
        assert np.array_equal(m, want)


def test_colour_bound_derivation():
    assert RM.colour_bound(1) < 1e-5 and RM.colour_bound(3) < RM.colour_bound(4)
    assert RM.DELTA_W > math.exp(4 * 2.0 ** -23 * math.log(1e4)) - 1 + 3 * 2.0 ** -23

"""CPU: the path selection and rounding bounds of tests/resample_model.py, against the library's own tile choice and against
numpy float32 emulations of the kernels' summation order; and every GPU case of tests/test_gpu_resample.py reaches the
path its id names."""
import ctypes
import math

import numpy as np
import pytest

import resample_model as M


def test_conv_tile_matches_library():
    from ivid_b200 import _lib
    L = _lib.lib()
    for H in range(1, 70):
        for W in (1, 2, 3, 4, 6, 8, 10, 12, 16, 20, 24, 32, 40, 48, 64, 80, 96, 128):
            v = [ctypes.c_int() for _ in range(4)]
            _lib.check(L.ivid_conv_tile(H, W, *[ctypes.byref(x) for x in v]))
            assert (v[0].value, v[1].value, v[2].value) == M.conv_tile(H, W), (H, W)
            assert bool(v[3].value) == M.conv_can_fuse_stats(H, W), (H, W)


def test_gn_stats_layout():
    assert M.gn_stats_layout(8) == (2, 128, 1)
    assert M.gn_stats_layout(96) == (24, 10, 1)          # 256 = 10 * 24 + 16: the last 16 threads idle
    assert M.gn_stats_layout(1024) == (256, 1, 1)
    assert M.gn_stats_layout(1280) == (256, 1, 2)        # 320 columns: the second round leaves 192 threads without one
    assert M.gn_stats_layout(1544) == (256, 1, 2)
    assert M.gn_stats_layout(2048) == (256, 1, 2)
    assert M.gn_stats_run(1280, 4096) == 256 and M.gn_stats_run(1280, 31) == 31
    assert M.gn_stats_run(96, 4096) == 26 and M.gn_stats_run(8, 257) == 2 and M.gn_stats_run(40, 1) == 1


def test_gn_prologue_paths():
    assert M.gn_prologue_fast(256, 32) and M.gn_prologue_fast(1024, 32) and M.gn_prologue_fast(96, 48)
    assert not M.gn_prologue_fast(1280, 32)                # C > 1024
    assert not M.gn_prologue_fast(320, 8)                  # 40 channels per group
    assert not M.gn_prologue_fast(96, 32)                  # 3 channels per group
    assert not M.gn_prologue_fast(40, 8)                   # C % 32 != 0


def test_stats_cases_reach_their_paths():
    ids = [M.stats_case_id(c) for c in M.STATS_CASES]
    assert len(set(ids)) == len(ids)
    kinds = {i.rsplit("-", 1)[1] for i in ids}
    assert kinds == {"full", "idle", "ragged", "rounds"}
    assert {c[0] for c in M.STATS_CASES} == set(M.STATS_WIDTHS)
    assert {c[1] for c in M.STATS_CASES} == set(M.STATS_HWS)
    assert {c[2] for c in M.STATS_CASES} == {1, 3, 33} and {c[3] for c in M.STATS_CASES} == {0, 10, 100}
    for C, HW, N, k in M.STATS_CASES:
        cols, rows, rounds = M.gn_stats_layout(C)
        kind = M.stats_case_id((C, HW, N, k)).rsplit("-", 1)[1]
        assert (kind == "idle") == (256 % cols != 0)
        assert (kind == "ragged") == ((C // 4) % cols != 0)
        assert (kind in ("ragged", "rounds")) == (rounds > 1)
    # several blocks (fp64 atomics across blocks) at every width class
    assert {M.stats_case_id(c).rsplit("-", 1)[1] for c in M.STATS_CASES if c[1] > 256} == kinds


def test_apply_cases_reach_their_paths():
    seen = set()
    for case in M.APPLY_CASES:
        tag, C0, C1, groups, film, with_stats, mode, H, W, N = case
        C = C0 + C1
        assert C0 % 8 == 0 and C1 % 8 == 0 and C % groups == 0 and groups <= 64
        assert mode != 2 or (H % 2 == 0 and W % 2 == 0)
        path = M.apply_path(case)
        assert tag.startswith(path), tag
        assert (f"m{mode}" in tag) and (("nullstats" in tag) == (not with_stats)), tag
        if "seam" in tag:
            assert C1 > 0 and C0 % (C // groups) != 0, f"{tag}: no group straddles the seam"
        seen.add((path, mode))
        seen.add((path, film))
        seen.add((path, with_stats))
    for path in ("fast", "loop"):
        assert {(path, m) for m in (0, 1, 2)} <= seen
        assert {(path, f) for f in ("ss", "add", None)} <= seen
        assert {(path, s) for s in (True, False)} <= seen
    assert any(c[1] == 1280 for c in M.APPLY_CASES) and any(c[1] + c[2] == 320 and c[3] == 8 for c in M.APPLY_CASES)
    assert any((c[1] + c[2]) // c[3] == 3 for c in M.APPLY_CASES)


def test_conv_cases_reach_their_paths():
    down = [M.conv_tile(c[3], c[4]) for c in M.DOWN_CASES]
    assert {(8, 8, 2), (4, 4, 8), (1, 1, 128), (16, 8, 1), (2, 2, 32)} <= set(down)
    assert {c[1] for c in M.DOWN_CASES} == {64, 96, 160}
    for C in (96, 160):
        assert 9 * C % 64 != 0 and M.conv_K(2, C) > 9 * C      # the last 64-column box runs past 9C
    assert any(c[3:] == (6, 10) and not M.conv_can_fuse_stats(6, 10) for c in M.DOWN_CASES)
    assert any(c[3:] == (32, 48) for c in M.DOWN_CASES)
    assert any(c[3:] == (1, 1) and c[2] > 128 for c in M.DOWN_CASES)    # two batch tiles, the second one a tail
    up = {(c[3], c[4]): M.slab(c[3], c[4]) for c in M.UP_CASES}
    assert up[(16, 16)] and up[(32, 48)] and not up[(12, 20)] and not up[(4, 4)]
    for c in M.DOWN_CASES + M.UP_CASES:
        cid = M.conv_case_id(c)
        assert ("fused" in cid) == M.conv_can_fuse_stats(c[3], c[4])


def _offset(rng, N, HW, C, k):
    sigma = rng.random(C) * 1.5 + 0.5
    return (rng.standard_normal((N, HW, C)) * sigma + k * sigma).astype(np.float32)


@pytest.mark.parametrize("C,HW", [(8, 257), (96, 4096), (256, 600), (1280, 300), (2048, 256)])
@pytest.mark.parametrize("k", [0, 10, 100])
def test_gn_stats_bound_holds_for_the_kernel_order(C, HW, k):
    rng = np.random.default_rng(C * 7 + HW + k)
    x = _offset(rng, 2, HW, C, k)
    got = M.gn_stats_emulate(x)
    x64 = x.astype(np.float64)
    bS, bQ = M.gn_stats_bound(x64, C, HW)
    rs = float((np.abs(got[..., 0] - x64.sum(1)) / bS).max())
    rq = float((np.abs(got[..., 1] - (x64 * x64).sum(1)) / bQ).max())
    assert rs <= 1.0 and rq <= 1.0, (rs, rq)


def test_gn_stats_bound_catches_a_dropped_row():
    """Summing only row 0 of the shared-memory reduction leaves out most pixels: far outside the bound."""
    C, HW = 96, 512
    x = _offset(np.random.default_rng(5), 1, HW, C, 1)
    _, rows, _ = M.gn_stats_layout(C)
    keep = np.zeros(HW, bool)
    for p0 in range(0, HW, 256):
        keep[p0:min(p0 + 256, HW):rows] = True
    wrong = M.gn_stats_emulate(x * keep[None, :, None])
    x64 = x.astype(np.float64)
    bS, _ = M.gn_stats_bound(x64, C, HW)
    assert float((np.abs(wrong[..., 0] - x64.sum(1)) / bS).max()) > 1e3


def test_pool_bound_holds_for_the_kernel_order():
    rng = np.random.default_rng(3)
    x = (rng.standard_normal((3, 16, 24, 40)) * 2 + rng.standard_normal(40)).astype(np.float32)
    x[0, :2, :2, :] = np.float32([1e8, -1e8, 1.0, 3.0])[:, None].reshape(2, 2, 1)   # cancellation
    got = M.pool_f32(x).astype(np.float64)
    x64 = x.astype(np.float64)
    p64 = 0.25 * (x64[:, 0::2, 0::2] + x64[:, 0::2, 1::2] + x64[:, 1::2, 0::2] + x64[:, 1::2, 1::2])
    assert float((np.abs(got - p64) / M.pool_bound(x64)).max()) <= 1.0
    # without cancellation the bound is 1.5 ulp of the mean at most (three roundings of sums no larger than it)
    xp = np.abs(x[1:])
    pp = 0.25 * (xp[:, 0::2, 0::2].astype(np.float64) + xp[:, 0::2, 1::2] + xp[:, 1::2, 0::2] + xp[:, 1::2, 1::2])
    assert float((M.pool_bound(xp.astype(np.float64)) / M.ulp32(pp)).max()) <= 2.0
    assert math.isclose(M.gamma(1), 2.0 ** -24, rel_tol=1e-6)

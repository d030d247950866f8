"""GPU: the device fusion (csrc/fusion.cu) against the fusion rule of oracle/fusion_ref.py.  The volumes (tsdf sum, weight,
colour sum, colour weight) and the meshes (faces, vertex positions, vertex colours) are bit-identical, on the analytic
sphere-and-plane scene and on the realistic views of the warp fixture, at grid sizes that are no multiple of a block."""
import os

import numpy as np
import pytest
import torch

import fusion_scene as fs
from conftest import ROOT
from ivid_b200.rgbd_3d import fusion
from oracle import fusion_ref as fr
from oracle import warp_ref

pytestmark = pytest.mark.gpu


def _bits(a):
    a = a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _check_against_oracle(tag, depths, colors, valid, mvs, fov, grid, trunc=3):
    ref = fr.integrate(depths, colors, valid, mvs, fov, grid.origin, grid.voxel, grid.dims, trunc)
    vol = fusion.tsdf_integrate(depths, colors, valid, mvs, fov, grid, trunc)
    for name, want in zip(("tsdf_sum", "weight", "color_sum", "color_weight"), ref):
        assert np.array_equal(_bits(vol[name]), _bits(want)), f"{tag}: {name} differs from the oracle"
    rv, rc, rf = fr.extract(*ref, grid.origin, grid.voxel)
    mesh = fusion.extract_surface(vol, grid)
    assert np.array_equal(mesh.faces.cpu().numpy(), rf), f"{tag}: faces differ"
    assert np.array_equal(_bits(mesh.vertices), _bits(rv)), f"{tag}: vertex positions differ"
    assert np.array_equal(mesh.colors.cpu().numpy(), rc), f"{tag}: vertex colours differ"
    again = fusion.extract_surface(vol, grid)
    assert all(torch.equal(mesh[k], again[k]) for k in ("vertices", "colors", "faces"))
    print(f"[fusion] {tag}: grid {grid.dims}, {int((ref[1] > 0).sum())} voxels seen, {rv.shape[0]} vertices, {rf.shape[0]} faces: "
          "volumes and mesh bit-identical to the oracle")
    return rv, rf


@pytest.fixture(scope="module")
def sphere_scene():
    S = fs.scene(n=64)
    S.valid = np.stack([fusion.view_validity(S.depths[v], S.fov, S.modelviews[v]) for v in range(27)])
    return S


def test_device_validity_is_the_oracle_rule(sphere_scene):
    S = sphere_scene
    for v in range(27):
        assert np.array_equal(S.valid[v], fs.oracle_validity(S.depths[v], S.modelviews[v]))
    assert 0.3 < S.valid.mean() < 0.95


@pytest.mark.parametrize("resolution", [61, 128])
def test_analytic_scene_matches_oracle(sphere_scene, resolution):
    S = sphere_scene
    pts = np.concatenate([fusion.world_points(S.depths[v], S.valid[v], S.fov, S.modelviews[v]) for v in range(27)])
    grid = fusion.default_grid(pts, resolution, 3)
    if resolution == 61:
        assert any(d % 2 for d in grid.dims) and int(np.prod(grid.dims)) % 256 != 0
    rv, rf = _check_against_oracle(f"sphere and plane, resolution {resolution}", S.depths, S.colors, S.valid, S.modelviews, S.fov, grid)
    assert rv.shape[0] > 500 and rf.shape[0] > 500


@pytest.mark.parametrize("resolution,trunc", [(61, 3), (96, 2.5)])
def test_warp_fixture_views_match_oracle(resolution, trunc):
    """The rgbd0 / rgbd1 views of the warp fixture: height fields with a foreground blob, i.e. realistic depth with
    discontinuities, with the fixture's planes, fov and tolerances."""
    wg = {k: v for i in (0, 1) for k, v in np.load(os.path.join(ROOT, "tests", "golden", f"warp_golden_part{i}.npz")).items()}
    near, far, fov, atol, rtol, erode = wg["params"]
    depths = np.stack([warp_ref.linearize_depth(wg[f"rgbd{i}"][:, :, 3], near, far).astype(np.float32) for i in (0, 1)])
    colors = np.stack([wg[f"rgbd{i}"][:, :, :3] for i in (0, 1)]).astype(np.float32)
    mvs = [wg["views"][0], wg["views"][1]]
    valid = np.stack([fusion.view_validity(depths[i], fov, mvs[i], None, atol, rtol, int(erode)) for i in (0, 1)])
    for i in (0, 1):
        assert np.array_equal(valid[i], fs.oracle_validity(depths[i], mvs[i], fov, atol, rtol, int(erode)))
    assert 0.2 < valid.mean() < 0.98
    pts = np.concatenate([fusion.world_points(depths[i], valid[i], fov, mvs[i]) for i in (0, 1)])
    grid = fusion.default_grid(pts, resolution, trunc)
    _check_against_oracle(f"warp fixture views, resolution {resolution}, trunc {trunc}", depths, colors, valid, mvs, fov, grid, trunc)


def test_fuse_views_is_the_oracle_pipeline(sphere_scene):
    """fuse_views (validity on the device mesh build, default grid, integrate, extract) against the oracle run on the grid
    it reports; max_depth drops the plane (depth about 2.5) and keeps the sphere (depth below 1)."""
    S = sphere_scene
    for max_depth in (None, 1.5):
        m = fusion.fuse_views(S.depths, S.colors, S.modelviews, fov=S.fov, resolution=80, max_depth=max_depth)
        valid = np.stack([fs.oracle_validity(S.depths[v], S.modelviews[v], max_depth=max_depth) for v in range(27)])
        ref = fr.integrate(S.depths, S.colors, valid, S.modelviews, S.fov, m.origin, m.voxel, m.dims, 3)
        rv, rc, rf = fr.extract(*ref, m.origin, m.voxel)
        assert np.array_equal(m.faces, rf) and np.array_equal(_bits(m.vertices), _bits(rv)) and np.array_equal(m.colors, rc)
        assert m.vertices.dtype == np.float32 and m.colors.dtype == np.uint8 and m.faces.dtype == np.int64
        if max_depth is not None:
            d, which = fs.surface_distance(m.vertices.astype(np.float64))
            assert (which == 1).all() and d.max() <= m.voxel, "only the sphere is left"


def test_empty_scene_gives_an_empty_mesh(sphere_scene):
    S = sphere_scene
    m = fusion.fuse_views(np.zeros_like(S.depths[:3]), S.colors[:3], S.modelviews[:3], fov=S.fov, resolution=33)
    assert m.vertices.shape == (0, 3) and m.colors.shape == (0, 3) and m.faces.shape == (0, 3)
    grid = fusion.default_grid(np.array([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]]), 33, 3)
    vol = fusion.tsdf_integrate(S.depths[:3], S.colors[:3], np.zeros((3, 64, 64), bool), S.modelviews[:3], S.fov, grid)
    assert float(vol.weight.abs().sum()) == 0 and float(vol.color_weight.abs().sum()) == 0
    mesh = fusion.extract_surface(vol, grid)
    assert mesh.vertices.shape[0] == 0 and mesh.faces.shape[0] == 0


def test_full_scale_scene():
    """27 views of 256^2 (the super-resolved scene size) at resolution 512 completes and stays on the surfaces."""
    S = fs.scene(n=256)
    m = fusion.fuse_views(S.depths, S.colors, S.modelviews, fov=S.fov, resolution=512)
    d, which = fs.surface_distance(m.vertices.astype(np.float64))
    print(f"[fusion] 27 x 256^2 at resolution 512: grid {m.dims}, {m.vertices.shape[0]} vertices, {m.faces.shape[0]} faces, "
          f"max distance to the surfaces {d.max() / m.voxel:.3f} voxels")
    assert m.vertices.shape[0] > 100000 and m.faces.shape[0] > 100000 and max(m.dims) >= 512
    assert d.max() <= m.voxel and (which == 1).sum() > 1000
    assert m.faces.min() >= 0 and m.faces.max() < m.vertices.shape[0]


def test_more_views_than_one_launch_carries(sphere_scene):
    """40 views: the integration runs in launches of 32 views and must equal the single-pass rule."""
    S = sphere_scene
    idx = list(range(27)) + list(range(13))
    pts = np.concatenate([fusion.world_points(S.depths[v], S.valid[v], S.fov, S.modelviews[v]) for v in range(27)])
    grid = fusion.default_grid(pts, 48, 3)
    _check_against_oracle("40 views (two launches)", S.depths[idx], S.colors[idx], S.valid[idx], [S.modelviews[v] for v in idx], S.fov, grid)


def test_export_cli(tmp_path):
    """save_scene -> python -m ivid_b200.inference.export -> PLY gives the arrays of fuse_views on the stored views, for a
    128^2 scene and a 256^2 (super-resolved size) one."""
    from ivid_b200.inference import load_scene_views, save_scene
    from ivid_b200.inference import export
    from ivid_b200.utils import edict
    os.makedirs(tmp_path / "scenes")
    mvs = fs.scene(n=8).modelviews[:9]
    for n in (128, 256):
        S = fs.scene(n=n, views=mvs)
        save_scene(str(tmp_path / "scenes" / f"{n:04d}.npz"), [edict(depth=S.depths[v][..., None], fov=S.fov, modelview=S.modelviews[v])
                                                              for v in range(len(mvs))], list(S.colors))
    export.main(["--scene_dir", str(tmp_path), "--output_dir", str(tmp_path / "out"), "--resolution", "72"])
    for n in (128, 256):
        views = load_scene_views(str(tmp_path / "scenes" / f"{n:04d}.npz"))
        assert views[0].color.shape == (n, n, 3)
        want = fusion.fuse_views(np.stack([v.depth[..., 0] for v in views]), np.stack([v.color for v in views]).astype(np.float32),
                                 [v.modelview for v in views], fov=views[0].fov, resolution=72)
        v, c, f = fs.read_ply(tmp_path / "out" / "meshes" / f"{n:04d}.ply")
        assert v.shape[0] > 500
        assert np.array_equal(v, want.vertices) and np.array_equal(c, want.colors) and np.array_equal(f, want.faces)

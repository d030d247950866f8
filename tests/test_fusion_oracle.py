"""CPU: the fusion rule of oracle/fusion_ref.py on the analytic sphere-and-plane scene (tests/fusion_scene.py), the PLY
writer, the default grid, and the argument checks of the Python layer and the C ABI (which run before any device work)."""
import ctypes

import numpy as np
import pytest

import fusion_scene as fs
from ivid_b200 import _lib
from ivid_b200.rgbd_3d import fusion
from oracle import fusion_ref as fr


@pytest.fixture(scope="module")
def scene():
    S = fs.scene(n=64)
    S.valid = np.stack([fs.oracle_validity(S.depths[v], S.modelviews[v]) for v in range(len(S.modelviews))])
    pts = np.concatenate([fusion.world_points(S.depths[v], S.valid[v], S.fov, S.modelviews[v]) for v in range(len(S.modelviews))])
    S.grid = fusion.default_grid(pts, 128, 3)
    S.volume = fr.integrate(S.depths, S.colors, S.valid, S.modelviews, S.fov, S.grid.origin, S.grid.voxel, S.grid.dims, 3)
    S.mesh = fr.extract(*S.volume, S.grid.origin, S.grid.voxel)
    return S


def test_silhouettes_are_invalid(scene):
    """The sphere's silhouettes are discontinuities: each view loses pixels around them and keeps both surfaces."""
    for v in range(len(scene.modelviews)):
        assert scene.hits[v].min() > 0, "every ray hits the sphere or the plane"
        assert not scene.valid[v].all() and scene.valid[v][scene.hits[v] == 1].any() and scene.valid[v][scene.hits[v] == 2].any()


def test_vertices_lie_on_the_surfaces(scene):
    """Every vertex lies within one voxel of the sphere or the plane."""
    verts, colors, faces = scene.mesh
    assert verts.shape[0] > 1000 and faces.shape[0] > 1000
    d, which = fs.surface_distance(verts.astype(np.float64))
    print(f"[fusion] {verts.shape[0]} vertices, {faces.shape[0]} faces; max distance to the surfaces "
          f"{d.max() / scene.grid.voxel:.3f} voxels; {(which == 1).sum()} on the sphere")
    assert d.max() <= scene.grid.voxel
    assert (which == 1).sum() > 100, "the sphere is part of the mesh"


def test_faces_point_out_of_the_surfaces(scene):
    verts, _, faces = scene.mesh
    a, b, c = (verts[faces[:, i]].astype(np.float64) for i in range(3))
    normal = np.cross(b - a, c - a)
    centre = (a + b + c) / 3
    _, which = fs.surface_distance(centre)
    sphere = which == 1
    assert sphere.sum() > 100
    assert ((normal[sphere] * centre[sphere]).sum(-1) > 0).all(), "sphere faces must face outwards"
    assert (normal[~sphere][:, 2] > 0).all(), "plane faces must face the cameras (+z)"


def test_edges_have_at_most_two_faces(scene):
    faces = scene.mesh[2]
    e = np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1)
    _, count = np.unique(e, axis=0, return_counts=True)
    assert count.max() <= 2
    assert faces.min() >= 0 and faces.max() < scene.mesh[0].shape[0]
    assert (faces[:, 0] != faces[:, 1]).all() and (faces[:, 1] != faces[:, 2]).all() and (faces[:, 0] != faces[:, 2]).all()


def test_vertex_colours_come_from_the_views(scene):
    verts, colors, _ = scene.mesh
    _, which = fs.surface_distance(verts.astype(np.float64))
    # the sphere is coloured 0.5 + 0.5 * p / r, so its vertices' colours follow their positions
    want = np.clip(0.5 + 0.5 * verts[which == 1] / fs.RADIUS, 0, 1) * 255
    assert np.abs(colors[which == 1].astype(np.float64) - want).mean() < 0.1 * 255


def test_all_invalid_view_changes_nothing(scene):
    S = scene
    k = 5
    base = fr.integrate(S.depths[:k], S.colors[:k], S.valid[:k], S.modelviews[:k], S.fov, S.grid.origin, S.grid.voxel, S.grid.dims, 3)
    valid = np.concatenate([S.valid[:k], np.zeros_like(S.valid[:1])])
    more = fr.integrate(np.concatenate([S.depths[:k], S.depths[k:k + 1]]), np.concatenate([S.colors[:k], S.colors[k:k + 1]]), valid,
                        S.modelviews[:k + 1], S.fov, S.grid.origin, S.grid.voxel, S.grid.dims, 3)
    for a, b in zip(base, more):
        assert np.array_equal(a, b)
    assert base[1].max() > 0


def test_single_view_tsdf_is_the_closed_form_sdf():
    """One camera at (0, 0, 1) facing the plane z = -1.5 alone: every pixel has depth 2.5 and a voxel at height z in the
    frustum gets tsdf = min(1, (z + 1.5) / (trunc * voxel)) as soon as z + 1.5 >= -trunc * voxel."""
    from ivid_b200.rgbd_3d.glm_compat import lookAt
    mv = lookAt((0.0, 0.0, 1.0), (0.0, 0.0, 0.0), (0.0, 1.0, 0.0))
    S = fs.scene(n=32, views=[mv], sphere=False)
    assert np.all(S.hits == 2) and np.all(S.depths == np.float32(2.5))
    valid = np.ones((1, 32, 32), bool)
    origin, voxel, dims, trunc = np.float32([-1.0, -1.0, -1.75]), np.float32(0.0625), [32, 32, 10], 2
    tsum, w, csum, cw = fr.integrate(S.depths, S.colors, valid, [mv], fs.FOV, origin, voxel, dims, trunc)
    k, j, i = np.meshgrid(*(np.arange(d) for d in dims[::-1]), indexing="ij")
    x, y, z = (origin[a] + (idx + 0.5) * np.float64(voxel) for a, idx in enumerate((i, j, k)))
    dist = 1.0 - z
    half = np.tan(np.deg2rad(fs.FOV) / 2) * dist
    tv = trunc * np.float64(voxel)
    sdf = 2.5 - dist
    seen = (np.abs(x) < half) & (np.abs(y) < half) & (sdf >= -tv)
    clear = (np.abs(np.abs(x) - half) > 1e-4) & (np.abs(np.abs(y) - half) > 1e-4) & (np.abs(sdf + tv) > 1e-4)
    assert seen[clear].sum() > 1000
    assert np.array_equal(w[clear] == 1, seen[clear]) and w.max() == 1
    want = np.minimum(1.0, sdf / tv)
    assert np.abs(tsum[seen & clear] - want[seen & clear]).max() < 1e-5
    near = seen & clear & (np.abs(sdf) <= tv - 1e-4)
    assert np.array_equal((cw == 1)[seen & clear & (np.abs(np.abs(sdf) - tv) > 1e-4)], near[seen & clear & (np.abs(np.abs(sdf) - tv) > 1e-4)])


def test_write_ply_round_trips(scene, tmp_path):
    verts, colors, faces = scene.mesh
    path = tmp_path / "scene.ply"
    fusion.write_ply(path, dict(vertices=verts, colors=colors, faces=faces))
    v, c, f = fs.read_ply(path)
    assert np.array_equal(v, verts) and np.array_equal(c, colors) and np.array_equal(f, faces)
    fusion.write_ply(tmp_path / "empty.ply", dict(vertices=np.zeros((0, 3)), colors=np.zeros((0, 3)), faces=np.zeros((0, 3))))
    v, c, f = fs.read_ply(tmp_path / "empty.ply")
    assert v.shape == (0, 3) and f.shape == (0, 3)


def test_default_grid():
    pts = np.array([[0.0, 0.0, 0.0], [2.0, 1.0, 0.5]])
    g = fusion.default_grid(pts, 8, 3)
    assert g.voxel == np.float32(0.25)
    assert np.array_equal(g.origin, np.float32([-1.0, -1.0, -1.0]))
    assert g.dims == [8 + 8, 4 + 8, 2 + 8]
    g = fusion.default_grid(np.zeros((0, 3)), 10, 1)      # no valid pixels: the cube of the cameras
    assert g.voxel == np.float32(0.2) and g.dims == [14, 14, 14]


def test_bad_arguments_raise_before_device_work():
    d = np.ones((1, 8, 8), np.float32); c = np.zeros((1, 8, 8, 3), np.float32); m = np.ones((1, 8, 8), bool); mv = [np.eye(4)]
    good = dict(origin=[0, 0, 0], voxel=0.1, dims=[4, 4, 4])
    cases = [(dict(good, dims=[1, 4, 4]), 3, "dims"), (dict(good, voxel=0.0), 3, "voxel"), (dict(good, voxel=-1.0), 3, "voxel"),
             (good, 0, "trunc"), (good, -2.0, "trunc"), (dict(good, dims=[2048, 1024, 1024]), 3, "32-bit")]
    for grid, trunc, what in cases:
        with pytest.raises(ValueError, match=what):
            fusion.tsdf_integrate(d, c, m, mv, 45, grid, trunc)
    with pytest.raises(ValueError, match="at least one view"):
        fusion.tsdf_integrate(d[:0], c[:0], m[:0], np.zeros((0, 4, 4)), 45, good, 3)
    with pytest.raises(ValueError, match="colors"):
        fusion.tsdf_integrate(d, c[..., :2], m, mv, 45, good, 3)
    with pytest.raises(ValueError, match="resolution"):
        fusion.fuse_views(d, c, mv, resolution=0)
    with pytest.raises(ValueError, match="trunc"):
        fusion.fuse_views(d, c, mv, trunc=0)
    with pytest.raises(ValueError, match="dims"):
        fusion.extract_surface({}, dict(good, dims=[4, 0, 4]))


def test_c_abi_rejects_bad_arguments_before_any_launch():
    """The entry points check every argument before they touch a pointer or the device (the fake pointers below are never
    dereferenced), so this runs without a GPU."""
    L = _lib.lib()
    fake = ctypes.c_void_p(64)
    mv = np.eye(4, dtype=np.float32)

    def grid(origin=(0.0, 0.0, 0.0), voxel=0.1, dims=(4, 4, 4)):
        g = _lib.FusionGridT()
        g.origin[:] = list(origin); g.voxel = voxel; g.dims[:] = list(dims)
        return g

    def integrate(g, views=1, n=8, focal=1.2, trunc=3.0):
        return L.ivid_fusion_integrate(fake, fake, fake, mv.ctypes.data, views, n, focal, ctypes.byref(g), trunc, fake, fake, fake, fake, None)

    bad = [integrate(grid(dims=(1, 4, 4))), integrate(grid(dims=(4, 4, -3))), integrate(grid(voxel=0.0)), integrate(grid(voxel=-0.5)),
           integrate(grid(voxel=float("nan"))), integrate(grid(origin=(0.0, float("inf"), 0.0))), integrate(grid(), trunc=0.0),
           integrate(grid(), trunc=-1.0), integrate(grid(), views=0), integrate(grid(), n=0), integrate(grid(), focal=0.0),
           integrate(grid(dims=(2048, 1024, 1024))), integrate(grid(dims=(65536, 65536, 2)))]
    assert bad == [_lib.IVID_ERR_INVALID_ARGUMENT] * len(bad)
    assert "32-bit" in _lib.last_error()
    assert L.ivid_fusion_integrate(None, fake, fake, mv.ctypes.data, 1, 8, 1.2, ctypes.byref(grid()), 3.0, fake, fake, fake, fake,
                                   None) == _lib.IVID_ERR_INVALID_ARGUMENT
    nv, nf = ctypes.c_int64(-1), ctypes.c_int64(-1)
    for g in (grid(dims=(4, 1, 4)), grid(voxel=0.0), grid(dims=(2048, 1024, 1024))):
        rc = L.ivid_fusion_extract(ctypes.byref(g), fake, fake, fake, fake, 0, 0, None, None, None, ctypes.byref(nv), ctypes.byref(nf), None)
        assert rc == _lib.IVID_ERR_INVALID_ARGUMENT
    assert L.ivid_fusion_extract(None, fake, fake, fake, fake, 0, 0, None, None, None, ctypes.byref(nv), ctypes.byref(nf),
                                 None) == _lib.IVID_ERR_INVALID_ARGUMENT
    assert nv.value == -1 and nf.value == -1

"""CPU: the warp oracle (numpy restatement of rgbd_3d/utils.py + C restatement of the GL pipeline) against the
committed golden fixture (tests/golden/make_warp_golden.py ran the reference's own utils.py around it)."""
import numpy as np
import pytest

from oracle import warp_ref
from conftest import ROOT
import os


@pytest.fixture(scope="module")
def wg():
    return {k: v for i in (0, 1) for k, v in np.load(os.path.join(ROOT, "tests", "golden", f"warp_golden_part{i}.npz")).items()}


def _meshes(wg, k):
    near, far, fov, atol, rtol, erode = (float(v) for v in wg["params"])   # python floats: numpy weak-scalar promotion
    ms, cs = [], []
    for i in range(k):
        rgbd = wg[f"rgbd{i}"]
        ms.append(warp_ref.depth_to_mesh(warp_ref.linearize_depth(rgbd[:, :, 3:], near, far), fov=fov, modelview=wg["views"][i],
                                         atol=atol, rtol=rtol, erode_rgb=int(erode)))
        cs.append(rgbd[:, :, :3])
    return ms, cs


def test_mesh_checksums(wg):
    ms, _ = _meshes(wg, 2)
    for i, m in enumerate(ms):
        vb = warp_ref.mesh_vertex_buffer(m)
        assert vb.shape == (130 * 130, 9) and m.faces.shape == (2 * 129 * 129, 3)
        assert np.allclose(vb.astype(np.float64).sum(0), wg[f"mesh{i}_colsum"], rtol=1e-9, atol=1e-6)
        assert np.array_equal(np.bincount(vb[:, 8].astype(np.int64), minlength=8), wg[f"mesh{i}_flaghist"])
        assert m.faces.astype(np.int64).sum() == wg[f"mesh{i}_faces_sum"][0]


def test_numeric_padding_mesh_checksums(wg):
    """depth_to_mesh(depth, 32, ...) — the meshing of inference/utils.py:load_scene (free-view rendering): same grid, border
    ring pushed out 32 pixels and NOT pulled to the near plane.  Pinned bit-identical to the reference by make_warp_golden."""
    near, far, fov, atol, rtol, erode = (float(v) for v in wg["params"])
    for i in range(2):
        d = warp_ref.linearize_depth(wg[f"rgbd{i}"][:, :, 3:], near, far)
        m = warp_ref.depth_to_mesh(d, fov=fov, modelview=wg["views"][i], atol=atol, rtol=rtol, erode_rgb=int(erode), padding=32)
        vb = warp_ref.mesh_vertex_buffer(m)
        assert np.allclose(vb.astype(np.float64).sum(0), wg[f"meshpad{i}_colsum"], rtol=1e-9, atol=1e-6)
        assert np.allclose(np.abs(vb.astype(np.float64)).sum(0), wg[f"meshpad{i}_abssum"], rtol=1e-9, atol=1e-6)
        assert np.array_equal(np.bincount(vb[:, 8].astype(np.int64), minlength=8), wg[f"meshpad{i}_flaghist"])
        assert m.faces.astype(np.int64).sum() == wg[f"meshpad{i}_faces_sum"][0]
        # differs from the frustum mesh only on the border ring
        f = warp_ref.depth_to_mesh(d, fov=fov, modelview=wg["views"][i], atol=atol, rtol=rtol, erode_rgb=int(erode))
        inner = np.ones((130, 130), bool); inner[0, :] = inner[-1, :] = inner[:, 0] = inner[:, -1] = False
        assert np.array_equal(m.vertices.position.reshape(130, 130, 3)[inner], f.vertices.position.reshape(130, 130, 3)[inner])
        assert not np.array_equal(m.vertices.position, f.vertices.position)


def test_aggregate_conditions_matches_golden(wg):
    near, far, fov, atol, rtol, erode = (float(v) for v in wg["params"])
    ms, cs = _meshes(wg, 2)
    rend = warp_ref.SoftwareAggregationRenderer(384, 128)
    for j in range(2):
        c = warp_ref.aggregate_conditions(rend, ms[: j + 1], cs[: j + 1], wg["views"][j + 1], fov=fov, near=near, far=far, atol=atol,
                                          rtol=rtol, erode_rgb=int(erode))
        for k in ["mask", "mask_rgb"]:
            assert (np.asarray(c[k], np.float32) != wg[f"cond{j}_{k}"]).mean() < 1e-3, k
        agree = (c["mask"] == wg[f"cond{j}_mask"])[..., 0]
        assert np.abs(np.asarray(c["depth"], np.float32) - wg[f"cond{j}_depth"])[agree].max() < 1e-5
        assert np.abs(np.asarray(c["color"], np.float32) - wg[f"cond{j}_color"]).max() <= 1.0 / 255 + 1e-6


def test_self_reprojection_property(wg):
    """A view rendered from its own camera reproduces its own colours (NEAREST texels at pixel centres) and depth."""
    near, far, fov, *_ = (float(v) for v in wg["params"])
    ms, cs = _meshes(wg, 1)
    raw = warp_ref.SoftwareAggregationRenderer(384, 128).render(ms, cs, wg["views"][0], fov, is_autoregressive=True)
    rec = np.array(raw.color).reshape(128, 3, 128, 3, 3)[:, 1, :, 1]
    assert np.abs(rec - cs[0]).max() < 1e-6
    assert np.abs(raw.depth[1::3, 1::3, 0] - warp_ref.linearize_depth(wg["rgbd0"][:, :, 3], near, far)).max() < 2e-3
    assert raw.mask_depth.mean() > 0.95      # discontinuity-flagged faces carry weight 1e-16 (mask_depth 0)


def test_depth_roundtrip_and_glm(wg):
    d = np.linspace(0.01, 0.99, 200).astype(np.float32)
    z = warp_ref.linearize_depth(d, 0.6, 5)
    assert np.abs(warp_ref.project_depth(z, 0.6, 5) - d).max() < 1e-6
    mv = warp_ref.view_on_sphere(0.3, -0.15)
    assert np.allclose(mv[:3, :3] @ mv[:3, :3].T, np.eye(3), atol=1e-6)          # rigid
    assert np.allclose(warp_ref.inverse(mv)[:3, 3], [np.sin(0.3) * np.cos(-0.15), np.sin(-0.15), np.cos(0.3) * np.cos(-0.15)], atol=1e-6)
    P = warp_ref.perspective(np.deg2rad(45), 1, 0.01, 200)
    assert abs(P[0, 0] - 1 / np.tan(np.deg2rad(22.5))) < 1e-6 and P[3, 2] == -1


def test_forward_backward_warp_matches_golden(wg):
    """Training-pair warp (utils.py:335-417 around SimpleRenderer, datasets/base.py:219-238) — §8(f) row 3 oracle, pinned
    against the reference's numpy / PIL steps by make_warp_golden.py."""
    fov = float(wg["params"][2])
    simple = warp_ref.SoftwareSimpleRenderer(384, 128, near=0.1, far=200)
    r = warp_ref.forward_backward_warp(simple, wg["rgbd0"], wg["views"][2], modelview0=wg["views"][0], padding=128, fov=fov, near=0.5, far=100)
    assert (np.asarray(r.mask, np.float32) != wg["fbw_mask"]).mean() < 1e-3
    agree = (r.mask == wg["fbw_mask"])[..., 0]
    assert np.abs(np.asarray(r.depth, np.float32) - wg["fbw_depth"])[agree].max() < 1e-5
    assert np.abs(np.asarray(r.color, np.float32) - wg["fbw_color"])[agree].max() <= 1.0 / 255 + 1e-6
    assert 0.5 < float(r.mask.mean()) < 0.95
    # property: warping to the SAME camera and back keeps (almost) everything and reproduces the input
    same = warp_ref.forward_backward_warp(simple, wg["rgbd0"], wg["views"][0], modelview0=wg["views"][0], padding=128, fov=fov, near=0.5, far=100)
    keep = same.mask[..., 0] > 0
    assert keep.mean() > 0.9
    cerr = np.abs(same.color - wg["rgbd0"][:, :, :3])[keep]
    assert np.quantile(cerr, 0.95) <= 2.0 / 255 + 1e-6 and cerr.max() < 0.1     # two 8-bit LANCZOS passes: ringing only at colour edges
    assert np.abs(same.depth[..., 0] - wg["rgbd0"][:, :, 3])[keep].max() < 1e-5

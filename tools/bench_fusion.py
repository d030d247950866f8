"""Micro-benchmark of the mesh export (csrc/fusion.cu): CUDA-event times of ivid_fusion_integrate and of the surface
extraction (the count call, the host read of the two counts and the fill call, as extract_surface runs them) for the
analytic sphere-and-plane scene of tests/fusion_scene.py at 27 views of 128^2 and 256^2, grid resolutions 256 and 512.

Rates come from the shapes: integrate does V * voxels voxel-view projections and writes 24 bytes per voxel (tsdf sum,
weight, colour sum, colour weight); extraction reads those 24 bytes per voxel at least once.  The card's name and power
limit are read in the same run.  Prints one JSON line."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import fusion_scene as fs  # noqa: E402
from ivid_b200.rgbd_3d import fusion  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power = q.stdout.strip().splitlines()[0].split(", ")
    return name, power


def timed(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    out = fn()                                          # warm-up: module load, memory pool
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(reps):
        out = fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps, out


def main():
    reps = int(os.environ.get("REPS", 5))
    name, power = card()
    rows = []
    for n in (128, 256):
        S = fs.scene(n=n)
        valid = np.stack([fusion.view_validity(S.depths[v], S.fov, S.modelviews[v]) for v in range(len(S.modelviews))])
        pts = np.concatenate([fusion.world_points(S.depths[v], valid[v], S.fov, S.modelviews[v]) for v in range(len(S.modelviews))])
        d = torch.from_numpy(S.depths).cuda(); c = torch.from_numpy(S.colors).cuda(); m = torch.from_numpy(valid).cuda()
        for res in (256, 512):
            grid = fusion.default_grid(pts, res, 3)
            nvox = int(np.prod(grid.dims))
            t_int, vol = timed(lambda: fusion.tsdf_integrate(d, c, m, S.modelviews, S.fov, grid, 3), reps)
            t_ext, mesh = timed(lambda: fusion.extract_surface(vol, grid), reps)
            V = len(S.modelviews)
            rows.append({"views": V, "image": n, "resolution": res, "dims": grid.dims, "voxels": nvox,
                         "integrate_ms": round(t_int, 3), "extract_ms": round(t_ext, 3),
                         "projections_per_s": V * nvox / (t_int / 1e3), "integrate_GBs": 24 * nvox / 1e9 / (t_int / 1e3),
                         "extract_GBs": 24 * nvox / 1e9 / (t_ext / 1e3),
                         "vertices": int(mesh.vertices.shape[0]), "faces": int(mesh.faces.shape[0])})
            del vol, mesh
            torch.cuda.empty_cache()
    print(json.dumps({"card": name, "power_limit": power, "reps": reps, "rows": rows}))


if __name__ == "__main__":
    main()

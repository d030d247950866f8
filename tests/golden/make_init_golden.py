"""Golden fixtures of starting a run from a given image, from the UNMODIFIED reference:

    diffuse_*   GaussianDiffusion.diffuse (gaussian_diffusion.py:45-64) with given noise at several t, linear and cosine
                schedules (T = 1000): what ivid_sampler_diffuse must reproduce
    prep_*      the datasets' RGBD preprocessing (datasets/base.py:92-126, BaseDataset.get_file + process_file) of a
                synthetic photo and disparity map: the conditional config's dataset.args at its image_size, and every
                prepocess_depth mode at a small size, from a landscape, a portrait and a grayscale image

    python tests/golden/make_init_golden.py        # needs the reference checkout (IVID_REF); writes tests/golden/init_golden.npz
"""
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg          # noqa: E402  (easydict shim + reference imports; does not regenerate anything on import)

# datasets/base.py imports glm and rgbd_3d for the training-pair warp, which get_file / process_file do not use
for name in ("glm", "rgbd_3d"):
    sys.modules.setdefault(name, types.ModuleType(name))
from diffusion.frameworks.gaussian_diffusion import GaussianDiffusion   # noqa: E402
from datasets.base import BaseDataset                                   # noqa: E402

COND_CONFIG = "rgbd_imagenet_adm_128_large_cond.json"
DIFFUSE_T = (0, 1, 7, 250, 499, 500, 998, 999)
MODES = ("none", "to_depth", "disparity_minmax", "depth_minmax", "z_buffer")


class _Net:
    def forward(self, x, t, classes=None):
        return x


def synthetic_view(h, w, gray, seed):
    """A smooth photo (uint8) and a disparity map in the range MiDaS writes (0 .. ~6e4, larger is nearer)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([127 + 100 * np.sin(xx / (5 + 3 * c) + yy / (7 + c)) for c in range(3)], -1) + rng.normal(0, 12, (h, w, 3))
    img = np.clip(img, 0, 255).astype(np.uint8)
    if gray:
        img = img[:, :, 0]
    disp = 2.0e4 + 1.5e4 * np.sin(xx / 11.0) * np.cos(yy / 9.0) + 4.0e4 * (yy / h) + rng.uniform(0, 500, (h, w))
    return img, disp.astype(np.float32)


def reference_view(img, disp, args):
    """BaseDataset.getitem of one file pair through the reference's own transforms."""
    from PIL import Image
    with tempfile.TemporaryDirectory() as d:
        Image.fromarray(img).save(os.path.join(d, "im.png"))
        np.savez(os.path.join(d, "im.npz"), disp)
        ds = BaseDataset(d, **args)
        ds.images, ds.depths = ["im.png"], ["im.npz"]
        return ds.getitem(0)["x_0"].numpy()


if __name__ == "__main__":
    out = {}
    rng = np.random.default_rng(11)
    x0 = rng.uniform(-1, 1, (2, 4, 8, 8)).astype(np.float32)
    noise = rng.standard_normal((2, 4, 8, 8)).astype(np.float32)
    out["diffuse_x0"], out["diffuse_noise"], out["diffuse_t"] = x0, noise, np.array(DIFFUSE_T, dtype=np.int64)
    for sched in ("linear", "cosine"):
        fw = GaussianDiffusion(_Net(), timesteps=1000, beta_schedule=sched)
        outs = []
        for t in DIFFUSE_T:
            tt = torch.full((2,), t, dtype=torch.int64)
            outs.append(fw.diffuse(torch.from_numpy(x0), tt, noise=torch.from_numpy(noise)).numpy())
        out[f"diffuse_{sched}"] = np.stack(outs)

    cond_args = json.load(open(os.path.join(mg.REF, "configs", COND_CONFIG)))["dataset"]["args"]
    base = {k: cond_args[k] for k in ("image_size", "normalize", "normalize_depth", "prepocess_depth", "near", "far")}
    cases = [("cond", 150, 200, False, dict(base))]
    for mode in MODES:
        for tag, h, w, gray in (("land", 45, 70, False), ("port", 90, 61, False), ("gray", 32, 32, True)):
            args = dict(base, image_size=32, prepocess_depth=mode, normalize_depth=mode not in ("none", "to_depth"))
            cases.append((f"{mode}_{tag}", h, w, gray, args))
    names = []
    for i, (tag, h, w, gray, args) in enumerate(cases):
        img, disp = synthetic_view(h, w, gray, seed=100 + i)
        out[f"prep_{tag}_image"], out[f"prep_{tag}_disparity"] = img, disp
        out[f"prep_{tag}_args"] = np.frombuffer(json.dumps(args).encode(), dtype=np.uint8)
        out[f"prep_{tag}_x0"] = reference_view(img, disp, args)
        names.append(tag)
    out["prep_cases"] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)
    path = os.path.join(HERE, "init_golden.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes, {len(names)} preprocessing cases)")

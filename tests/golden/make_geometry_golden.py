"""Golden eps of the UNMODIFIED reference UNet at input sizes other than a square power of two, on the tiny test architecture
with the oracle's synthetic weights (adm.py:526-566 accepts any H x W divisible by 2^(levels-1); attention placement follows
image_size).  The oracle is asserted bit-equal to the reference for every case.

    np2         image_size=48, attention at 24 and 12           T = 576, 144
    np2_single  the same, num_heads=1, num_head_channels=-1      one head of 128 at T = 576, 144
    short       channel_mult=[1,2,2,2], attention at 8 and 4     T = 64, 16
    rect        a 40 x 24 input to the 32 model                  T = 240, 60
    big         a 64 x 64 input to the 32 model                  T = 1024, 256
    sr4 / sr3   SuperResCFG.model_inference of the tiny SR model, 8^2 -> 32^2 and 16^2 -> 48^2, classes, strength 0.5;
                also the upsampled half of make_cond_inputs (sr_cfg.py:31-36, scale_factor = s)

    python tests/golden/make_geometry_golden.py     # needs /root/reference; writes tests/golden/geometry_golden.npz
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg          # noqa: E402  (easydict shim + reference imports; does not regenerate anything on import)
from oracle import sampler_ref, unet_ref       # noqa: E402

# tag -> (config overrides of make_golden.TINY, batch, H, W)
UNET_CASES = (("np2", dict(image_size=48, attention_resolutions=[24, 12]), 2, 48, 48),
              ("np2_single", dict(image_size=48, attention_resolutions=[24, 12], num_heads=1, num_head_channels=-1), 2, 48, 48),
              ("short", dict(channel_mult=[1, 2, 2, 2], attention_resolutions=[8, 4]), 2, 32, 32),
              ("rect", dict(), 2, 40, 24),
              ("big", dict(), 1, 64, 64))
# tag -> (low-res size, high-res size)
SR_CASES = (("sr4", 8, 32), ("sr3", 16, 48))
SR_STRENGTH = 0.5

if __name__ == "__main__":
    out = {}
    for tag, extra, N, H, W in UNET_CASES:
        cfg = dict(mg.TINY, **extra)
        sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
        net = mg.ref_model(cfg, sd)
        rng = np.random.default_rng(5)
        x = torch.from_numpy(rng.standard_normal((N, 4, H, W)).astype(np.float32))
        t = torch.tensor([700, 3][:N]); c = torch.tensor([4, -1][:N])
        with torch.no_grad():
            ref = net(x, t, c)
        ora = unet_ref.unet_forward(cfg, sd, x, t, c)
        assert torch.equal(ref, ora), f"{tag}: oracle differs from the reference by {float((ref - ora).abs().max())}"
        out[f"{tag}_cfg"] = np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8)
        out[f"{tag}_x"] = x.numpy(); out[f"{tag}_t"] = t.numpy(); out[f"{tag}_c"] = c.numpy(); out[f"{tag}_eps"] = ref.numpy()
        print(f"{tag}: {H}x{W} eps std {float(ref.std()):.3f}")
    cfg = dict(mg.TINY_SR)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    fw = mg.ref_frameworks.SuperResCFG(mg.ref_model(cfg, sd), timesteps=1000, beta_schedule="linear")
    model = lambda xx, tt, cc: unet_ref.unet_forward(cfg, sd, xx, tt, cc)
    for tag, lo, hi in SR_CASES:
        rng = np.random.default_rng(9)
        x = torch.from_numpy(rng.standard_normal((2, 4, hi, hi)).astype(np.float32))
        y = torch.from_numpy(rng.uniform(-1, 1, (2, 4, lo, lo)).astype(np.float32))
        t = torch.tensor([700, 3]); c = torch.tensor([4, 7])
        ci = fw.make_cond_inputs(x, y)
        assert torch.equal(ci, sampler_ref.make_sr_inputs(x, y))
        with torch.no_grad():
            ref = fw.model_inference(x, t, y, c, strength=SR_STRENGTH)
        ora = sampler_ref.cond_eps(model, sampler_ref.make_sr_inputs(x, y), t, c, SR_STRENGTH)
        assert torch.equal(ref, ora), f"{tag}: oracle differs from the reference by {float((ref - ora).abs().max())}"
        out[f"{tag}_cfg"] = np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8)
        out[f"{tag}_x"] = x.numpy(); out[f"{tag}_y"] = y.numpy(); out[f"{tag}_t"] = t.numpy(); out[f"{tag}_c"] = c.numpy()
        out[f"{tag}_eps"] = ref.numpy()
        out[f"{tag}_up"] = ci[:, 4:].numpy()        # the x half of make_cond_inputs is x itself
        print(f"{tag}: {lo}^2 -> {hi}^2 eps std {float(ref.std()):.3f}")
    path = os.path.join(HERE, "geometry_golden.npz")
    np.savez_compressed(path, **out)
    print(f"written {path} ({os.path.getsize(path) / 1024:.0f} KiB)")

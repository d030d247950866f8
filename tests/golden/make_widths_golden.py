"""Golden eps of the UNMODIFIED reference UNet at channel widths that are not multiples of 64, on the tiny test architecture
(make_golden.TINY at 32^2, N = 2) with the oracle's synthetic weights.  The reference builds every level at
int(channel_mult[i] * model_channels) channels (adm.py:367,385,454) and only needs num_groups to divide each width
(GroupNorm32).  The oracle is asserted bit-equal to the reference for every case.

    mc96      model_channels=96, channel_mult=[1,2,2], attention at 16 and 8     concats 192+192, 192+96, 96+96
    mc32      model_channels=32, channel_mult=[1,2,4], attention at 8            GroupNorm groups of one channel
    frac      model_channels=64, channel_mult=[1,1.5,2], attention at 8          widths 64, 96, 128
    g8        num_groups=8, model_channels=40, channel_mult=[1,2,3.2], none       widths 40, 80, 128 (groups of 5 and 10)
    narrow8   num_groups=8, model_channels=8, channel_mult=[1,2,8], none          widths 8, 16, 64: the output head runs at
              final width 8, and no full-resolution ResBlock reaches 64 channels
    legacy96  mc96 with use_scale_shift_norm=False, resblock_updown=False         stride-2 conv (im2col) and upsample conv
    inpaint96 InpaintCFG.model_inference at mc96 with in_channels=10, classes, strength 0.5, injected hole noise
    g4_20     num_groups=4, model_channels=20, channel_mult=[1,3.2]              widths 20, 64, 84, 40: the reference runs it,
              this package raises NotImplementedError (20 is not a multiple of 8); only the config is stored

    python tests/golden/make_widths_golden.py     # needs /root/reference; writes tests/golden/widths_golden.npz
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

MC96 = dict(model_channels=96, channel_mult=[1, 2, 2], attention_resolutions=[16, 8])
# tag -> config overrides of make_golden.TINY
UNET_CASES = (("mc96", MC96),
              ("mc32", dict(model_channels=32, channel_mult=[1, 2, 4], attention_resolutions=[8])),
              ("frac", dict(model_channels=64, channel_mult=[1, 1.5, 2], attention_resolutions=[8])),
              ("g8", dict(num_groups=8, model_channels=40, channel_mult=[1, 2, 3.2], attention_resolutions=[])),
              ("narrow8", dict(num_groups=8, model_channels=8, channel_mult=[1, 2, 8], attention_resolutions=[])),
              ("legacy96", dict(MC96, use_scale_shift_norm=False, resblock_updown=False)))
INPAINT = dict(MC96, in_channels=10)
G4_20 = dict(num_groups=4, model_channels=20, channel_mult=[1, 3.2], attention_resolutions=[])
STRENGTH = 0.5

if __name__ == "__main__":
    out = {}
    N, S = 2, 32
    t = torch.tensor([700, 3]); c = torch.tensor([4, -1])
    for tag, extra in UNET_CASES + (("g4_20", G4_20),):
        cfg = dict(mg.TINY, **extra)
        sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
        net = mg.ref_model(cfg, sd)
        rng = np.random.default_rng(5)
        x = torch.from_numpy(rng.standard_normal((N, 4, S, S)).astype(np.float32))
        with torch.no_grad():
            ref = net(x, t, c)
        ora = unet_ref.unet_forward(cfg, sd, x, t, c)
        assert torch.equal(ref, ora), f"{tag}: oracle differs from the reference by {float((ref - ora).abs().max())}"
        out[f"{tag}_cfg"] = np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8)
        if tag != "g4_20":
            out[f"{tag}_x"] = x.numpy(); out[f"{tag}_t"] = t.numpy(); out[f"{tag}_c"] = c.numpy(); out[f"{tag}_eps"] = ref.numpy()
        print(f"{tag}: eps std {float(ref.std()):.3f}")

    cfg = dict(mg.TINY, **INPAINT)
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    fw = mg.ref_frameworks.InpaintCFG(mg.ref_model(cfg, sd), timesteps=1000, beta_schedule="linear")
    rng = np.random.default_rng(11)
    x = torch.from_numpy(rng.standard_normal((N, 4, S, S)).astype(np.float32))
    y = torch.from_numpy(rng.uniform(-1, 1, (N, 4, S, S)).astype(np.float32))
    mask = torch.from_numpy((rng.uniform(size=(N, 1, S, S)) < 0.7).astype(np.float32))
    mask_rgb = mask * torch.from_numpy((rng.uniform(size=(N, 1, S, S)) < 0.8).astype(np.float32))
    z_rgb = torch.from_numpy(rng.standard_normal((N, 3, S, S)).astype(np.float32))
    z_d = torch.from_numpy(rng.standard_normal((N, 1, S, S)).astype(np.float32))
    ci = torch.tensor([2, 9])
    with torch.no_grad(), mg.FixedNoise([z_rgb, z_d]):
        ref = fw.model_inference(x, t, y, mask, ci, strength=STRENGTH, mask_rgb=mask_rgb)
    model = lambda xx, tt, cc: unet_ref.unet_forward(cfg, sd, xx, tt, cc)
    ora = sampler_ref.cond_eps(model, sampler_ref.make_inpaint_inputs(x, y, mask, mask_rgb, z_rgb, z_d), t, ci, STRENGTH)
    assert torch.equal(ref, ora), f"inpaint96: oracle differs from the reference by {float((ref - ora).abs().max())}"
    out["inpaint96_cfg"] = np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8)
    for k, v in dict(x=x, t=t, c=ci, y=y, mask=mask, mask_rgb=mask_rgb, noise=torch.cat([z_rgb, z_d], 1), eps=ref).items():
        out[f"inpaint96_{k}"] = v.numpy()
    print(f"inpaint96: eps std {float(ref.std()):.3f}")

    path = os.path.join(HERE, "widths_golden.npz")
    np.savez_compressed(path, **out)
    print(f"written {path} ({os.path.getsize(path) / 1024:.0f} KiB)")

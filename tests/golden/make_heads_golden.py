"""Golden eps of the UNMODIFIED reference UNet at attention head widths other than 64 (adm.py:266-273 num_heads /
num_head_channels, QKVAttention adm.py:233-253), on the tiny test architecture with the oracle's synthetic weights; pins the
oracle's attention for any head width.

    hc128   num_head_channels=128                  1 x 128 at T=256, 2 x 128 at T=64
    nh4     num_heads=4, num_head_channels=-1      4 x 64 and 4 x 192 in one network
    single  num_heads=1, num_head_channels=-1      1 x 256 at T=256, 1 x 512 at T=64 (the reference's constructor defaults)

    python tests/golden/make_heads_golden.py        # needs /root/reference; writes tests/golden/heads_golden.npz
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg          # noqa: E402  (easydict shim + reference imports; does not regenerate anything on import)
from oracle import unet_ref       # noqa: E402

CASES = (("hc128", dict(channel_mult=[1, 2, 4], num_head_channels=128)),
         ("nh4", dict(model_channels=256, channel_mult=[1, 1, 3], num_heads=4, num_head_channels=-1)),
         ("single", dict(model_channels=128, channel_mult=[1, 2, 4], num_heads=1, num_head_channels=-1)))

if __name__ == "__main__":
    out = {}
    for tag, extra in CASES:
        cfg = dict(mg.TINY, **extra)
        sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
        net = mg.ref_model(cfg, sd)
        rng = np.random.default_rng(5)
        x = torch.from_numpy(rng.standard_normal((2, 4, 32, 32)).astype(np.float32))
        t = torch.tensor([700, 3]); c = torch.tensor([4, -1])
        with torch.no_grad():
            ref = net(x, t, c)
        ora = unet_ref.unet_forward(cfg, sd, x, t, c)
        assert torch.equal(ref, ora), f"{tag}: oracle differs from the reference by {float((ref - ora).abs().max())}"
        out[f"{tag}_cfg"] = np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8)
        out[f"{tag}_x"] = x.numpy(); out[f"{tag}_t"] = t.numpy(); out[f"{tag}_c"] = c.numpy(); out[f"{tag}_eps"] = ref.numpy()
        print(f"{tag}: eps std {float(ref.std()):.3f}")
    np.savez_compressed(os.path.join(HERE, "heads_golden.npz"), **out)
    print("written", {k: v.shape for k, v in out.items()})

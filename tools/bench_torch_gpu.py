"""Secondary baseline (SURVEY.md §8d): the PyTorch restatement of the reference path (oracle/unet_ref.py +
oracle/sampler_ref.py, i.e. what the reference's own modules launch) run EAGERLY on the same GPU through stock
PyTorch kernels (cuDNN / cuBLAS), for the bench workload: one DDPM + classifier-free-guidance denoising step of batch 16
on the large 128x128 model (two sequential batch-16 forwards, as the reference does).  Measurement tooling only.

    python tools/bench_torch_gpu.py [--steps 5]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (LARGE_CFG, GUIDANCE)
from oracle import sampler_ref, unet_ref  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=16)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    sd = {k: v.to(dev) for k, v in unet_ref.make_synthetic_state_dict(bench.LARGE_CFG, seed=1234).items()}
    tb = sampler_ref.Tables(sampler_ref.get_betas("linear", 1000))
    B = args.batch
    out = {"workload": "DDPM+CFG denoising step, batch %d, large 128x128 model, eager PyTorch %s on %s" % (
        B, torch.__version__, torch.cuda.get_device_name(0)), "modes": {}}
    for mode in ("fp32_tf32", "fp16_autocast"):
        torch.backends.cuda.matmul.allow_tf32 = True
        torch.backends.cudnn.allow_tf32 = True          # PyTorch 1.11 default of the reference environment
        g = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(B, 4, 128, 128, generator=g, device=dev)
        classes = (torch.arange(B, device=dev) % 1000)

        def model(xx, t, c):
            if mode == "fp16_autocast":
                with torch.autocast("cuda", dtype=torch.float16):
                    return unet_ref.unet_forward(bench.LARGE_CFG, sd, xx, t, c).float()
            return unet_ref.unet_forward(bench.LARGE_CFG, sd, xx, t, c)

        def one(i):
            nonlocal x
            t = torch.full((B,), 999 - i, device=dev, dtype=torch.long)
            eps = sampler_ref.cfg_eps(model, x, t, classes, bench.GUIDANCE)
            x, _ = sampler_ref.ddpm_step(tb, x, t, eps, torch.randn(x.shape, generator=g, device=dev))

        try:
            with torch.no_grad():
                for i in range(3):
                    one(i)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(args.steps):
                    one(3 + i)
                e1.record()
                torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            out["modes"][mode] = {"ms_per_step": ms, "samples_per_s": B / (1000 * ms * 1e-3), "finite": bool(torch.isfinite(x).all())}
        except Exception as e:  # noqa: BLE001 - report, do not hide
            out["modes"][mode] = {"error": repr(e)[:300]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

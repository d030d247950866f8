"""Forward time of AdmUnet2d at channel widths that are and are not multiples of 64: the rgbd_singlecategory_adm_128_small
backbone with channel_mult=[1,1,2,2,4] (the shipped [1,1,2,3,4] gives a 288-wide attention level at 96 channels, which the
reference rejects with 64-channel heads) at model_channels 96, 128, 160 and 192; 128 and 192 are the controls.  Widths
that are not multiples of 64 pad K to whole 64-channel chunks and Cout to the tile inside the GEMM, so this measures what
the padding costs.  Prints one JSON line.

    python tools/bench_widths.py [--batch 32] [--iters 20] [--warmup 5]

ms: CUDA events around `iters` back-to-back forwards (CUDA-graph replays), after `warmup` forwards.  TFLOP/s are algorithmic:
the FLOPs the plan tags its launches with (real channel counts, no padding), over that time.  Needs a GPU: there is no
fallback."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch                                      # noqa: E402

import ivid_b200.backbones as backbones           # noqa: E402
from ivid_b200 import _lib                        # noqa: E402
from oracle import unet_ref                       # noqa: E402

SMALL_128 = dict(image_size=128, in_channels=4, out_channels=4, model_channels=128, num_res_blocks=2, num_classes=None,
                 has_null_class=False, channel_mult=[1, 1, 2, 2, 4], attention_resolutions=[32, 16, 8], num_groups=32,
                 num_heads=None, num_head_channels=64, dropout=0.0, use_fp16=True)


def _card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def _algorithmic_flops(net, x, t):
    L = _lib.lib()
    _lib.check(L.ivid_unet_profile_begin(net._handle))
    net(x, t)
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 20)
    _lib.check(L.ivid_unet_profile_end(net._handle, buf, len(buf)))
    prof = json.loads(buf.value.decode())
    return sum(v["flops"] for k, v in prof.items() if not k.startswith("_"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--widths", type=int, nargs="+", default=[96, 128, 160, 192])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_widths needs a CUDA device")
    card = _card()
    rows = []
    for mc in args.widths:
        cfg = dict(SMALL_128, model_channels=mc)
        net = backbones.AdmUnet2d(**cfg)
        net.load_state_dict(unet_ref.make_synthetic_state_dict(cfg, seed=0))
        net = net.cuda()
        g = torch.Generator().manual_seed(mc)
        x = torch.randn(args.batch, 4, 128, 128, generator=g).cuda()
        t = torch.randint(0, 1000, (args.batch,), generator=g).cuda()
        for _ in range(args.warmup):
            net(x, t)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(args.iters):
            net(x, t)
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / args.iters
        flops = _algorithmic_flops(net, x, t)
        widths = sorted({int(m * mc) for m in cfg["channel_mult"]})
        rows.append(dict(model_channels=mc, widths=widths, padded=any(w % 64 for w in widths), ms=round(ms, 3),
                         gflop=round(flops / 1e9, 1), tflops=round(flops / ms / 1e9, 1)))
        print(f"mc={mc}: {ms:.2f} ms/forward, {flops / ms / 1e9:.1f} TFLOP/s algorithmic", file=sys.stderr)
        del net
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=card, batch=args.batch, image=128, channel_mult=SMALL_128["channel_mult"], results=rows)))


if __name__ == "__main__":
    main()

"""CPU model of WHERE the CUDA plan rounds to fp16 (test infrastructure; runnable as a script for the attribution table).

The network is the oracle's (`oracle/unet_ref.py`, fp32 torch CPU) with a rounding injected at every place where
`ivid_b200/csrc/unet.cu` stores or feeds a 16-bit value; each place is a switch.  Two presets matter to the parity tests:

  PLAN        every rounding of the shipped CUDA plan: fp16 tensor-core operands (activations, weights, qkv, softmax
              probabilities, attention output), the fp16 hidden tensor of a ResBlock, the fp16 copies of block outputs that
              feed GroupNorm / the 1x1 skip conv; the network input and the output conv carry two-term (hi+lo) splits.
  TF32_CLASS  ONLY the GEMM / conv operands rounded to a 10-bit mantissa, everything else fp32: what the unmodified
              reference computes on the hardware it was tested on (README.md:15: A100) with the PyTorch it pins
              (environment.yml:10: 1.11.0, where torch.backends.cudnn.allow_tf32 and cuda.matmul.allow_tf32 both default
              to True), i.e. the deviation from strict fp32 that the reference's own GPU path has.  It is the floor of ANY
              implementation that feeds 10-bit-mantissa operands to tensor cores; the eps tests report it next to ours.

    python tests/precision_model.py [tiny|tiny_cond|tiny_sr|large|small]     # attribution of the eps error by source
"""
from __future__ import annotations

import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from oracle import unet_ref  # noqa: E402

SOURCES = ["x_in", "w_stem", "act", "w", "h16", "x16", "qkv16", "p16", "ao16", "w_out", "act_out"]
PLAN = dict(x_in="split", w_stem="split", act=1, w=1, h16=1, x16=1, qkv16=1, p16=1, ao16=1, w_out="split", act_out="split")
PLAN_R01 = dict(PLAN, x_in=1, w_stem=1, w_out=1, act_out=1)        # round-1 plan: no splits
TF32_CLASS = dict(x_in=1, w_stem=1, act=1, w=1, qkv16=1, ao16=1, w_out=1, act_out=1)


def r16(t, on=True):
    return t.half().float() if on else t


def split2(t):
    """hi + lo fp16 pair: what an operand carried as two fp16 tensors resolves to."""
    hi = t.half().float()
    return hi + (t - hi).half().float()


@torch.no_grad()
def forward(cfg, sd, x, times, classes, P):
    """unet_ref.unet_forward with the roundings selected by P (keys of SOURCES; value 1 = fp16, "split" = hi+lo pair)."""
    c = unet_ref._cfg_defaults(cfg)
    groups = c["num_groups"]
    head_ch = c["num_head_channels"]
    args = times[:, None] * sd["time_embed.0.freqs"][None, :]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    emb = F.linear(emb, sd["time_embed.1.weight"], sd["time_embed.1.bias"])
    emb = F.linear(F.silu(emb), sd["time_embed.3.weight"], sd["time_embed.3.bias"])
    if c["num_classes"] is not None and classes is not None:
        ce = sd["label_emb.weight"][classes * (classes >= 0).long()]
        if c["has_null_class"]:
            ce = ce * (classes >= 0).unsqueeze(1)
        emb = emb + ce

    def R(t, key):
        mode = P.get(key, False)
        return split2(t) if mode == "split" else r16(t, bool(mode))

    W = lambda name, key="w": R(sd[name], key)
    A = lambda t, key="act": R(t, key)

    def gn(t, p):
        return F.group_norm(t.float(), groups, sd[p + ".weight"], sd[p + ".bias"], 1e-5)

    def gn_from16(t, p):
        """GroupNorm whose statistics come from the fp32 tensor but whose values are read from its fp16 copy."""
        if not P.get("x16", False):
            return gn(t, p)
        N, C = t.shape[:2]
        tg = t.reshape(N, groups, -1)
        mean = tg.mean(-1, keepdim=True)
        var = tg.var(-1, unbiased=False, keepdim=True)
        y = ((r16(t).reshape(N, groups, -1) - mean) / torch.sqrt(var + 1e-5)).reshape(t.shape)
        shp = [1, C] + [1] * (t.dim() - 2)
        return y * sd[p + ".weight"].reshape(shp) + sd[p + ".bias"].reshape(shp)

    def resblock(x, p, mode):
        h = F.silu(gn_from16(x, p + ".in_layers.0") if mode == "same" else gn(x, p + ".in_layers.0"))
        if mode == "up":
            h = F.interpolate(h, scale_factor=2, mode="nearest"); x = F.interpolate(x, scale_factor=2, mode="nearest")
        elif mode == "down":
            h = F.avg_pool2d(h, 2); x = F.avg_pool2d(x, 2)
        h = F.conv2d(A(h), W(p + ".in_layers.2.weight"), sd[p + ".in_layers.2.bias"], padding=1)
        h = r16(h, bool(P.get("h16", False)))       # hidden tensor stored in fp16 (statistics of the rounded values)
        emb_out = F.linear(F.silu(emb), sd[p + ".emb_layers.1.weight"], sd[p + ".emb_layers.1.bias"])[:, :, None, None]
        scale, shift = torch.chunk(emb_out, 2, dim=1)
        h = gn(h, p + ".out_layers.0") * (1 + scale) + shift
        h = F.conv2d(A(F.silu(h)), W(p + ".out_layers.3.weight"), sd[p + ".out_layers.3.bias"], padding=1)
        if (p + ".skip_connection.weight") in sd:
            x = F.conv2d(A(x), W(p + ".skip_connection.weight"), sd[p + ".skip_connection.bias"])     # a GEMM: fp16 operand
        return x + h

    def attention(x, p, hc):
        b, ch, hh, ww = x.shape
        xf = x.reshape(b, ch, -1)
        qkv = F.conv1d(A(gn_from16(xf, p + ".norm")), W(p + ".qkv.weight"), sd[p + ".qkv.bias"])
        qkv = r16(qkv, bool(P.get("qkv16", False)))
        heads, T = ch // hc, xf.shape[-1]
        q, k, v = qkv.reshape(b * heads, hc * 3, T).split(hc, dim=1)
        w = torch.einsum("bct,bcs->bts", q, k) * (1 / math.sqrt(hc))
        e = torch.exp(w - w.max(dim=-1, keepdim=True).values)
        l = e.sum(-1, keepdim=True)
        e = r16(e, bool(P.get("p16", False)))
        o = r16(torch.einsum("bts,bcs->bct", e / l, v).reshape(b, -1, T), bool(P.get("ao16", False)))
        return (xf + F.conv1d(o, W(p + ".proj_out.weight"), sd[p + ".proj_out.bias"])).reshape(b, ch, hh, ww)

    blocks, _ = unet_ref._topology(cfg)
    hs = []
    h = x.float()
    for b in blocks:
        if b["group"] == "output":
            h = torch.cat([h, hs.pop()], dim=1)
        for l in b["layers"]:
            if l[0] == "conv":
                h = F.conv2d(A(h, "x_in"), W(l[1] + ".weight", "w_stem"), sd[l[1] + ".bias"], padding=1)
            elif l[0] == "res":
                h = resblock(h, l[1], l[4])
            else:
                h = attention(h, l[1], head_ch if head_ch != -1 else l[2] // c["num_heads"])
        if b["group"] == "input":
            hs.append(h)
    h = F.silu(gn_from16(h, "out.0"))
    return F.conv2d(A(h, "act_out"), W("out.2.weight", "w_out"), sd["out.2.bias"], padding=1)


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "tiny"
    g = {k: v for i in (0, 1) for k, v in np.load(os.path.join(ROOT, "tests", "golden", f"unet_sampler_golden_part{i}.npz")).items()}
    key = {"tiny": "tiny_cfg", "tiny_cond": "tiny_cond_cfg", "tiny_sr": "tiny_sr_cfg",
           "large": "schemacfg_rgbd_imagenet_adm_128_large_cfg", "small": "schemacfg_rgbd_singlecategory_adm_128_small"}[which]
    cfg = json.loads(bytes(g[key]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    S = cfg["image_size"]
    rng = np.random.default_rng(11)
    N = 2 if which.startswith("tiny") else 1
    x = torch.from_numpy(rng.standard_normal((N, cfg["in_channels"], S, S)).astype(np.float32))
    t = torch.tensor([999, 37][:N])
    cl = torch.tensor([3, -1][:N]) if cfg.get("num_classes") else None
    ref = unet_ref.unet_forward(cfg, sd, x, t, cl)
    rows = [("round-1 plan (no splits)", PLAN_R01), ("shipped plan", PLAN), ("TF32-class reference (GEMM operands only)", TF32_CLASS)]
    if which.startswith("tiny"):
        rows += [("only " + k, {k: 1}) for k in SOURCES]
    rows += [("shipped plan, hidden tensor fp32", dict(PLAN, h16=0)), ("shipped plan, GroupNorm reads fp32", dict(PLAN, x16=0)),
             ("shipped plan, both", dict(PLAN, h16=0, x16=0)), ("shipped plan, weights hi+lo everywhere (2x MMA)", dict(PLAN, w="split")),
             ("shipped plan, activations hi+lo everywhere (2x MMA)", dict(PLAN, act="split"))]
    for name, P in rows:
        print(f"{name:55s} {rel(forward(cfg, sd, x, t, cl, P), ref):.3e}")


if __name__ == "__main__":
    main()

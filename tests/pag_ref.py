"""Float64 model of perturbed-attention guidance (PAG; Ahn et al. 2024, arXiv:2403.17377).

The perturbed forward is oracle/unet_ref.unet_forward with the attention map of the selected layers replaced by the identity:
QKVAttention returns V, and the layer computes x + proj_out(V).  The oracle itself is not changed: `perturbed_forward`
swaps its attention function for the duration of one call, and the default path of every other caller stays as it is.

The mix: eps = G + w (eps_c - eps_p), G the eps of the step without PAG:
  cfg 1: (1+s) eps_c - s eps_u;  cfg 2: (1+s) eps_c;  cfg 0: eps_c.
`mix64` evaluates it in float64; `mix32` in fp32 with every operation rounded on its own, in the order of the step kernels'
mix_eps4 (G first, then sub, mul, add), which the native mix reproduces bit for bit."""
from __future__ import annotations

import contextlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle import unet_ref


def identity_attention(x, sd, p, groups, head_ch):
    """AttentionBlock.forward with the attention map replaced by the identity: the output of QKVAttention is V."""
    b, c, hh, ww = x.shape
    xf = x.reshape(b, c, -1)
    qkv = F.conv1d(unet_ref._group_norm(xf, sd, p + ".norm", groups), sd[p + ".qkv.weight"], sd[p + ".qkv.bias"])
    heads = c // head_ch
    T = xf.shape[-1]
    _, _, v = qkv.reshape(b * heads, head_ch * 3, T).split(head_ch, dim=1)
    h = F.conv1d(v.reshape(b, -1, T), sd[p + ".proj_out.weight"], sd[p + ".proj_out.bias"])
    return (xf + h).reshape(b, c, hh, ww)


@contextlib.contextmanager
def _perturbed(layers):
    orig = unet_ref._attention
    chosen = set(layers)

    def attention(x, sd, p, groups, head_ch):
        return (identity_attention if p in chosen else orig)(x, sd, p, groups, head_ch)

    unet_ref._attention = attention
    try:
        yield
    finally:
        unet_ref._attention = orig


def perturbed_forward(cfg, sd, x, times, classes=None, layers=("middle_block.1",), taps=None):
    """unet_ref.unet_forward with every layer in `layers` taking the identity attention map (all rows perturbed)."""
    with _perturbed(layers):
        return unet_ref.unet_forward(cfg, sd, x, times, classes, taps=taps)


def attention_layers(cfg):
    """Names of the attention layers in state-dict order (the index order of the C ABI)."""
    return [k[: -len(".qkv.weight")] for k in unet_ref.unet_param_shapes(cfg) if k.endswith(".qkv.weight")]


def mix64(ec, ep, w, cfg=0, s=0.0, eu=None):
    """G + w (eps_c - eps_p) in float64."""
    ec = np.asarray(ec, np.float64); ep = np.asarray(ep, np.float64)
    if cfg == 1:
        g = (1.0 + s) * ec - s * np.asarray(eu, np.float64)
    elif cfg == 2:
        g = (1.0 + s) * ec
    else:
        g = ec
    return g + w * (ec - ep)


def mix32(ec, ep, w, cfg=0, s=0.0, eu=None):
    """The same in fp32, one rounding per operation, in the order of the native step (numpy fp32 never contracts to FMA)."""
    f = np.float32
    ec = np.asarray(ec, f); ep = np.asarray(ep, f)
    s32, w32 = f(s), f(w)
    one_s = f(f(1.0) + s32)
    if cfg == 1:
        g = (one_s * ec).astype(f) - (s32 * np.asarray(eu, f)).astype(f)
    elif cfg == 2:
        g = (one_s * ec).astype(f)
    else:
        g = ec
    return (g.astype(f) + (w32 * (ec - ep).astype(f)).astype(f)).astype(f)


def torch_mix64(ec, ep, w, cfg=0, s=0.0, eu=None):
    """mix64 on torch tensors (float64 result)."""
    return torch.from_numpy(mix64(ec.double().cpu().numpy(), ep.double().cpu().numpy(), w, cfg, s,
                                  None if eu is None else eu.double().cpu().numpy()))

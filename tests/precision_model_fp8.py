"""CPU model of the fp8 mode's roundings (test infrastructure; AdmUnet2d.set_precision("fp8"), DESIGN.md §2).

`forward` is `precision_model.forward` under the shipped plan's roundings (`precision_model.PLAN`), except for the
ResBlock 3x3 convs that the fp8 packer takes:

  * the conv operand is rounded to e4m3 (clamped to +-448 first: the kernels saturate, torch's cast alone turns values
    beyond ~464 into NaN), straight from fp32 as `gn_apply` does;
  * the weights become e4m3(w * 2^e) * 2^-e, with the power-of-two scale of `fp8_exponent`;
  * the 1x1 skip weights of such a conv2 become fp16(w * 2^e) * 2^-e; their operand stays fp16.

A conv qualifies when its input width is a multiple of 16 and, for conv2, `fp8_skip_ok` holds for its skip weights.

The convs are told apart by their bias tensors, which `precision_model.forward` passes straight from the state dict:
while `forward` runs, F.conv2d / F.conv1d are wrapped to apply the roundings above to the convs so identified, and the
fp16 operand rounding (the plan's `act` switch, turned off here so that the e4m3 operands are rounded from fp32) to
the other convs that `act` covers: fp16 ResBlock convs, skip convs and the attention qkv GEMM.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

import precision_model as PM


def e4m3(t):
    """What the kernels store: satfinite e4m3, round to nearest even."""
    return t.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).float()


def fp8_exponent(w):
    """The packer's weight scale: e with max|w| * 2^e in (224, 448], 0 for an all-zero tensor."""
    m = float(w.abs().max())
    if m == 0.0:
        return 0
    f, k = math.frexp(m)
    return (9 if f <= 0.875 else 8) - k


def fp8_skip_ok(w_skip, e):
    """The packer keeps a conv fp16 when its scaled skip weights overflow fp16 or drop into its subnormals."""
    a = w_skip.abs().double()
    sa = a * 2.0 ** e
    return not bool((sa > 65504).any() or ((a >= 2.0 ** -14) & (sa < 2.0 ** -14)).any())


def _exponent_if_fp8(sd, p, kind):
    """e of the ResBlock conv `kind` ("conv1" / "conv2") of block p when it runs fp8, else None."""
    w = sd[p + (".in_layers.2.weight" if kind == "conv1" else ".out_layers.3.weight")]
    if w.shape[1] % 16 != 0:
        return None
    e = fp8_exponent(w)
    ws = sd.get(p + ".skip_connection.weight") if kind == "conv2" else None
    if ws is not None and not fp8_skip_ok(ws, e):
        return None
    return e


@torch.no_grad()
def forward(cfg, sd, x, times, classes):
    roles = {}
    for suffix, kind in ((".in_layers.2.bias", "conv1"), (".out_layers.3.bias", "conv2"), (".skip_connection.bias", "skip"),
                         (".qkv.bias", "qkv")):
        for k, v in sd.items():
            if k.endswith(suffix):
                roles[id(v)] = (kind, k[:-len(suffix)])
    conv2d, conv1d = F.conv2d, F.conv1d

    def conv2d_fp8(inp, weight, bias=None, *args, **kwargs):
        kind, p = roles.get(id(bias), (None, None)) if bias is not None else (None, None)
        if kind is None:
            return conv2d(inp, weight, bias, *args, **kwargs)
        e = _exponent_if_fp8(sd, p, "conv2" if kind == "skip" else kind)
        if e is not None and kind != "skip":
            name = p + (".in_layers.2.weight" if kind == "conv1" else ".out_layers.3.weight")
            return conv2d(e4m3(inp), e4m3(sd[name] * 2.0 ** e) * 2.0 ** -e, bias, *args, **kwargs)
        if e is not None:
            weight = (sd[p + ".skip_connection.weight"] * 2.0 ** e).half().float() * 2.0 ** -e
        return conv2d(PM.r16(inp), weight, bias, *args, **kwargs)

    def conv1d_fp8(inp, weight, bias=None, *args, **kwargs):
        if bias is not None and roles.get(id(bias), (None,))[0] == "qkv":
            inp = PM.r16(inp)
        return conv1d(inp, weight, bias, *args, **kwargs)

    F.conv2d, F.conv1d = conv2d_fp8, conv1d_fp8
    try:
        return PM.forward(cfg, sd, x, times, classes, dict(PM.PLAN, act=0))
    finally:
        F.conv2d, F.conv1d = conv2d, conv1d

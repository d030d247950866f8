"""float64 references and error bounds for the two ends of the network and the embedding path (test infrastructure, CPU).

The stem and the output head carry two-term fp16 splits (DESIGN.md §2): the stem's operand channels are x_hi | x_lo | x_hi
against weight columns Wh | Wh | Wl (`pack_input_kernel`, `cond_pack_kernel`, `pack_stem_rows`), and the head's 1x1 GEMM
reads a_hi | a_lo | a_hi against Wh | Wh | Wl (`pack_out_rows`) into 9 * Co tap columns that `eps_gather_kernel` adds.
Both are checked per element against float64 with the bounds below; `split_products` emulates the split, with switches
that drop one of its terms, so that tests/test_network_ends_model.py can show the bounds see each term.

The embedding path (`posenc_kernel`, the three `linear_*_kernel`s, `silu_transpose_kernel`, `film_table_kernel`) is fp32
on CUDA cores.  Each fp32 Linear adds at most (K + 2) 2^-24 (|W||x| + |b| + |label row|) and carries its input error
through |W|.  `linear_kernel` / `embedding_kernels` mirror the launch rule of `launch_linear` / `launch_film_table`
(csrc/ops.cu)."""
from __future__ import annotations

import json
import math
import os

import numpy as np

import torch
import torch.nn.functional as F

from oracle import unet_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U23, U24 = 2.0 ** -23, 2.0 ** -24
SPLIT_RESIDUE = 2.0 ** -20      # |x - hi - lo| <= 2^-22 |x|, the same for W, and the dropped lo * Wl <= 2^-24 |x w|
SUB16 = 2.0 ** -25              # half the fp16 subnormal spacing: the absolute error of a lo term that is subnormal
TRANSCENDENTAL = 2.0 ** -22     # cosf / sinf of |a| <= 1000 and expf, absolute on values of magnitude <= 1
STEM_COLUMNS = 64               # the stem's packed operand channels per tap
MODES = ("split", "no_lo", "no_wl", "none")


# ----------------------------------------------------------------------------------------------------------------------
# the two-term split
# ----------------------------------------------------------------------------------------------------------------------
def hi_lo(t):
    """(hi, lo) fp16 terms of t as float64: hi = fp16(t), lo = fp16(t - hi) (split2 of tests/precision_model.py)."""
    t = t.float()
    hi = t.half().float()
    return hi.double(), (t - hi).half().double()


def split_products(x, w, mode="split", conv=None):
    """float64 sum of the products the split forms: conv(x, w) over (x_hi, Wh) + (x_lo, Wh) + (x_hi, Wl).  Modes drop a
    term: "no_lo" the operand's lo, "no_wl" the weight's lo, "none" both (plain fp16 operands)."""
    conv = conv or (lambda a, b: F.conv2d(a, b, padding=1))
    xh, xl = hi_lo(x)
    wh, wl = hi_lo(w)
    y = conv(xh, wh)
    if mode in ("split", "no_wl"):
        y = y + conv(xl, wh)
    if mode in ("split", "no_lo"):
        y = y + conv(xh, wl)
    return y


def off_grid(t, frac=0.45):
    """|t| moved onto an fp16 value with mantissa in [1, 1.0625), then 0.45 fp16 ulp above it: the value's lo term is
    0.45 ulp of hi and positive everywhere, so a dropped lo shifts every product the same way."""
    a = t.abs().double().clamp_min(2.0 ** -8)
    e = torch.floor(torch.log2(a))
    m = 1.0 + torch.frac(a / 2.0 ** e * 16.0) / 16.0           # mantissa in [1, 1.0625)
    hi = (m * 2.0 ** e).float().half().double()
    ulp = 2.0 ** (torch.floor(torch.log2(hi)) - 10)
    return (hi + frac * ulp).float()


def golden_cfgs():
    """The network configurations the tests use, from the golden files' cfg JSON.  "g4_40" is g4_20 (num_groups=4,
    model_channels=20) with channel_mult [2, 3.2]: g4_20 itself has widths that are not multiples of 8 and is refused, and
    this is the narrowest runnable network whose embedding width 4 * 20 = 80 is not a multiple of 32."""
    g = {}
    for f in ("unet_sampler_golden_part0", "unet_sampler_golden_part1", "heads_golden", "widths_golden"):
        g.update(np.load(os.path.join(ROOT, "tests", "golden", f + ".npz")))
    cfg = lambda k: json.loads(bytes(g[k]).decode())
    out = {"tiny": cfg("tiny_cfg"), "tiny_cond": cfg("tiny_cond_cfg"), "tiny_sr": cfg("tiny_sr_cfg"),
           "large": cfg("schemacfg_rgbd_imagenet_adm_128_large_cfg"), "single": cfg("single_cfg"), "g8": cfg("g8_cfg"),
           "mc96": cfg("mc96_cfg"), "g4_20": cfg("g4_20_cfg")}
    out["g4_40"] = dict(out["g4_20"], channel_mult=[2, 3.2])
    return out


def coherent_state_dict(cfg, seed=1234):
    """Synthetic weights with the two split GEMMs made coherent: all-positive stem and out.2 weights just off the fp16
    grid (`off_grid`), and out.0's bias raised by 2 so that the head's activation y = SiLU(GN) is mostly positive."""
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=seed)
    for k in ("input_blocks.0.0.weight", "out.2.weight"):
        sd[k] = off_grid(sd[k])
    sd["out.0.bias"] = sd["out.0.bias"] + 2.0
    return sd


def stem_input(N, C, H, W, seed):
    """A positive network input just off the fp16 grid."""
    return off_grid(torch.randn(N, C, H, W, generator=torch.Generator().manual_seed(seed)))


# ----------------------------------------------------------------------------------------------------------------------
# stem
# ----------------------------------------------------------------------------------------------------------------------
def stem_reference(x, w, b):
    """float64 conv3x3 of the fp32 network input x [N, Cin, H, W] (or the assembled conditional input) with the fp32 stem
    weights, plus the bias, and S = sum |x w| per output element."""
    x64, w64 = x.double(), w.double()
    ref = F.conv2d(x64, w64, b.double(), padding=1)
    S = F.conv2d(x64.abs(), w64.abs(), padding=1)
    return ref, S


def stem_bound(S, w, b, delta_in=None):
    """Split residue 2^-20 S, fp32 accumulation of the K = 9 * 64 packed columns and the bias (K + 1) 2^-23 (S + |b|),
    fp16-subnormal lo terms, and for conditional stems sum |w| delta_in, delta_in the assembly's fp32 rounding per input
    element (`cond_delta`)."""
    K = 9 * STEM_COLUMNS
    w64 = w.double().abs()
    bnd = SPLIT_RESIDUE * S + (K + 1) * U23 * (S + b.double().abs()[None, :, None, None])
    ones = torch.ones_like(S[:, :1])
    bnd = bnd + SUB16 * F.conv2d(ones.expand(-1, w.shape[1], -1, -1), w64, padding=1)
    if delta_in is not None:
        bnd = bnd + F.conv2d(delta_in.double(), w64, padding=1)
    return bnd


def cond_delta(kind, x, y, mask=None, mask_rgb=None, noise=None):
    """Per input element, how far the kernel's fp32 assembly of the conditional input may be from the oracle's fp32 torch
    assembly.  Inpaint: a filled value y m + z (1 - m) is three fp32 roundings ((1 - m), two products, the sum) in each,
    so 3 2^-23 (|y m| + |z (1 - m)|) (the kernel may contract to FMA where torch does not).  Super-resolution: 4 fp32 ulp of
    max |y| on each bilinear tap (source index, weights and the two-level lerp).  x and the mask channels are copied."""
    N, _, H, W = x.shape
    if kind == "sr":
        d = torch.zeros(N, 8, H, W, dtype=torch.float64)
        d[:, 4:] = 4 * U23 * float(y.abs().max())
        return d
    mr = mask_rgb if mask_rgb is not None else mask
    fill = lambda yc, m, z: 3 * U23 * ((yc * m).abs() + (z * (1 - m)).abs()).double()
    parts = [torch.zeros(N, 4, H, W, dtype=torch.float64)]
    if mask_rgb is not None:
        parts.append(torch.zeros(N, 1, H, W, dtype=torch.float64))
    parts += [fill(y[:, :3], mr, noise[:, :3]), fill(y[:, 3:], mask, noise[:, 3:]), torch.zeros(N, 1, H, W, dtype=torch.float64)]
    return torch.cat(parts, 1)


# ----------------------------------------------------------------------------------------------------------------------
# output head
# ----------------------------------------------------------------------------------------------------------------------
GAMMA12 = 12 * U24     # relative error of a fused GroupNorm statistic (tests/test_gpu_fused_epilogue.py)


def head_reference(h, sd, groups):
    """The head of a forward whose last output block returned h [N, C, H, W] (fp32).  GroupNorm statistics from the fp32
    values, normalised values from their fp16 copy (what `unet.cu` does: the out.0 apply reads the block's fp16 copy), then
    y = SiLU(GN) and eps = conv3x3(y, W) + b, all float64.  Returns eps, y (NCHW) and dy, the per-element bound on the
    kernel's y before its own output rounding: the apply slack of tests/test_gpu_fused_epilogue.py plus the error of fused
    statistics (as test_in_block_chain_at_dc_offset derives it)."""
    import test_gpu_fused_epilogue as FE
    x32 = h.permute(0, 2, 3, 1).contiguous()
    x16 = x32.half()
    v = x32.double()
    N, H, W, C = v.shape
    stats = torch.stack([v.sum((1, 2)), (v * v).sum((1, 2))], -1)
    y, A, Bm, mean, rstd = FE._gn_ref(x16, groups, sd["out.0.weight"], sd["out.0.bias"], None, 0, False, True, stats=stats)
    vg = v.reshape(N, H * W, groups, -1)
    n = vg.shape[1] * vg.shape[3]
    abs_mean, sq_mean = vg.abs().sum((1, 3)) / n, (vg * vg).sum((1, 3)) / n
    var = (sq_mean - mean * mean).clamp_min(1e-30)
    dmean = GAMMA12 * abs_mean
    drstd = GAMMA12 * (sq_mean + 2 * mean.abs() * abs_mean) / (2 * var) + GAMMA12
    cpg = C // groups
    dm_c, dr_c, m_c = (t.repeat_interleave(cpg, 1)[:, None, None, :] for t in (dmean, drstd, mean))
    x16d = x16.double()
    widen = (dm_c + (x16d - m_c).abs() * dr_c) * A.abs()[:, None, None, :]
    dy = FE._slack(x16, A, Bm, True) + 1.1 * widen
    to_nchw = lambda t: t.permute(0, 3, 1, 2)
    y, dy = to_nchw(y), to_nchw(dy)
    eps = F.conv2d(y, sd["out.2.weight"].double(), sd["out.2.bias"].double(), padding=1)
    return eps, y, dy


def conv_pad_k(C):
    """Packed K columns of a conv segment of C channels (csrc/ops.cu conv_pad_k): whole 64-channel chunks."""
    return -(-C // 64) * 64


def head_bound(y, dy, w, b, split=True):
    """Split head (9 * Co <= 64): sum |w| (dy + 2^-25) for the apply and its lo term, the split residue 2^-20 on
    S = sum |y w| and 2^-25 sum |y| for subnormal weight lo terms, the GEMM over 3 Cp columns, the 9-tap fp32 add and the
    bias: (3 Cp + 10) 2^-23 (S + |b|).  Unsplit head (`conv_gemm<16>` NCHW over fp16 y and W): the fp16 rounding of y
    (2^-11 |y| + 2^-25) and of W (2^-11 |w| + 2^-25) and the fp32 accumulation over K = 9 Cp columns."""
    C = y.shape[1]
    Cp = conv_pad_k(C)
    wa = w.double().abs()
    S = F.conv2d(y.abs(), wa, padding=1)
    ya1 = F.conv2d(y.abs(), torch.ones_like(wa), padding=1)
    bb = b.double().abs()[None, :, None, None]
    if split:
        return F.conv2d(dy + SUB16, wa, padding=1) + SPLIT_RESIDUE * S + SUB16 * ya1 + (3 * Cp + 10) * U23 * (S + bb)
    return (F.conv2d(dy + 2.0 ** -11 * y.abs() + SUB16, wa, padding=1) + 2.0 ** -11 * S + SUB16 * ya1
            + (9 * Cp + 1) * U23 * (S + bb))


# ----------------------------------------------------------------------------------------------------------------------
# embedding path
# ----------------------------------------------------------------------------------------------------------------------
def _linear_bound(W, x, dx, b, extra=None):
    """(K + 2) 2^-24 (|W||x| + |b| + |extra|) for one fp32 Linear (K FMAs, the bias, the label row), plus its input error
    carried through |W|."""
    K = W.shape[1]
    Wa = W.double().abs()
    mag = x.abs() @ Wa.T + b.double().abs()
    if extra is not None:
        mag = mag + extra.abs()
    return (K + 2) * U24 * mag + dx @ Wa.T


def _silu64(v):
    return v / (1 + torch.exp(-v))


def embedding_reference(cfg, sd, t, classes):
    """emb [N, 4 mc] in float64 and its bound.  a = fp32(t * freq) exactly as torch forms it, cos / sin in float64, then
    Linear -> SiLU -> Linear -> + label row (the null class -1 and classes=None add 0)."""
    a = t[:, None] * sd["time_embed.0.freqs"][None, :]          # fp32, the product the kernel rounds too
    a = a.double()
    e0 = torch.cat([torch.cos(a), torch.sin(a)], -1)
    d0 = torch.full_like(e0, TRANSCENDENTAL)
    W1, b1, W2, b2 = (sd[k] for k in ("time_embed.1.weight", "time_embed.1.bias", "time_embed.3.weight", "time_embed.3.bias"))
    e1 = e0 @ W1.double().T + b1.double()
    d1 = _linear_bound(W1, e0, d0, b1)
    s = _silu64(e1)
    ds = 1.1 * d1 + 2.0 ** -21 * s.abs()                         # SiLU slope <= 1.1; v / (1 + expf(-v)) in fp32
    emb = s @ W2.double().T + b2.double()
    lab = torch.zeros_like(emb)
    if classes is not None:
        real = classes >= 0
        lab[real] = sd["label_emb.weight"][classes[real]].double()
    emb = emb + lab
    return emb, _linear_bound(W2, s, ds, b2, extra=lab)


def film_weights(cfg, sd):
    """The stacked emb_layers.1 weights and biases of every ResBlock, in creation order (the FiLM table's columns)."""
    blocks, _ = unet_ref._topology(cfg)
    names = [l[1] for b in blocks for l in b["layers"] if l[0] == "res"]
    W = torch.cat([sd[p + ".emb_layers.1.weight"] for p in names], 0)
    b = torch.cat([sd[p + ".emb_layers.1.bias"] for p in names], 0)
    return W, b


def film_reference(cfg, sd, emb_tap):
    """float64 W_f silu(emb) + b_f from the kernel's own emb tap [N, E] (fp32), and its bound."""
    W, b = film_weights(cfg, sd)
    s = _silu64(emb_tap.double())
    return s @ W.double().T + b.double(), _linear_bound(W, s, 2.0 ** -21 * s.abs(), b)


# ----------------------------------------------------------------------------------------------------------------------
# launch rule mirror (csrc/ops.cu launch_linear / launch_film_table, csrc/unet.cu embeddings)
# ----------------------------------------------------------------------------------------------------------------------
def linear_kernel(K, O):
    if K in (256, 512, 1024) and O <= 8192:
        return f"linear_warp_kernel<{K // 128}>"
    if K % 32 == 0:
        return "linear_tiled_kernel<4>" if O >= 128 * 64 else "linear_tiled_kernel<2>"
    return "linear_rows_kernel"


def film_total(cfg):
    return sum(s[0] for k, s in unet_ref.unet_param_shapes(cfg).items() if k.endswith(".emb_layers.1.weight"))


def embedding_kernels(cfg):
    """Which kernel each embedding stage of a network runs: {"time_embed.1", "time_embed.3", "film"} -> kernel name; the
    film table's name carries ", partial tile" when its width is not a multiple of its 128-column tile."""
    mc = cfg["model_channels"]
    E, FT = 4 * mc, film_total(cfg)
    film = "film_table_kernel" + (", partial tile" if FT % 128 else ", full tiles") if E % 32 == 0 else linear_kernel(E, FT)
    return {"time_embed.1": linear_kernel(mc, E), "time_embed.3": linear_kernel(E, E), "film": film}


def worst(got, ref, bound):
    """max |got - ref| / bound (a non-finite output counts as infinitely far) and the index of that element."""
    r = (got.double() - ref).abs() / bound
    r = torch.where(torch.isfinite(got.double()), r, torch.full_like(r, math.inf))
    i = int(torch.argmax(r))
    return float(r.reshape(-1)[i]), tuple(int(v) for v in torch.unravel_index(torch.tensor(i), r.shape))

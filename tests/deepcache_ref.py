"""Test infrastructure: the reference UNet forward (oracle/unet_ref.py) with feature reuse between denoising steps
(DeepCache, Ma, Fang, Wang, CVPR 2024, arXiv:2312.00858), in fp32 on the CPU.

L is the number of output blocks; output block L-1-j reads input block j's output as its skip tensor.  A reuse forward at
branch b runs the embeddings, input blocks 0..b, output blocks L-1-b..L-1 and the head, and takes the output of output
block L-2-b (the middle block when L-2-b < 0) from a tensor cached by an earlier full forward.  Built on the oracle's own
layer functions, which it leaves unchanged.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from oracle import unet_ref as U


def _embedding(c, sd, times, classes):
    # unet_ref.unet_forward's embedding, unchanged (adm.py:545-555)
    args = times[:, None] * sd["time_embed.0.freqs"][None, :]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    emb = F.linear(emb, sd["time_embed.1.weight"], sd["time_embed.1.bias"])
    emb = F.linear(F.silu(emb), sd["time_embed.3.weight"], sd["time_embed.3.bias"])
    if c["num_classes"] is not None and classes is not None:
        ce = sd["label_emb.weight"][classes * (classes >= 0).long()]
        if c["has_null_class"]:
            ce = ce * (classes >= 0).unsqueeze(1)
        emb = emb + ce
    return emb


def _layer(c, sd, l, h, emb):
    groups = c["num_groups"]
    if l[0] == "conv":
        return F.conv2d(h, sd[l[1] + ".weight"], sd[l[1] + ".bias"], padding=1)
    if l[0] == "res":
        return U._resblock(h, emb, sd, l[1], l[4], groups)
    if l[0] == "down":
        return (F.conv2d(h, sd[l[1] + ".op.weight"], sd[l[1] + ".op.bias"], stride=2, padding=1) if c["conv_resample"]
                else F.avg_pool2d(h, 2))
    if l[0] == "up":
        h = F.interpolate(h, scale_factor=2, mode="nearest")
        return F.conv2d(h, sd[l[1] + ".conv.weight"], sd[l[1] + ".conv.bias"], padding=1) if c["conv_resample"] else h
    hc = c["num_head_channels"] if c["num_head_channels"] != -1 else l[2] // c["num_heads"]
    return U._attention(h, sd, l[1], groups, hc)


def cached_block_name(cfg: dict, branch: int) -> str:
    """The block whose output a reuse forward at `branch` reads: output block L-2-b, or the middle block."""
    blocks, _ = U._topology(cfg)
    L = sum(b["group"] == "output" for b in blocks)
    return f"output_blocks.{L - 2 - branch}" if L - 2 - branch >= 0 else "middle_block"


@torch.no_grad()
def unet_forward(cfg: dict, sd: Dict[str, torch.Tensor], x: torch.Tensor, times: torch.Tensor,
                 classes: Optional[torch.Tensor] = None, capture: Optional[str] = None,
                 reuse: Optional[Tuple[int, torch.Tensor]] = None):
    """unet_ref.unet_forward, plus:
      capture = a block prefix ("output_blocks.13", "middle_block"): returns (eps, that block's output);
      reuse = (b, h): the reuse forward at branch b, with h as the output of cached_block_name(cfg, b).
    Without either it computes what unet_ref.unet_forward computes."""
    c = U._cfg_defaults(cfg)
    assert classes is None or c["num_classes"] is not None, "this model is not class-conditioned"
    emb = _embedding(c, sd, times, classes)
    blocks, _ = U._topology(cfg)
    n_in = sum(b["group"] == "input" for b in blocks)
    L = sum(b["group"] == "output" for b in blocks)
    if reuse is not None:
        branch, cached = reuse
        assert 0 <= branch <= c["num_res_blocks"], f"cache_branch must be in [0, {c['num_res_blocks']}]"
        keep = set(range(branch + 1)) | set(range(n_in + 1 + L - 1 - branch, n_in + 1 + L))
    captured = None
    hs = []
    h = x.float()
    for bi, b in enumerate(blocks):
        if reuse is not None and bi not in keep:
            if bi == n_in + L - 1 - branch:          # the block before output block L-1-b: its output is the cached tensor
                h = cached.float()
            continue
        if b["group"] == "output":
            h = torch.cat([h, hs.pop()], dim=1)
        for l in b["layers"]:
            h = _layer(c, sd, l, h, emb)
        if b["group"] == "input":
            hs.append(h)
        if b["prefix"] == capture:
            captured = h
    h = F.silu(U._group_norm(h, sd, "out.0", c["num_groups"]))
    eps = F.conv2d(h, sd["out.2.weight"], sd["out.2.bias"], padding=1)
    if capture is not None:
        assert captured is not None, f"no block {capture!r} ran"
        return eps, captured
    return eps

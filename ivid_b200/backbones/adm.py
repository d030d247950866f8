"""AdmUnet2d — host-side mirror of the reference backbone class (diffusion/backbones/adm.py:289-566).

Same constructor kwargs, same state-dict keys/shapes (enumerated from the native topology builder, so there is a single
source of truth), same `.forward(x, times, classes)` contract — but the forward runs the hand-written sm_90a kernels
behind the C ABI (include/ivid_b200.h) instead of ~625 ATen/cuDNN launches.  There is no CPU path: calling forward
without a CUDA device raises.
"""
from __future__ import annotations

import ctypes
import json
import math
from typing import Optional

import torch
import torch.nn as nn

from .. import _lib

__all__ = ["AdmUnet2d", "PAG_DEFAULT_LAYERS"]

# perturbed-attention guidance: every ADM network has an attention layer in its middle block (not a claim that it is best)
PAG_DEFAULT_LAYERS = ("middle_block.1",)


class _Params(nn.Module):
    """Plain container; children/parameters are attached under the reference's dotted names."""


def _attach(root: nn.Module, dotted: str, tensor: torch.Tensor, is_buffer: bool) -> None:
    parts = dotted.split(".")
    mod = root
    for p in parts[:-1]:
        if p not in mod._modules:
            mod.add_module(p, _Params())
        mod = mod._modules[p]
    if is_buffer:
        mod.register_buffer(parts[-1], tensor)
    else:
        mod.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=False))


class AdmUnet2d(nn.Module):
    """The full UNet model with attention and timestep embedding (reference adm.py:289).

    Args are those of the reference constructor (adm.py:318-337).
    """

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, num_classes=None, has_null_class=False,
                 use_fp16=False, num_groups=32, num_heads=1, num_head_channels=-1, use_scale_shift_norm=True,
                 resblock_updown=True):
        super().__init__()
        self.image_size = image_size
        self.in_channels = in_channels
        self.model_channels = model_channels
        self.out_channels = out_channels
        self.num_res_blocks = num_res_blocks
        self.attention_resolutions = attention_resolutions
        self.dropout = dropout
        self.channel_mult = channel_mult
        self.conv_resample = conv_resample
        self.num_classes = num_classes
        self.has_null_class = has_null_class if num_classes is not None else False
        # Reference: torso dtype fp16 when use_fp16 (adm.py:351).  Here the tensor-core operands are always fp16 with
        # fp32 accumulation, fp32 residual stream, fp32 GroupNorm / softmax / embeddings (DESIGN.md "precision").
        self.dtype = torch.float16 if use_fp16 else torch.float32
        self.num_groups = num_groups
        self.num_heads = num_heads
        self.num_head_channels = num_head_channels

        cfg = dict(image_size=image_size, in_channels=in_channels, model_channels=model_channels,
                   out_channels=out_channels, num_res_blocks=num_res_blocks,
                   attention_resolutions=list(attention_resolutions), dropout=dropout, channel_mult=list(channel_mult),
                   conv_resample=conv_resample, num_classes=num_classes, has_null_class=has_null_class,
                   use_fp16=use_fp16, num_groups=num_groups, num_heads=num_heads, num_head_channels=num_head_channels,
                   use_scale_shift_norm=use_scale_shift_norm, resblock_updown=resblock_updown)
        self._cfg_json = json.dumps(cfg)
        L = _lib.lib()
        self._handle = ctypes.c_void_p()
        _lib.check(L.ivid_unet_create(self._cfg_json.encode(), ctypes.byref(self._handle)))
        self._packed_device = None     # device index the native arena currently lives on
        self._packed_version = None
        self.precision = "fp16"

        # Parameters / buffers with the reference's names, shapes and default initialisation
        # (nn.Conv/Linear defaults, zero_module for out_layers.3 / proj_out / out.2: adm.py:182,278,486).
        n = ctypes.c_int()
        _lib.check(L.ivid_unet_num_params(self._handle, ctypes.byref(n)))
        name = ctypes.c_char_p()
        shape = (ctypes.c_int64 * 4)()
        ndim = ctypes.c_int()
        isbuf = ctypes.c_int()
        self._schema = []
        for i in range(n.value):
            _lib.check(L.ivid_unet_param_info(self._handle, i, ctypes.byref(name), shape, ctypes.byref(ndim), ctypes.byref(isbuf)))
            key = name.value.decode()
            shp = tuple(int(shape[j]) for j in range(ndim.value))
            self._schema.append((key, shp, bool(isbuf.value)))
            _attach(self, key, self._default_init(key, shp), bool(isbuf.value))

    # ------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _default_init(key: str, shape) -> torch.Tensor:
        if key == "time_embed.0.freqs":
            half = shape[0]
            return torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
        if key == "label_emb.weight":
            return torch.randn(shape)
        zeroed = key.endswith(("out_layers.3.weight", "out_layers.3.bias", "proj_out.weight", "proj_out.bias")) or key.startswith("out.2.")
        if zeroed:
            return torch.zeros(shape)
        is_norm = any(s in key for s in (".in_layers.0.", ".out_layers.0.", ".norm.", "out.0."))
        if is_norm:
            return torch.ones(shape) if key.endswith("weight") else torch.zeros(shape)
        if len(shape) >= 2:                      # nn.Conv / nn.Linear default: kaiming_uniform(a=sqrt(5))
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            bound = 1.0 / math.sqrt(fan_in)
            return torch.empty(shape).uniform_(-bound, bound)
        # bias of conv / linear: U(-1/sqrt(fan_in), 1/sqrt(fan_in)); fan_in unknown here -> small uniform
        return torch.empty(shape).uniform_(-0.02, 0.02)

    @property
    def device(self):
        return next(self.parameters()).device

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                _lib.lib().ivid_unet_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------------------------
    def _version(self):
        return tuple(p._version for p in self.parameters()) + tuple(id(p) for p in self.parameters())

    def _apply(self, fn, *a, **k):   # .cuda() / .to() invalidate the packed arena
        r = super()._apply(fn, *a, **k)
        self._packed_device = None
        return r

    def load_state_dict(self, state_dict, strict=True, **kw):
        r = super().load_state_dict(state_dict, strict=strict, **kw)
        self._packed_device = None
        return r

    def repack(self) -> None:
        """Pack the current parameters into the native device arena (fp16 K-major conv/GEMM operands etc.)."""
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("ivid_b200.AdmUnet2d runs on CUDA (sm_90a) only: call .cuda() first — there is no CPU path")
        L = _lib.lib()
        sd = self.state_dict()
        for key, shp, _ in self._schema:
            t = sd[key].detach().to("cpu", torch.float32).contiguous()
            assert tuple(t.shape) == shp, f"size mismatch for {key}"
            s = (ctypes.c_int64 * max(len(shp), 1))(*shp)
            _lib.check(L.ivid_unet_set_param(self._handle, key.encode(), _lib.ptr(t), s, len(shp)))
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        _lib.check(L.ivid_unet_finalize(self._handle, idx))
        self._packed_device = idx
        self._packed_version = self._version()

    def set_precision(self, precision: str) -> None:
        """Operands of the ResBlock 3x3 convs: "fp16" (default) or "fp8" (e4m3 activations, power-of-two-scaled e4m3
        weights, fp32 accumulation; DESIGN.md §2).  fp8 changes the numbers.  The weights are repacked at the next use."""
        if precision not in ("fp16", "fp8"):
            raise ValueError(f"precision must be 'fp16' or 'fp8', got {precision!r}")
        _lib.check(_lib.lib().ivid_unet_set_precision(self._handle, 0 if precision == "fp16" else 1))
        self.precision = precision
        self._packed_device = None

    def _ensure_packed(self):
        if self._packed_device is None or self._packed_version != self._version():
            self.repack()

    def weight_arena(self):
        """(device pointer, bytes) of the packed weights — what a rank-0 loader broadcasts with NCCL at init."""
        self._ensure_packed()
        p = ctypes.c_void_p()
        n = ctypes.c_uint64()
        _lib.check(_lib.lib().ivid_unet_weight_arena(self._handle, ctypes.byref(p), ctypes.byref(n)))
        return p.value, n.value

    # ------------------------------------------------------------------------------------------------------------
    @property
    def attention_layers(self):
        """Names of the attention layers ("input_blocks.7.1", "middle_block.1", ...) in state-dict order; the position of a
        name is the layer index of the C ABI's perturbed-attention entry points."""
        return [k[: -len(".qkv.weight")] for k, _, _ in self._schema if k.endswith(".qkv.weight")]

    def pag_layer_indices(self, layers):
        """Indices of the named attention layers (AssertionError for an empty selection, an unknown or a repeated name)."""
        assert not isinstance(layers, str), f"pag_layers must be a sequence of layer names, got the string {layers!r}"
        layers = list(layers)
        assert layers, "pag_layers must name at least one attention layer"
        names = self.attention_layers
        for name in layers:
            assert name in names, f"{name!r} is not an attention layer of this network (attention layers: {names})"
        assert len(set(layers)) == len(layers), f"pag_layers lists a layer twice: {layers}"
        return [names.index(name) for name in layers]

    def _check_input(self, x, classes):
        """The input assertions of forward() and forward_perturbed() (adm.py:540-549)."""
        assert classes is None or self.num_classes is not None, "this model is not class-conditioned"
        if classes is not None:
            assert bool(torch.all(classes >= 0)) or self.has_null_class, "this model does not have a null class"
            assert classes.shape == (x.shape[0],), "classes must be a 1-D batch of labels"
        assert x.dim() == 4 and x.shape[1] == self.in_channels, \
            f"expected input [N,{self.in_channels},H,W], got {tuple(x.shape)}"

    @torch.no_grad()
    def forward_perturbed(self, x, times, classes=None, layers=PAG_DEFAULT_LAYERS):
        """forward() with the attention map of every layer in `layers` replaced by the identity (perturbed-attention
        guidance, Ahn et al. 2024, arXiv:2403.17377): each such layer computes x + proj_out(V), V the value channels of its
        qkv projection.  Every row of the batch is perturbed.  Same arguments and return as forward()."""
        idx = self.pag_layer_indices(layers)
        self._check_input(x, classes)
        self._ensure_packed()
        N, _, H, W = x.shape
        xx = x.to(torch.float32).contiguous()
        tt = times.to(device=x.device, dtype=torch.int64).contiguous()
        cc = classes.to(device=x.device, dtype=torch.int64).contiguous() if classes is not None else None
        out = torch.empty((N, self.out_channels, H, W), dtype=torch.float32, device=x.device)
        arr = (ctypes.c_int * len(idx))(*idx)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().ivid_unet_forward_perturbed(self._handle, _lib.ptr(xx), N, H, W, None, _lib.ptr(tt), _lib.ptr(cc),
                                                              _lib.ptr(out), N, 0, arr, len(idx), -1, _lib.cur_stream(x.device)))
        return out.type(x.dtype)

    @torch.no_grad()
    def forward(self, x, times, classes=None):
        """Apply the model to an input batch (reference adm.py:526-566).

        x: [N, C, H, W] fp32 cuda; times: [N] long; classes: [N] long (-1 = null class) or None.  Returns eps [N, out, H, W].
        H and W need not equal image_size (which only places the attention blocks): like the reference, any size divisible
        by 2^(len(channel_mult) - 1) runs, and other sizes raise RuntimeError.
        """
        self._check_input(x, classes)
        self._ensure_packed()
        N, _, H, W = x.shape
        xx = x.to(torch.float32).contiguous()
        tt = times.to(device=x.device, dtype=torch.int64).contiguous()
        cc = classes.to(device=x.device, dtype=torch.int64).contiguous() if classes is not None else None
        out = torch.empty((N, self.out_channels, H, W), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().ivid_unet_forward_hw(self._handle, _lib.ptr(xx), N, H, W, None, _lib.ptr(tt), _lib.ptr(cc),
                                                       _lib.ptr(out), N, _lib.cur_stream(x.device)))
        return out.type(x.dtype)

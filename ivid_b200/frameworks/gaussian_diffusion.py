"""Diffusion frameworks — host-side mirrors of the reference classes (same names, ctor kwargs, attributes):

    GaussianDiffusion        diffusion/frameworks/gaussian_diffusion.py:12-116
    ClassifierFreeGuidance   diffusion/frameworks/classifier_free_guidance.py:12-75
    InpaintCFG               diffusion/frameworks/inpaint_cfg.py:11-128
    SuperResCFG              diffusion/frameworks/sr_cfg.py:11-96

`model_inference` keeps the reference semantics but evaluates both classifier-free-guidance halves in ONE batch-2N
native forward (SURVEY.md K12).  Training losses are out of scope of the sampling hot path (SURVEY.md §8).
"""
from __future__ import annotations

import ctypes
import inspect
import math
import numbers

import numpy as np
import torch
import torch.nn.functional as F

from .. import _lib
from ..utils import edict
from .utils import get_betas_by_name

__all__ = ["GaussianDiffusion", "ClassifierFreeGuidance", "InpaintCFG", "SuperResCFG"]


def _extract(arr, timesteps, broadcast_shape):
    # reference frameworks/utils.py:63-80
    res = torch.from_numpy(arr).to(device=timesteps.device)[timesteps].float()
    while len(res.shape) < len(broadcast_shape):
        res = res[..., None]
    return res.expand(broadcast_shape)


def _unwrap(backbone):
    return backbone.module if hasattr(backbone, "module") else backbone


def check_pag(pag_scale, pag_layers, net):
    """Perturbed-attention guidance arguments, checked before any device work: pag_scale None or a finite real >= 0, and
    pag_layers None (the default layers) or a non-empty sequence of distinct attention-layer names of `net`.  Returns
    (pag_scale, layer indices) when the perturbed rows run (pag_scale > 0), else None.  pag_layers without pag_scale is an
    error: it would silently do nothing."""
    from ..backbones.adm import PAG_DEFAULT_LAYERS
    if pag_scale is None:
        assert pag_layers is None, "pag_layers needs pag_scale"
        return None
    assert isinstance(pag_scale, numbers.Real) and not isinstance(pag_scale, bool), f"pag_scale must be a real number, got {pag_scale!r}"
    assert math.isfinite(pag_scale) and pag_scale >= 0, f"pag_scale must be finite and >= 0, got {pag_scale!r}"
    idx = _unwrap(net).pag_layer_indices(PAG_DEFAULT_LAYERS if pag_layers is None else pag_layers)
    return (float(pag_scale), idx) if pag_scale > 0 else None


class GaussianDiffusion:
    """Utilities for sampling diffusion models (reference gaussian_diffusion.py:12)."""

    def __init__(self, backbone, timesteps=1000, beta_schedule="linear"):
        self.backbone = backbone
        self.timesteps = timesteps
        self.beta_schedule = beta_schedule
        self.backbone_args = edict(inspect.signature(_unwrap(backbone).forward).parameters)
        betas = get_betas_by_name(self.beta_schedule, self.timesteps).astype(np.float64)
        self.betas = betas
        assert len(betas.shape) == 1, "betas must be 1-D"
        assert (betas > 0).all() and (betas <= 1).all(), "betas must be in (0, 1]"
        alphas = 1.0 - betas
        self.alphas_cumprod = np.cumprod(alphas, axis=0)
        self.sqrt_alphas_cumprod = np.sqrt(self.alphas_cumprod)
        self.sqrt_one_minus_alphas_cumprod = np.sqrt(1.0 - self.alphas_cumprod)

    # --- q(x_t | x_0) helpers (gaussian_diffusion.py:45-74); plain torch, not on the hot path -------------------
    def diffuse(self, x_0, t, noise=None):
        if noise is None:
            noise = torch.randn_like(x_0)
        assert noise.shape == x_0.shape, "noise must have same shape as x_0"
        return (_extract(self.sqrt_alphas_cumprod, t, x_0.shape) * x_0
                + _extract(self.sqrt_one_minus_alphas_cumprod, t, x_0.shape) * noise)

    def reverse_diffuse(self, x_t, t, noise):
        assert noise.shape == x_t.shape, "noise must have same shape as x_t"
        return ((x_t - _extract(self.sqrt_one_minus_alphas_cumprod, t, x_t.shape) * noise)
                / _extract(self.sqrt_alphas_cumprod, t, x_t.shape))

    # --- native helpers -------------------------------------------------------------------------------------------
    def _native_forward(self, x, t, classes, strength, cond=None, keep=(), pag=None):
        """eps of one call of `model_inference`, entirely behind the C ABI.

        strength > 0 with a class-conditional model: both classifier-free-guidance halves run as ONE batch-2N forward
        sharing x (the second half gets the null class), then `ivid_cfg_mix` forms (1+s)*eps_c - s*eps_u.  Otherwise a
        single forward, scaled by (1+strength) as the reference does (classifier_free_guidance.py:40-41).
        `cond` is an `_lib.CondT` describing the conditional-input assembly (InpaintCFG / SuperResCFG) or None.
        `pag` = (pag_scale, layer indices) from check_pag adds N perturbed rows to the same forward (classes [c, -1, c]) and
        mixes all blocks with `ivid_guidance_mix`, the step kernels' arithmetic."""
        net = _unwrap(self.backbone)
        net._ensure_packed()
        L = _lib.lib()
        dev = x.device
        N = x.shape[0]
        xx = x.to(torch.float32).contiguous()
        H, W = x.shape[-2:]
        out_shape = (N, net.out_channels, H, W)
        # classes None: both halves of the reference's expression are the same null-class forward, (1+s)e - s*e = e
        two = strength > 0 and classes is not None
        if two:
            assert net.num_classes is not None, "this model is not class-conditioned"
            assert net.has_null_class, "this model does not have a null class"
        nf = 2 * N if two else N
        if pag is not None:
            return self._pag_forward(net, xx, t, classes, strength, two, cond, pag)
        tt = t.to(device=dev, dtype=torch.int64)
        if two:
            tt = tt.repeat(2)
            null = torch.full((N,), -1, dtype=torch.int64, device=dev)
            cc = torch.cat([classes.to(dev, torch.int64), null])
        else:
            cc = classes.to(dev, torch.int64) if classes is not None else None
        tt = tt.contiguous()
        cc = cc.contiguous() if cc is not None else None
        eps = torch.empty((nf,) + out_shape[1:], dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            st = _lib.cur_stream(dev)
            _lib.check(L.ivid_unet_forward_hw(net._handle, _lib.ptr(xx), N, H, W, ctypes.byref(cond) if cond is not None else None,
                                              _lib.ptr(tt), _lib.ptr(cc), _lib.ptr(eps), nf, st))
            if not two:
                return eps if (strength >= 0 and (classes is None or strength == 0)) else (1 + strength) * eps
            out = torch.empty(out_shape, dtype=torch.float32, device=dev)
            _lib.check(L.ivid_cfg_mix(_lib.ptr(eps), float(strength), _lib.ptr(out), out.numel(), st))
        del keep
        return out

    def _pag_forward(self, net, xx, t, classes, strength, two, cond, pag):
        """[cond | null (two) | perturbed] rows in one forward, then G + w (eps_c - eps_perturbed) (include/ivid_b200.h)."""
        L = _lib.lib()
        dev = xx.device
        N, _, H, W = xx.shape
        blocks = 3 if two else 2
        tt = t.to(device=dev, dtype=torch.int64).repeat(blocks).contiguous()
        cc = None
        if classes is not None:
            c = classes.to(dev, torch.int64)
            parts = [c, torch.full((N,), -1, dtype=torch.int64, device=dev), c] if two else [c, c]
            cc = torch.cat(parts).contiguous()
        # G as _native_forward forms it: the mix (two), (1+s) eps_c for strength < 0, eps_c otherwise
        cfg = 1 if two else (2 if strength < 0 else 0)
        w, idx = pag
        arr = (ctypes.c_int * len(idx))(*idx)
        eps = torch.empty((blocks * N, net.out_channels, H, W), dtype=torch.float32, device=dev)
        out = torch.empty((N, net.out_channels, H, W), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            st = _lib.cur_stream(dev)
            _lib.check(L.ivid_unet_forward_perturbed(net._handle, _lib.ptr(xx), N, H, W, ctypes.byref(cond) if cond is not None else None,
                                                     _lib.ptr(tt), _lib.ptr(cc), _lib.ptr(eps), blocks * N, (blocks - 1) * N, arr,
                                                     len(idx), -1, st))
            _lib.check(L.ivid_guidance_mix(_lib.ptr(eps), out.numel(), cfg, float(strength), 1, w, _lib.ptr(out), st))
        return out

    def _cfg_forward(self, x, t, classes, strength, pag=None):
        return self._native_forward(x, t, classes, strength, pag=pag)

    @torch.no_grad()
    def model_inference(self, x, t, classes=None, pag_scale=None, pag_layers=None, **kwargs):
        """Predicted noise (gaussian_diffusion.py:76-91).  pag_scale=w > 0 (extension; perturbed-attention guidance, Ahn et
        al. 2024, arXiv:2403.17377) returns eps_c + w (eps_c - eps_perturbed), eps_perturbed the forward with the attention
        maps of `pag_layers` (names, default ("middle_block.1",)) replaced by the identity, both rows of one forward."""
        pag = check_pag(pag_scale, pag_layers, self.backbone)
        if pag is not None:
            return self._native_forward(x, t, classes, 0.0, pag=pag)
        kwargs = {k: v for k, v in kwargs.items() if k in self.backbone_args}
        return self.backbone(x, t, classes, **kwargs)

    def training_losses(self, *a, **k):
        raise NotImplementedError("training is outside the sampling hot path this package implements")


class ClassifierFreeGuidance(GaussianDiffusion):
    """Diffusion model with classifier-free guidance (classifier_free_guidance.py:12)."""

    def __init__(self, backbone, *, p_uncond=0.1, **kwargs):
        super().__init__(backbone, **kwargs)
        self.p_uncond = p_uncond

    @torch.no_grad()
    def model_inference(self, x, t, classes=None, strength=3.0, pag_scale=None, pag_layers=None, **kwargs):
        # classifier_free_guidance.py:38-42; pag_scale / pag_layers as in GaussianDiffusion.model_inference, added to the mix
        pag = check_pag(pag_scale, pag_layers, self.backbone)
        return self._cfg_forward(x, t, classes, strength, pag=pag)


class InpaintCFG(GaussianDiffusion):
    """Image inpainting with classifier-free guidance (inpaint_cfg.py:11)."""

    def __init__(self, backbone, *, p_uncond=0.1, p_uncond_img=0.0, **kwargs):
        super().__init__(backbone, **kwargs)
        self.p_uncond = p_uncond
        self.p_uncond_img = p_uncond_img

    def make_cond_inputs(self, x, y, mask, noise=None, **kwargs):
        """The 9/10-channel network input of inpaint_cfg.py:24-49 as an fp32 tensor (API parity; the sampling path never
        materialises it — `model_inference` hands the pieces to the fused native assembly instead).
        Holes of the warped RGB / depth are filled with N(0,1): rgb noise is drawn before depth noise, as the
        reference does, unless `noise` [N,4,H,W] injects the draws."""
        m_rgb = kwargs.get("mask_rgb", mask)
        z = noise if noise is not None else self._draw_cond_noise(y)
        filled_rgb = torch.lerp(z[:, :3], y[:, :3], m_rgb)          # y*m + z*(1-m)
        filled_d = torch.lerp(z[:, 3:], y[:, 3:], mask)
        parts = [x] + ([m_rgb] if "mask_rgb" in kwargs else []) + [filled_rgb, filled_d, mask]
        return torch.cat(parts, dim=1)

    @staticmethod
    def _draw_cond_noise(y):
        # two torch draws in the reference's order (inpaint_cfg.py:44,46): keeps the global RNG stream identical
        return torch.cat([torch.randn_like(y[:, :3]), torch.randn_like(y[:, 3:])], dim=1)

    def make_uncond_inputs(self, x):
        # inpaint_cfg.py:52-58: noise everywhere, empty mask
        return torch.cat([x, torch.randn_like(x), x.new_zeros(x[:, :1].shape)], dim=1)

    @torch.no_grad()
    def model_inference(self, x, t, y, mask, classes=None, strength=3.0, noise=None, pag_scale=None, pag_layers=None, **kwargs):
        """inpaint_cfg.py:61-83.  The conditional input is assembled inside the native forward (cond_pack_kernel);
        `noise` [N,4,H,W] injects the hole-filling draws, default = torch draws in the reference's order.  pag_scale /
        pag_layers as in GaussianDiffusion.model_inference; the perturbed rows share the conditional rows' hole noise."""
        pag = check_pag(pag_scale, pag_layers, self.backbone)
        dev = x.device
        f32 = lambda v: None if v is None else v.to(device=dev, dtype=torch.float32).contiguous()
        yy, mm, mr = f32(y), f32(mask), f32(kwargs.get("mask_rgb"))
        zz = f32(noise) if noise is not None else self._draw_cond_noise(yy)
        cond = _lib.CondT()
        cond.kind = 1
        cond.y_dev, cond.mask_dev, cond.mask_rgb_dev, cond.noise_dev = yy.data_ptr(), mm.data_ptr(), (mr.data_ptr() if mr is not None else None), zz.data_ptr()
        # classes None -> single null-class forward without (1+s) scaling (inpaint_cfg.py:77-78)
        return self._native_forward(x, t, classes, strength if classes is not None else 0.0, cond, keep=(yy, mm, mr, zz), pag=pag)


class SuperResCFG(GaussianDiffusion):
    """Image super-resolution with classifier-free guidance (sr_cfg.py:11)."""

    def __init__(self, backbone, *, p_uncond=0.1, **kwargs):
        super().__init__(backbone, **kwargs)
        self.p_uncond = p_uncond

    def make_cond_inputs(self, x, y, **kwargs):
        """cat[x, bilinear-upsampled y] of sr_cfg.py:23-36 as an fp32 tensor (API parity; `model_inference` uses the fused
        native assembly, which applies the same align_corners=False stencil in-kernel)."""
        scale = x.shape[-1] // y.shape[-1]
        up = F.interpolate(y, scale_factor=scale, mode="bilinear", align_corners=False)
        return torch.cat([x, up], dim=1)

    @staticmethod
    def _scale(x, y):
        """The integer upsampling factor s of y -> x; RuntimeError unless y * s == x in both dimensions."""
        s = x.shape[-1] // y.shape[-1] if y.shape[-1] > 0 else 0
        if s < 1 or y.shape[-1] * s != x.shape[-1] or y.shape[-2] * s != x.shape[-2]:
            raise RuntimeError(f"SuperResCFG: x {tuple(x.shape[-2:])} is not an integer multiple of y {tuple(y.shape[-2:])}")
        return s

    @torch.no_grad()
    def model_inference(self, x, t, y, classes=None, strength=3.0, pag_scale=None, pag_layers=None, **kwargs):
        # sr_cfg.py:39-60; pag_scale / pag_layers as in GaussianDiffusion.model_inference
        pag = check_pag(pag_scale, pag_layers, self.backbone)
        yy = y.to(device=x.device, dtype=torch.float32).contiguous()
        cond = _lib.CondT()
        cond.kind = 2
        cond.sr_scale = self._scale(x, yy)
        cond.y_dev = yy.data_ptr()
        return self._native_forward(x, t, classes, strength if classes is not None else 0.0, cond, keep=(yy,), pag=pag)

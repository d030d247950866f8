"""float64 statement of dynamic thresholding (Saharia et al. 2022, "Imagen", arXiv:2205.11487, sec. 2.3) as ivid_b200 runs it
with `dynamic_threshold=p` or `(p, s_max)` (include/ivid_b200.h, ivid_step_args_t).  Test infrastructure only.

Per sample n over its M = C*H*W elements, with v_0 <= ... <= v_{M-1} the sorted |x0|:
    pos = p (M - 1) in double, k = floor(pos), f = pos - k
    q   = v_k + f (v_{min(k+1, M-1)} - v_k) in double, rounded once to the data's precision
    s   = min(max(q, 1), s_max)
    x0 <- clamp(x0, -s, s) / s
On fp32 data every step is the device's (q rounded to fp32, the clamp and the division in fp32); on float64 data it is the
float64 reference.  The step functions restate the DDPM / DDIM / DPM-Solver++ steps of oracle/sampler_ref.py and
oracle/dpm_ref.py with the thresholding in place of their clip, in whatever precision they are given.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import dpm_ref


def quantile(a: np.ndarray, p: float):
    """The p-quantile of the 1-D array a (linear interpolation), in a's dtype."""
    v = np.sort(np.asarray(a).ravel())
    M = v.size
    pos = p * (M - 1)
    k = math.floor(pos)
    f = pos - k
    k1 = min(k + 1, M - 1)
    return v.dtype.type(float(v[k]) + f * (float(v[k1]) - float(v[k])))


def threshold(x0: np.ndarray, p: float, s_max: float | None = None):
    """(s [N], thresholded x0) of x0 [N, ...] (float32 or float64), every sample on its own."""
    x0 = np.asarray(x0)
    dt = x0.dtype.type
    hi = dt(math.inf if s_max is None else s_max)
    s = np.empty(x0.shape[0], dtype=x0.dtype)
    out = np.empty_like(x0)
    for n in range(x0.shape[0]):
        q = quantile(np.abs(x0[n]), p)
        s[n] = min(max(q, dt(1.0)), hi)
        out[n] = np.clip(x0[n], -s[n], s[n]) / s[n]
    return s, out


def _threshold_t(x0: torch.Tensor, p: float, s_max):
    return torch.from_numpy(threshold(x0.detach().cpu().numpy(), p, s_max)[1]).to(x0.device)


def _ex(arr: np.ndarray, t: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
    # sampler_ref._ex in the precision of `like`: float64 table -> index -> cast -> broadcast
    return torch.from_numpy(arr).to(t.device)[t].to(like.dtype).view(-1, *([1] * (like.dim() - 1)))


def ddpm_step(tb, x_t, t, eps, noise, p, s_max=None, x0=None):
    """sampler_ref.ddpm_step with x0 thresholded.  x0 (optional) replaces sqrt(1/acp) x_t - sqrt(1/acp - 1) eps."""
    if x0 is None:
        x0 = _ex(tb.sqrt_recip_alphas_cumprod, t, x_t) * x_t - _ex(tb.sqrt_recipm1_alphas_cumprod, t, x_t) * eps
    x0 = _threshold_t(x0, p, s_max)
    mean = _ex(tb.posterior_mean_coef1, t, x_t) * x0 + _ex(tb.posterior_mean_coef2, t, x_t) * x_t
    logvar = _ex(tb.posterior_log_variance_clipped, t, x_t)
    nz = (t != 0).to(x_t.dtype).view(-1, *([1] * (x_t.dim() - 1)))
    return mean + nz * torch.exp(0.5 * logvar) * noise, x0


def _guide(x0, nz, replace_rgb=None, replace_depth=None, constrain_depth=None):
    """DdimSampler.sample_once's replace / constrain guidance (ddim.py:86-95) on x0, as sampler_ref.ddim_step applies it."""
    x0 = x0.clone()
    if replace_rgb is not None:
        w, rgb, m = replace_rgb
        x0[:, :3] = (1 - nz) * x0[:, :3] + nz * ((w * rgb + (1 - w) * x0[:, :3]) * m + x0[:, :3] * (1 - m))
    if replace_depth:
        w, d, m = replace_depth
        x0[:, 3:] = (w * d + (1 - w) * x0[:, 3:]) * m + x0[:, 3:] * (1 - m)
        if constrain_depth:
            cw, convex = constrain_depth
            x0[:, 3:] = x0[:, 3:] * m + (cw * torch.maximum(x0[:, 3:], convex) + (1 - cw) * x0[:, 3:]) * (1 - m)
    return x0


def ddim_step(tb, x_t, t, t_prev, eps, noise, p, s_max=None, eta=0.0, x0=None, **guidance):
    """sampler_ref.ddim_step with x0 thresholded before the guidance."""
    srac = _ex(tb.sqrt_recip_alphas_cumprod, t - 1, x_t)
    srm1 = _ex(tb.sqrt_recipm1_alphas_cumprod, t - 1, x_t)
    if x0 is None:
        x0 = srac * x_t - srm1 * eps
    nz = (t_prev != 0).to(x_t.dtype).view(-1, *([1] * (x_t.dim() - 1)))
    x0 = _guide(_threshold_t(x0, p, s_max), nz, **guidance)
    eps2 = (srac * x_t - x0) / srm1
    ab = _ex(tb.alphas_cumprod, t - 1, x_t)
    abp = _ex(tb.alphas_cumprod_prev, t_prev, x_t)
    sigma = eta * torch.sqrt((1 - abp) / (1 - ab)) * torch.sqrt(1 - ab / abp)
    mean = torch.sqrt(abp) * x0 + torch.sqrt(1 - abp - sigma ** 2) * eps2
    return mean + nz * sigma * noise, x0


def dpm_d0(acp, x_t, t, t_prev, eps, p, s_max=None, x0=None, **guidance):
    """dpm_ref.guided_x0 (numpy) with x0 thresholded before the guidance: D0 of DPM-Solver++."""
    if x0 is None:
        x0 = np.sqrt(1.0 / acp[t - 1]) * x_t - np.sqrt(1.0 / acp[t - 1] - 1.0) * eps
    x0 = threshold(np.asarray(x0), p, s_max)[1]
    g = {k: tuple(torch.from_numpy(np.asarray(v)) if isinstance(v, np.ndarray) else v for v in val) if val else val
         for k, val in guidance.items()}
    return _guide(torch.from_numpy(x0), 1.0 if t_prev != 0 else 0.0, **g).numpy()


def dpm_update(acp, x_t, d0, t, t_prev, d_prev=None, t_last=None, z=None):
    """x_{t_prev} of DPM-Solver++ from D0: the ODE update of oracle/dpm_ref.py, or the SDE one when z is given."""
    if z is None:
        return dpm_ref.update(acp, x_t, d0, t, t_prev, d_prev, t_last)
    import dpm_sde_ref
    return dpm_sde_ref.sde_update(acp, x_t, d0, z, t, t_prev, d_prev, t_last)

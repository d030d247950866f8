"""DdpmSampler / DdimSampler — host-side mirrors of the reference samplers
(diffusion/samplers/ddpm.py:12-187, diffusion/samplers/ddim.py:12-165) — and DpmSolverSampler, a DPM-Solver++(2M)
sampler, and UniPcSampler, the UniPC predictor-corrector, with the same surface that the reference does not have.

Same constructor (`Sampler(framework)`), same float64 numpy table attributes, same `.sample(...)` / `.sample_once(...)`
signatures and return dict (`samples`, `pred_x_t`, `pred_x_0`).  The step itself — UNet forward with both
classifier-free-guidance halves, eps mix, x_{t-1} update, multiview replace/constrain guidance — runs natively behind
the C ABI; `.sample()` keeps the whole reverse process on the device (no per-step host round trips).

RNG: the reference draws `torch.randn_like` inside every step.  `rng="philox"` (default) draws in-kernel
(Philox4x32-10, seeded from torch's generator); `rng="torch"` draws with torch exactly where the reference does
(one `randn_like(x_t)` per step; for InpaintCFG additionally rgb then depth noise before the model call), which keeps
the torch RNG stream consumption identical to the reference.
"""
from __future__ import annotations

import ctypes
import math
import numbers

import numpy as np
import torch

from .. import _lib
from ..frameworks.gaussian_diffusion import ClassifierFreeGuidance, GaussianDiffusion, InpaintCFG, SuperResCFG
from ..utils import edict
from .options import SamplerOptions

__all__ = ["DdpmSampler", "DdimSampler", "DpmSolverSampler", "UniPcSampler", "init_steps"]


def _unwrap(backbone):
    return backbone.module if hasattr(backbone, "module") else backbone


def _f32(t, device):
    return None if t is None else t.to(device=device, dtype=torch.float32).contiguous()


def _check_interval(guidance_interval, T):
    """(t_lo, t_hi) as ints, or None.  Both bounds are inclusive model times (the t the network receives), 0 <= t_lo <= t_hi < T."""
    if guidance_interval is None:
        return None
    assert len(guidance_interval) == 2, f"guidance_interval must be (t_lo, t_hi), got {guidance_interval!r}"
    lo, hi = (int(v) for v in guidance_interval)
    assert 0 <= lo <= hi < T, f"guidance_interval must satisfy 0 <= t_lo <= t_hi < {T}, got ({lo}, {hi})"
    return lo, hi


def _check_cache(cache_interval, cache_branch, num_res_blocks):
    """Feature reuse (DeepCache) arguments: cache_interval None (no reuse) or an int >= 1, and cache_branch an int in
    [0, num_res_blocks], one of the top-level blocks.  Returns cache_interval as an int, 0 for None."""
    if cache_interval is not None:
        assert isinstance(cache_interval, numbers.Integral) and cache_interval >= 1, \
            f"cache_interval must be None or an integer >= 1, got {cache_interval!r}"
    assert isinstance(cache_branch, numbers.Integral) and 0 <= cache_branch <= num_res_blocks, \
        f"cache_branch must be an integer in [0, num_res_blocks] = [0, {num_res_blocks}], got {cache_branch!r}"
    return int(cache_interval) if cache_interval is not None else 0


def _check_threshold(dynamic_threshold, clip_denoised):
    """Dynamic thresholding argument: None, a ratio p in (0, 1], or a pair (p, s_max) with s_max >= 1 (None: no upper bound).
    It replaces clip_denoised, so the two exclude each other.  Returns (p, s_max) as floats, s_max = inf without a bound, or None."""
    if dynamic_threshold is None:
        return None
    if isinstance(dynamic_threshold, (tuple, list)):
        assert len(dynamic_threshold) == 2, f"dynamic_threshold must be p or (p, s_max), got {dynamic_threshold!r}"
        p, s_max = dynamic_threshold
    else:
        p, s_max = dynamic_threshold, None
    real = lambda v: isinstance(v, numbers.Real) and not isinstance(v, bool)
    assert real(p) and 0.0 < float(p) <= 1.0, f"dynamic_threshold ratio p must be in (0, 1], got {p!r}"
    s_max = math.inf if s_max is None else s_max
    assert real(s_max) and float(s_max) >= 1.0, f"dynamic_threshold s_max must be >= 1, got {s_max!r}"
    assert not clip_denoised, "clip_denoised and dynamic_threshold exclude each other"
    return float(p), float(s_max)


def _check_apg(apg, framework, classes, strength):
    """Adaptive projected guidance argument: None, eta, (eta, r) or (eta, r, beta), eta >= 0, the norm bound r >= 0 (0: none)
    and the momentum beta in (-1, 1), all finite; r and beta default to 0.  It acts on the classifier-free mix, so it needs
    a framework with one, classes and strength > 0.  Returns (eta, r, beta) as floats, or None."""
    if apg is None:
        return None
    vals = tuple(apg) if isinstance(apg, (tuple, list)) else (apg,)
    assert 1 <= len(vals) <= 3, f"apg must be eta, (eta, r) or (eta, r, beta), got {apg!r}"
    eta, r, beta = vals + (0.0,) * (3 - len(vals))
    real = lambda v: isinstance(v, numbers.Real) and not isinstance(v, bool) and math.isfinite(v)
    assert real(eta) and eta >= 0.0, f"apg eta must be finite and >= 0, got {eta!r}"
    assert real(r) and r >= 0.0, f"apg norm bound r must be finite and >= 0, got {r!r}"
    assert real(beta) and -1.0 < beta < 1.0, f"apg momentum beta must lie in (-1, 1), got {beta!r}"
    assert isinstance(framework, (ClassifierFreeGuidance, InpaintCFG, SuperResCFG)), \
        f"apg acts on classifier-free guidance, which {type(framework).__name__} does not have"
    assert classes is not None, "apg acts on classifier-free guidance, which needs classes"
    assert math.isfinite(strength) and strength > 0.0, f"apg needs a guidance strength > 0, got {strength!r}"
    return float(eta), float(r), float(beta)


def init_steps(init_strength, steps):
    """Executed steps n of a run started from an image (SDEdit): round(init_strength * steps), at least 1 and at most steps.
    The run then starts at grid step start_step = steps - n."""
    return min(steps, max(1, int(init_strength * steps + 0.5)))


def _check_init(init, init_strength, noise, image_size, channels):
    """The arguments of a run started from an image, checked before any device work: init [N, channels, H, W] with
    init_strength in (0, 1], noise (the z of the forward diffusion) of init's shape, and no image_size (init sets the size)."""
    if init is None:
        assert init_strength is None, "init_strength needs init"
        return
    assert init_strength is not None, "init needs init_strength, the share of the schedule to run in (0, 1]"
    assert isinstance(init_strength, numbers.Real) and not isinstance(init_strength, bool) and 0.0 < init_strength <= 1.0, \
        f"init_strength must be in (0, 1], got {init_strength!r}"
    assert torch.is_tensor(init) and init.dim() == 4 and init.shape[1] == channels, \
        f"init must be an [N,{channels},H,W] tensor, got {tuple(init.shape) if torch.is_tensor(init) else type(init).__name__}"
    assert image_size is None, "init sets the sample size: do not pass image_size with it"
    assert noise is None or tuple(noise.shape) == tuple(init.shape), \
        f"noise (the forward diffusion's z) must have init's shape {tuple(init.shape)}, got {tuple(noise.shape)}"


class _NativeSampler:
    KIND = 0
    UNIPC = False     # kind 2 only: the UniPC update instead of DPM-Solver++

    def __init__(self, framework):
        self.framework = framework
        betas = np.ascontiguousarray(self.framework.betas, dtype=np.float64)
        alphas = 1.0 - betas
        # attribute parity with the reference (ddpm.py:26-41, ddim.py:26-31)
        self.alphas_cumprod = np.cumprod(alphas, axis=0)
        self.alphas_cumprod_prev = np.append(1.0, self.alphas_cumprod[:-1])
        self.sqrt_recip_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod)
        self.sqrt_recipm1_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod - 1)
        self._handle = ctypes.c_void_p()
        _lib.check(_lib.lib().ivid_sampler_create(betas.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), len(betas),
                                                  ctypes.byref(self._handle)))
        self._keep = []   # tensors referenced by raw pointer during a native call

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                _lib.lib().ivid_sampler_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    def native_table(self, which: int) -> np.ndarray:
        out = np.empty(len(self.framework.betas), dtype=np.float64)
        _lib.check(_lib.lib().ivid_sampler_table(self._handle, which, out.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), len(out)))
        return out

    # ------------------------------------------------------------------------------------------------------------
    def _guidance(self, kwargs):
        """(uses_cfg, strength): whether the framework mixes in a null-class forward, and model_inference's strength
        (default 3.0); 0.0 for a framework without classifier-free guidance."""
        uses_cfg = isinstance(self.framework, (ClassifierFreeGuidance, InpaintCFG, SuperResCFG))
        return uses_cfg, float(kwargs.get("strength", 3.0)) if uses_cfg else 0.0

    def _step_args(self, device, classes, clip_denoised, eta, kwargs, step_noise=None, cond_noise=None, seed=0, hw=None,
                   order=0, prev=None, sde=False, interval=None, cache=None, threshold=None, prev_x=None, corrected=None, pag=None,
                   apg=None, apg_state=None):
        fw = self.framework
        a = _lib.StepArgsT()
        keep = []

        def P(t):
            if t is None:
                return None
            t = _f32(t, device)
            keep.append(t)
            return t.data_ptr()

        a.kind = self.KIND
        uses_cfg, a.strength = self._guidance(kwargs)
        a.use_cfg = 1 if uses_cfg else 0
        a.clip_denoised = 1 if clip_denoised else 0
        a.eta = float(eta)
        if classes is not None:
            c = classes.to(device=device, dtype=torch.int64).contiguous()
            keep.append(c)
            a.classes_dev = c.data_ptr()
        if isinstance(fw, InpaintCFG):
            assert "y" in kwargs and "mask" in kwargs, "InpaintCFG.model_inference needs y and mask"
            a.cond.kind = 1
            a.cond.y_dev = P(kwargs["y"])
            a.cond.mask_dev = P(kwargs["mask"])
            a.cond.mask_rgb_dev = P(kwargs.get("mask_rgb"))
            a.cond.noise_dev = P(cond_noise)
        elif isinstance(fw, SuperResCFG):
            assert "y" in kwargs, "SuperResCFG.model_inference needs y"
            a.cond.kind = 2
            a.cond.y_dev = P(kwargs["y"])
            if hw is not None:
                a.cond.sr_scale = SuperResCFG._scale(torch.empty(0, 0, *hw), kwargs["y"])
        rr = kwargs.get("replace_rgb")
        if rr is not None:
            assert self.KIND in (1, 2), "replace_rgb is a DdimSampler / DpmSolverSampler argument"
            a.replace_rgb_weight = float(rr[0]); a.replace_rgb_dev = P(rr[1]); a.replace_rgb_mask_dev = P(rr[2])
        rd = kwargs.get("replace_depth")
        if rd:
            a.replace_depth_weight = float(rd[0]); a.replace_depth_dev = P(rd[1]); a.replace_depth_mask_dev = P(rd[2])
            cd = kwargs.get("constrain_depth")
            if cd:
                a.constrain_depth_weight = float(cd[0]); a.constrain_depth_dev = P(cd[1])
        a.step_noise_dev = P(step_noise)
        a.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        if hw is not None:
            a.height, a.width = int(hw[0]), int(hw[1])
        a.order = int(order)
        step_t = lambda t: int(t[0]) if torch.is_tensor(t) and t.dim() > 0 else int(t)
        if self.UNIPC:
            # up to three (t_last, pred_x_0) pairs, newest first, and the corrector's base
            a.unipc = 1
            slots = (("prev_x0_dev", "t_last"), ("prev2_x0_dev", "t_last2"), ("prev3_x0_dev", "t_last3"))
            for (x_field, t_field), (t_last, x0_last) in zip(slots, prev or ()):
                setattr(a, t_field, step_t(t_last))
                setattr(a, x_field, P(x0_last))
            a.prev_xt_dev = P(prev_x)
            a.corrected_xt_dev = _lib.ptr(corrected).value
        elif prev is not None:
            t_last, x0_last = prev
            a.t_last = step_t(t_last)
            a.prev_x0_dev = P(x0_last)
        a.sde = 1 if sde else 0
        if interval is not None:
            a.guidance_interval = 1
            a.guidance_t_lo, a.guidance_t_hi = interval
        if cache is not None:
            a.cache_interval, a.cache_branch, a.cache_reuse = (int(v) for v in cache)
        if threshold is not None:
            a.dynamic_threshold = 1
            a.threshold_ratio = threshold[0]
            a.threshold_max = 0.0 if math.isinf(threshold[1]) else threshold[1]
        if pag is not None:
            layers = (ctypes.c_int * len(pag[1]))(*pag[1])
            keep.append(layers)
            a.pag, a.pag_scale, a.pag_layers, a.pag_num_layers = 1, pag[0], layers, len(pag[1])
        if apg is not None:
            a.apg = 1
            a.apg_eta, a.apg_norm, a.apg_momentum = apg
            a.apg_state_dev = _lib.ptr(apg_state).value
        return a, keep

    def _net(self):
        net = _unwrap(self.framework.backbone)
        net._ensure_packed()
        return net

    def _native_step(self, x_t, t, t_prev, classes, clip_denoised, eta, kwargs, noise, cond_noise, order=0, prev=None,
                     sde=False, interval=None, cache=None, threshold=None, prev_x=None, pag=None, apg=None, apg_state=None):
        """One step.  `t` / `t_prev` are host ints (ivid_sampler_step) or the [N] tensors sample_once receives
        (ivid_sampler_step_dev: the step is read on the device, no host sync; t_prev None for DDPM).  With `apg`, the
        momentum state m_prev (None: zero history) is copied, and the copy receives m: it is the returned `apg_state`."""
        net = self._net()
        dev = x_t.device
        x_t = _f32(x_t, dev)
        corrected = torch.empty_like(x_t) if self.UNIPC else None
        if apg is not None:
            apg_state = torch.zeros_like(x_t) if apg_state is None else _f32(apg_state, dev).clone()
        a, keep = self._step_args(dev, classes, clip_denoised, eta, kwargs, step_noise=noise, cond_noise=cond_noise,
                                  hw=x_t.shape[-2:], order=order, prev=prev, sde=sde, interval=interval, cache=cache,
                                  threshold=threshold, prev_x=prev_x, corrected=corrected, pag=pag, apg=apg,
                                  apg_state=apg_state)
        x_prev = torch.empty_like(x_t)
        x0 = torch.empty_like(x_t)
        L = _lib.lib()
        head = (self._handle, net._handle, _lib.ptr(x_t), _lib.ptr(x_prev), _lib.ptr(x0), x_t.shape[0])
        with torch.cuda.device(dev):
            if torch.is_tensor(t):
                td = t.to(device=dev, dtype=torch.int64).contiguous()
                tp = t_prev.to(device=dev, dtype=torch.int64).contiguous() if t_prev is not None else None
                rc = L.ivid_sampler_step_dev(*head, _lib.ptr(td), _lib.ptr(tp), ctypes.byref(a), _lib.cur_stream(dev))
            else:
                rc = L.ivid_sampler_step(*head, int(t), int(t_prev), ctypes.byref(a), _lib.cur_stream(dev))
            _lib.check(rc)
        del keep
        out = edict({"pred_x_prev": x_prev, "pred_x_0": x0})
        if self.UNIPC:
            out.corrected_x_t = corrected
        if apg is not None:
            out.apg_state = apg_state
        return out

    def _sample_once(self, x_t, t, t_prev, classes, clip_denoised, eta, kwargs, noise, opts, reuse_features, order=0,
                     prev=None, sde=False, prev_x=None, apg_state=None):
        """The body of every sample_once: the host checks before any device work or torch draw, the step noise (drawn as
        the reference draws it, or the injected `noise` and kwargs' `cond_noise`), then the step with t / t_prev read on
        the device (all samples of a batch share the step, ddpm.py:177-179, ddim.py:154-158: no host sync)."""
        B = x_t.shape[0]
        assert t.shape == (B,), "t must be a 1D tensor of shape (B,)"
        assert self.KIND == 0 or t_prev.shape == (B,), "t_prev must be a 1D tensor of shape (B,)"
        opts = opts.resolve(self.framework, classes, self._guidance(kwargs)[1], clip_denoised)
        assert apg_state is None or opts.apg is not None, "apg_state needs apg"
        assert apg_state is None or tuple(apg_state.shape) == tuple(x_t.shape), \
            f"apg_state must have x_t's shape {tuple(x_t.shape)}, got {tuple(apg_state.shape)}"
        if noise is None:
            noise, cond_noise = self._draw_step_noise(x_t, kwargs)
        else:
            cond_noise = kwargs.pop("cond_noise", None)
        # the DPM-Solver++ ODE update reads no step noise
        return self._native_step(x_t, t, t_prev, classes, clip_denoised, eta, kwargs, noise if self.KIND != 2 or sde else None,
                                 cond_noise, order=order, prev=prev, sde=sde, prev_x=prev_x, apg_state=apg_state,
                                 **opts.step_kwargs(reuse_features))

    def _draw_step_noise(self, x_t, kwargs):
        """torch draws in the reference's order: InpaintCFG rgb, depth (inside model_inference), then randn_like(x_t)."""
        cond_noise = None
        if isinstance(self.framework, InpaintCFG):
            y = kwargs["y"]
            n_rgb = torch.randn_like(y[:, :3])
            n_d = torch.randn_like(y[:, 3:])
            cond_noise = torch.cat([n_rgb, n_d], dim=1)
        return torch.randn_like(x_t), cond_noise

    def _reuse_schedule(self, model_times, classes, kwargs, interval, cache_interval, pag=None):
        """Whether each step of a run reuses the cached features, by ivid_sampler_run's rule: a full forward at the first
        step, where the forward switches plans (the guided batch of 2N or 3N rows and the unguided batch-N plan), and
        cache_interval steps after the last full one."""
        _, strength = self._guidance(kwargs)
        reuse, last_full, last_rows = [], 0, 0
        for i, tm in enumerate(model_times):
            inside = interval is None or interval[0] <= tm <= interval[1]
            rows = 1 + (classes is not None and strength > 0 and inside) + (pag is not None and inside)
            full = cache_interval <= 1 or i == 0 or rows != last_rows or i - last_full >= cache_interval
            if full:
                last_full = i
            last_rows = rows
            reuse.append(not full)
        return reuse

    def _run(self, num, image_size, noise, classes, steps, clip_denoised, eta, verbose, rng, return_trajectory, kwargs, opts,
             order=0, sde=False, init=None, init_strength=None):
        opts = opts.resolve(self.framework, classes, self._guidance(kwargs)[1], clip_denoised)   # before any device work
        _check_init(init, init_strength, noise, image_size, _unwrap(self.framework.backbone).out_channels)
        net = self._net()
        net.eval()
        if image_size is None:
            image_size = net.image_size
        device = net.device
        if init is not None:
            x_init = _f32(init, device)
            img = torch.empty_like(x_init)
        else:
            # as in the reference (ddpm.py:168-176), given noise is used as-is and defines the sample size
            img = noise if noise is not None else torch.randn((num, net.out_channels, image_size, image_size), device=device)
            assert img.dim() == 4 and img.shape[1] == net.out_channels, f"noise must be [N,{net.out_channels},H,W], got {tuple(img.shape)}"
            img = _f32(img, device).clone()
        num = img.shape[0]
        shape = tuple(img.shape)
        T = self.framework.timesteps
        nsteps = T if self.KIND == 0 else (steps if steps is not None else T)
        ret = edict({"samples": None, "pred_x_t": [], "pred_x_0": []})
        start = 0
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if rng == "philox" else 0
        if init is not None:
            # SDEdit: x at grid step start = steps - n is q(x_t | init) at that step's model time, jump * n - 1 (n - 1 for DDPM)
            n = init_steps(init_strength, nsteps)
            start = nsteps - n
            jump = 1 if self.KIND == 0 else T // nsteps
            # z: the given noise, Philox(seed) on a stream no step uses, or (rng="torch") randn_like(x_0) as diffuse draws it
            z = _f32(noise, device) if noise is not None else (torch.randn_like(x_init) if rng == "torch" else None)
            with torch.cuda.device(device):
                _lib.check(_lib.lib().ivid_sampler_diffuse(self._handle, _lib.ptr(x_init), _lib.ptr(z), num, x_init[0].numel(),
                                                           jump * n - 1, seed, _lib.ptr(img), _lib.cur_stream(device)))
        if rng == "torch":
            if self.KIND == 0:
                sched = [(i, 0) for i in range(T)][::-1]
            else:
                jump = T // nsteps
                sched = [(jump * (i + 1), jump * i) for i in reversed(range(nsteps))]
            sched = sched[start:]
            prev, prev_x, apg_state = None, None, None
            reuse = self._reuse_schedule([t if self.KIND == 0 else t - 1 for (t, _) in sched], classes, kwargs, opts.interval,
                                         opts.cache_interval, opts.pag)
            for i, (t, t_prev) in enumerate(sched):
                z, cond_noise = self._draw_step_noise(img, kwargs)
                # the DPM-Solver++ ODE update draws z only to consume the torch RNG as DdimSampler does
                out = self._native_step(img, t, t_prev, classes, clip_denoised, eta, kwargs, z if self.KIND != 2 or sde else None,
                                        cond_noise, order=order, prev=prev, sde=sde, prev_x=prev_x, apg_state=apg_state,
                                        **opts.step_kwargs(reuse[i]))
                if opts.apg is not None:
                    apg_state = out.apg_state
                if self.UNIPC:
                    prev, prev_x = ([(t, out.pred_x_0)] + (prev or []))[:order], out.corrected_x_t
                elif self.KIND == 2 and order != 1:
                    prev = (t, out.pred_x_0)
                img = out.pred_x_prev
                if return_trajectory:
                    ret.pred_x_t.append(out.pred_x_prev)
                    ret.pred_x_0.append(out.pred_x_0)
        elif rng == "philox":
            a, keep = self._step_args(device, classes, clip_denoised, eta, kwargs, seed=seed, hw=shape[-2:], order=order, sde=sde,
                                      **opts.step_kwargs())
            a.start_step = start
            traj0 = trajt = None
            if return_trajectory:
                traj0 = torch.empty((nsteps - start,) + shape, dtype=torch.float32, device=device)
                trajt = torch.empty((nsteps - start,) + shape, dtype=torch.float32, device=device)
            with torch.cuda.device(device):
                _lib.check(_lib.lib().ivid_sampler_run(self._handle, net._handle, _lib.ptr(img), num, int(nsteps), ctypes.byref(a),
                                                       None, None, _lib.ptr(traj0), _lib.ptr(trajt), _lib.cur_stream(device)))
            del keep
            if return_trajectory:
                ret.pred_x_t = list(trajt.unbind(0))
                ret.pred_x_0 = list(traj0.unbind(0))
        else:
            raise ValueError("rng must be 'philox' or 'torch'")
        ret.samples = img
        net.train()   # the reference toggles eval()/train() around sampling (ddpm.py:166,186)
        return ret


class DdpmSampler(_NativeSampler):
    """Generate samples with the DDPM ancestral schedule (reference ddpm.py:12)."""
    KIND = 0

    def __init__(self, framework):
        super().__init__(framework)
        betas = self.framework.betas
        alphas = 1.0 - betas
        self.posterior_variance = betas * (1.0 - self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_log_variance_clipped = np.log(np.append(self.posterior_variance[1], self.posterior_variance[1:]))
        self.posterior_mean_coef1 = betas * np.sqrt(self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_mean_coef2 = (1.0 - self.alphas_cumprod_prev) * np.sqrt(alphas) / (1.0 - self.alphas_cumprod)

    @torch.no_grad()
    def sample_once(self, x_t, t, classes=None, clip_denoised=False, noise=None, guidance_interval=None, reuse_features=False,
                    cache_branch=0, dynamic_threshold=None, pag_scale=None, pag_layers=None, apg=None, apg_state=None, **kwargs):
        """x_{t-1} from x_t (ddpm.py:111-131).  `t` is the [N] tensor of steps minus 1 (all equal).
        `noise` (extension) injects the randn_like draw; default draws it with torch like the reference.
        `guidance_interval=(t_lo, t_hi)` (extension): the step is guided only if t lies in [t_lo, t_hi] (see `sample`).
        `reuse_features=True` (extension): the step's forward reuses the deep features of the last full forward of the same
        batch and size at branch `cache_branch` (see `sample`); RuntimeError if no full forward has run on it.
        `dynamic_threshold=p` or `(p, s_max)` (extension): dynamic thresholding of x_0 (see `sample`).
        `pag_scale` / `pag_layers` (extension): perturbed-attention guidance (see `sample`).
        `apg` (extension): adaptive projected guidance (see `sample`).  `apg_state` is the momentum state the previous step
        returned as `out.apg_state` (None at the first step: zero history); the step returns its own, so steps chained with
        apg_state = out.apg_state reproduce a run, as `prev` / `prev_x` chain the multistep samplers."""
        opts = SamplerOptions(guidance_interval, None, cache_branch, dynamic_threshold, pag_scale, pag_layers, apg)
        return self._sample_once(x_t, t, None, classes, clip_denoised, 0.0, kwargs, noise, opts, reuse_features, apg_state=apg_state)

    @torch.no_grad()
    def sample(self, num, steps=None, image_size=None, noise=None, classes=None, clip_denoised=False, verbose=True,
               rng="philox", return_trajectory=False, guidance_interval=None, cache_interval=None, cache_branch=0,
               dynamic_threshold=None, init=None, init_strength=None, pag_scale=None, pag_layers=None, apg=None, **kwargs):
        """Run the full reverse process (ddpm.py:134-187).  `steps` is accepted and ignored exactly as in the reference.
        pred_x_t / pred_x_0 are only materialised with return_trajectory=True (the reference keeps 2x1000 tensors alive;
        its callers read `.samples` only: inference/sample.py:82).

        guidance_interval=(t_lo, t_hi) (extension; Kynkaanniemi et al. 2024, arXiv:2404.07724): classifier-free guidance
        only at the steps whose model time t (the t the network receives) lies in [t_lo, t_hi], 0 <= t_lo <= t_hi < T;
        every other step is the same step at strength 0 and runs one batch-N forward instead of the batch-2N one.  None
        (default) guides every step.  No effect without classes.

        cache_interval=N, cache_branch=b (extension; DeepCache, Ma, Fang, Wang, CVPR 2024, arXiv:2312.00858): a full network
        forward every N steps; the steps in between recompute only the shallow branch b (the stem, input blocks 0..b, the
        last b + 1 output blocks and the head) and reuse the deeper up-path features of the last full forward.  A step where
        the guidance interval switches between the guided and the unguided forward is always full.  0 <= b <=
        num_res_blocks; b = 0 is the cheapest.  None (default) or 1 runs every forward in full.  The update, the noise and the
        torch RNG consumption are those of a run without reuse; eps is an approximation.

        dynamic_threshold=p or (p, s_max) (extension; Saharia et al. 2022, arXiv:2205.11487, sec. 2.3): at every step, where
        clip_denoised would clamp x_0, each sample's x_0 is clamped to [-s, s] and divided by s, s = min(max(q, 1), s_max) and q
        the p-quantile of |x_0| over the sample (linear interpolation, as numpy.quantile); s_max defaults to no bound, p in
        (0, 1], s_max >= 1.  The guidance and the update then read the thresholded x_0 (include/ivid_b200.h).  Excludes
        clip_denoised; s_max = 1 is clip_denoised=True.  The noise and the torch RNG consumption are unchanged.

        init=x_0, init_strength=s (extension; SDEdit, Meng et al. 2022, arXiv:2108.01073): start from the image x_0 ([N, C, H, W]
        in the model's [-1, 1] range; it sets N and the size, so image_size must stay None) instead of x_T.  Of the schedule's
        `steps` steps (T for DDPM) the last n = min(steps, max(1, round(s * steps))) run, 0 < s <= 1: x_0 is diffused to the
        first of them by q(x_t | x_0) (GaussianDiffusion.diffuse at model time jump * n - 1), with `noise` as its z if given,
        and the run goes on from there.  Low s stays close to x_0; s = 1 runs the whole schedule from a noised x_0.  Each
        executed step is the step of a full run; the multistep history and feature reuse start afresh at the first one.
        pred_x_t / pred_x_0 hold the n executed steps.  rng="torch" draws z with randn_like(x_0) before the steps.

        pag_scale=w, pag_layers=names (extension; perturbed-attention guidance, Ahn et al. 2024, arXiv:2403.17377): every
        guided step adds N rows to its forward, the conditional forward with the attention maps of the named attention layers
        (default ("middle_block.1",)) replaced by the identity, and uses eps = G + w (eps_c - eps_perturbed), G the eps of the
        step without it (the classifier-free mix, if any).  It works without classes, so it guides class-free models too.  The
        guidance interval gates it like classifier-free guidance.  w >= 0; None or 0 is the run without it, bit for bit.  The
        noise and the torch RNG consumption are unchanged (the InpaintCFG hole noise is shared by the perturbed rows).

        apg=eta, (eta, r) or (eta, r, beta) (extension; adaptive projected guidance, Sadat, Hilliges, Weber, ICLR 2025,
        arXiv:2410.02416): every guided step replaces the classifier-free mix by an update in x_0 space.  Per sample, with
        D_c / D_u the x_0 of the conditional / null-class eps and m = (D_c - D_u) + beta m_prev (momentum across guided steps),
        the update is scaled to norm at most r and its part parallel to D_c weighted by eta: D = D_c + s c (m - k D_c),
        c = min(1, r / |m|), k = (1 - eta) <m, D_c> / |D_c|^2, s the strength (include/ivid_b200.h).  eta >= 0, r >= 0 (0: no
        bound, the default), -1 < beta < 1 (default 0).  eta = 1, r = 0, beta = 0 is classifier-free guidance up to rounding.
        Needs a classifier-free-guidance framework, classes and strength > 0.  Clipping or dynamic thresholding, the
        multiview guidance and the update read D.  The noise and the torch RNG consumption are unchanged; None (default) is
        the run without it, bit for bit."""
        opts = SamplerOptions(guidance_interval, cache_interval, cache_branch, dynamic_threshold, pag_scale, pag_layers, apg)
        return self._run(num, image_size, noise, classes, None, clip_denoised, 0.0, verbose, rng, return_trajectory, kwargs, opts,
                         init=init, init_strength=init_strength)


class DdimSampler(_NativeSampler):
    """Generate samples using DDIM (reference ddim.py:12), including the multiview replace/constrain guidance."""
    KIND = 1

    @torch.no_grad()
    def sample_once(self, x_t, t, t_prev, classes=None, clip_denoised=False, eta=0.0, replace_rgb=None,
                    replace_depth=None, constrain_depth=None, noise=None, guidance_interval=None, reuse_features=False,
                    cache_branch=0, dynamic_threshold=None, pag_scale=None, pag_layers=None, apg=None, apg_state=None, **kwargs):
        """x_{t_prev} from x_t (ddim.py:48-103).  t / t_prev are [N] tensors of actual steps (1 means one step).
        `guidance_interval=(t_lo, t_hi)`: the step is guided only if its model time t - 1 lies in [t_lo, t_hi].
        `reuse_features` / `cache_branch` / `dynamic_threshold` / `pag_scale` / `pag_layers` / `apg` / `apg_state` as in
        DdpmSampler.sample_once."""
        kw = dict(kwargs, replace_rgb=replace_rgb, replace_depth=replace_depth, constrain_depth=constrain_depth)
        opts = SamplerOptions(guidance_interval, None, cache_branch, dynamic_threshold, pag_scale, pag_layers, apg)
        return self._sample_once(x_t, t, t_prev, classes, clip_denoised, eta, kw, noise, opts, reuse_features, apg_state=apg_state)

    @torch.no_grad()
    def sample(self, num, image_size=None, noise=None, classes=None, steps=None, clip_denoised=False, eta=0.0,
               verbose=True, rng="philox", return_trajectory=False, guidance_interval=None, cache_interval=None, cache_branch=0,
               dynamic_threshold=None, init=None, init_strength=None, pag_scale=None, pag_layers=None, apg=None, **kwargs):
        """Run `steps` DDIM steps (ddim.py:106-165).  `guidance_interval=(t_lo, t_hi)` as in DdpmSampler.sample, on the model
        time t - 1 of each step; `cache_interval` / `cache_branch` / `dynamic_threshold` as in DdpmSampler.sample (the replace /
        constrain guidance acts on the thresholded x_0).  `init` / `init_strength`, `pag_scale` / `pag_layers` and `apg` as
        in DdpmSampler.sample (the replace / constrain guidance acts on the APG-guided x_0)."""
        opts = SamplerOptions(guidance_interval, cache_interval, cache_branch, dynamic_threshold, pag_scale, pag_layers, apg)
        return self._run(num, image_size, noise, classes, steps, clip_denoised, eta, verbose, rng, return_trajectory, kwargs, opts,
                         init=init, init_strength=init_strength)


class DpmSolverSampler(_NativeSampler):
    """DPM-Solver++(2M) (Lu et al. 2022), the second-order multistep solver in data-prediction form, on DdimSampler's
    time grid (jump = T // steps, model called at t - 1) with the same guidance (classifier-free mix, multiview replace /
    constrain applied to x_0 exactly as DdimSampler.sample_once applies it).  The update is fused into the output head like
    the DDPM / DDIM steps (include/ivid_b200.h, kind 2).

    With alpha = sqrt(alphas_cumprod), sigma = sqrt(1 - alphas_cumprod) at t - 1 (s) and t_prev - 1 (p), h = lambda_p -
    lambda_s for lambda = log(alpha / sigma), and D the guided x_0 (order 1) or (1 + 1/(2r)) D0 - 1/(2r) D_{-1} (order 2):
      sde=False (ODE, deterministic):  x_p = sigma_p/sigma_s x_t + alpha_p (1 - e^-h) D;          order 1 = DDIM, eta = 0
      sde=True  (SDE-DPM-Solver++(2M)): x_p = sigma_p/sigma_s e^-h x_t + alpha_p (1 - e^-2h) D
                                              + sigma_p sqrt(1 - e^-2h) z,  z ~ N(0, 1);        order 1 = DDIM, eta = 1"""
    KIND = 2

    @torch.no_grad()
    def sample_once(self, x_t, t, t_prev, classes=None, clip_denoised=False, prev=None, replace_rgb=None, replace_depth=None,
                    constrain_depth=None, noise=None, sde=False, guidance_interval=None, reuse_features=False, cache_branch=0,
                    dynamic_threshold=None, pag_scale=None, pag_layers=None, apg=None, apg_state=None, **kwargs):
        """x_{t_prev} from x_t.  t / t_prev are [N] tensors of actual steps, as for DdimSampler.sample_once.
        `prev = (t_last, pred_x_0)` of the previous step selects the second-order update, None the first-order one.
        With sde=True `noise` is the injected z of the update; with sde=False the update does not use it.  When it is None
        the torch RNG is consumed exactly as DdimSampler.sample_once consumes it (InpaintCFG hole noise, then one
        randn_like(x_t), which is z for sde=True); `cond_noise` injects the hole noise.  `guidance_interval`, `reuse_features`,
        `cache_branch` and `dynamic_threshold` as for DdimSampler.sample_once (D0, and so pred_x_0, is thresholded);
        `pag_scale` / `pag_layers` and `apg` / `apg_state` as for DdpmSampler.sample_once."""
        kw = dict(kwargs, replace_rgb=replace_rgb, replace_depth=replace_depth, constrain_depth=constrain_depth)
        opts = SamplerOptions(guidance_interval, None, cache_branch, dynamic_threshold, pag_scale, pag_layers, apg)
        return self._sample_once(x_t, t, t_prev, classes, clip_denoised, 0.0, kw, noise, opts, reuse_features,
                                 order=2 if prev is not None else 1, prev=prev, sde=sde, apg_state=apg_state)

    @torch.no_grad()
    def sample(self, num, image_size=None, noise=None, classes=None, steps=None, order=2, clip_denoised=False, verbose=True,
               rng="philox", return_trajectory=False, sde=False, guidance_interval=None, cache_interval=None, cache_branch=0,
               dynamic_threshold=None, init=None, init_strength=None, pag_scale=None, pag_layers=None, apg=None, **kwargs):
        """Run `steps` DPM-Solver++ steps of order `order` (1 or 2), the SDE variant with sde=True.  The first step and the
        final step (to t_prev = 0, which returns x_0 as DDIM does and draws no noise) are first order.  The SDE's step noise
        is drawn where DdimSampler draws it (`rng`).  `guidance_interval` as in DdimSampler.sample; the history D_{-1} of a
        step after an unguided one is that step's unguided D0.  `cache_interval` / `cache_branch` as in DdpmSampler.sample;
        the history D_{-1} of a step is that step's D0, from whichever forward ran.  `dynamic_threshold` as in
        DdpmSampler.sample: D0 is the thresholded, guided x_0, and so is the history.  `init` / `init_strength` as in
        DdpmSampler.sample; the first executed step is first order.  `pag_scale` / `pag_layers` as in DdpmSampler.sample; the
        history holds the PAG-guided D0.  `apg` as in DdpmSampler.sample; the history holds the APG-guided D0.  Same return
        dict as DdimSampler.sample."""
        assert order in (1, 2), f"order must be 1 or 2, got {order}"
        opts = SamplerOptions(guidance_interval, cache_interval, cache_branch, dynamic_threshold, pag_scale, pag_layers, apg)
        return self._run(num, image_size, noise, classes, steps, clip_denoised, 0.0, verbose, rng, return_trajectory, kwargs, opts,
                         order=order, sde=bool(sde), init=init, init_strength=init_strength)


class UniPcSampler(_NativeSampler):
    """UniPC (Zhao et al. 2023, "UniPC: A Unified Predictor-Corrector Framework for Fast Sampling of Diffusion Models",
    arXiv:2302.04867), data prediction with B(h) = e^h - 1 ("bh2"), multistep of order 1 to 3, on DdimSampler's time grid with
    DpmSolverSampler's guidance (classifier-free mix, multiview replace / constrain applied to x_0).  Each step first corrects
    the previous prediction x_t with the model output D0 this step computes anyway (the corrector UniC, which raises the order
    by one at no extra network evaluation), then predicts x_{t_prev} from the corrected x_t (UniP, at orders 1 and 2 the
    DPM-Solver++ update).  The network always sees the uncorrected prediction.  The corrector, predictor and history update
    run fused into the output head (include/ivid_b200.h, kind 2 with unipc = 1)."""
    KIND = 2
    UNIPC = True

    @torch.no_grad()
    def sample_once(self, x_t, t, t_prev, classes=None, clip_denoised=False, prev=None, prev_x=None, order=2, replace_rgb=None,
                    replace_depth=None, constrain_depth=None, noise=None, guidance_interval=None, reuse_features=False,
                    cache_branch=0, dynamic_threshold=None, pag_scale=None, pag_layers=None, apg=None, apg_state=None, **kwargs):
        """One UniPC step from x_t.  t / t_prev are [N] tensors of actual steps, as for DdimSampler.sample_once.
        `prev` is a list of up to three `(t_last, pred_x_0)` pairs of the previous steps, newest first, and `prev_x` the
        previous step's `corrected_x_t` (the corrector's base; required with `prev`).  With n pairs (at most `order` are used)
        the step corrects at order min(order, n) and predicts at order min(order, n + 1); the step to t_prev = 0 returns x_0.
        Returns `pred_x_prev` (the prediction the next step's network sees), `pred_x_0` and `corrected_x_t` (x_t itself
        without `prev`).  Chain steps with prev = ([(t, pred_x_0)] + prev)[:3] and prev_x = corrected_x_t.  `noise` is not used; the
        torch RNG is consumed as DpmSolverSampler.sample_once consumes it.  `guidance_interval`, `reuse_features`,
        `cache_branch`, `dynamic_threshold`, `pag_scale` / `pag_layers` and `apg` / `apg_state` as for DdimSampler.sample_once."""
        assert order in (1, 2, 3), f"order must be 1, 2 or 3, got {order}"
        prev = list(prev) if prev is not None else []
        assert len(prev) <= 3, f"prev holds at most three (t_last, pred_x_0) pairs, got {len(prev)}"
        assert not prev or prev_x is not None, "prev needs prev_x, the previous step's corrected_x_t"
        kw = dict(kwargs, replace_rgb=replace_rgb, replace_depth=replace_depth, constrain_depth=constrain_depth)
        opts = SamplerOptions(guidance_interval, None, cache_branch, dynamic_threshold, pag_scale, pag_layers, apg)
        return self._sample_once(x_t, t, t_prev, classes, clip_denoised, 0.0, kw, noise, opts, reuse_features,
                                 order=order, prev=prev, prev_x=prev_x, apg_state=apg_state)

    @torch.no_grad()
    def sample(self, num, image_size=None, noise=None, classes=None, steps=None, order=2, clip_denoised=False, verbose=True,
               rng="philox", return_trajectory=False, guidance_interval=None, cache_interval=None, cache_branch=0,
               dynamic_threshold=None, init=None, init_strength=None, pag_scale=None, pag_layers=None, apg=None, **kwargs):
        """Run `steps` UniPC steps of order `order` (1, 2 or 3; 2 is the paper's choice for guided sampling).  Step i predicts
        at order min(order, i + 1) and corrects at the previous step's order; the first step has no corrector and the final
        step (to t_prev = 0) returns x_0 as DDIM does.  pred_x_t holds the predictions the network saw.  Draws no step noise;
        the torch RNG is consumed as DpmSolverSampler.sample(sde=False) consumes it.  `guidance_interval`, `cache_interval` /
        `cache_branch` and `dynamic_threshold` as in DpmSolverSampler.sample: the history holds the D0 of whichever forward
        ran, thresholded.  `init` / `init_strength`, `pag_scale` / `pag_layers` and `apg` as in DdpmSampler.sample; the order
        ramp starts at the first executed step.  Same return dict as DdimSampler.sample."""
        assert order in (1, 2, 3), f"order must be 1, 2 or 3, got {order}"
        opts = SamplerOptions(guidance_interval, cache_interval, cache_branch, dynamic_threshold, pag_scale, pag_layers, apg)
        return self._run(num, image_size, noise, classes, steps, clip_denoised, 0.0, verbose, rng, return_trajectory, kwargs, opts,
                         order=order, init=init, init_strength=init_strength)

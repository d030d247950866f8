"""Super-resolution stage of the multiview pipeline: the V views of a scene, generated at S x S, re-sampled at S' = s * S by a
SuperResCFG network (the reference's rgbd_*_adm_256_128_small_sr configs, 128^2 -> 256^2), view by view in the order they
were generated.  Each view after the first is guided towards the super-resolved views before it, warped to its camera at S'
by the device warp, with the replace guidance the conditional stage uses (sample.py:104-119):

    view 0:  SR sampler (y = low-res view 0)                                         -> RGBD at S' on the GPU
    view j:  DeviceWarp.aggregate at S' of the SR views 0 .. j-1                    -> condition maps at S'
             SR sampler (y = low-res view j) with replace guidance from those maps    -> RGBD at S' on the GPU

The network forward with its conditional-input assembly, the fused step and the warp are native; nothing in the step loop
runs in PyTorch.
"""
from __future__ import annotations

import numbers

import torch

from .. import frameworks
from ..rgbd_3d import DeviceWarp
from ..samplers.options import SamplerOptions, solver_sampler

__all__ = ["superresolve_views", "check_superres"]


def _unwrap(backbone):
    return backbone.module if hasattr(backbone, "module") else backbone


def check_superres(framework_sr, S, size=None, replace=(0.1, 0.2)):
    """The stage's own arguments, checked before any device work: framework_sr a SuperResCFG, the output size S' = size or
    the SR backbone's image_size an integer multiple s >= 2 of the input size S, and replace None or two weights in [0, 1].
    Returns (S', s).  Raises ValueError."""
    if not isinstance(framework_sr, frameworks.SuperResCFG):
        raise ValueError(f"framework_sr must be a SuperResCFG, got {type(framework_sr).__name__}")
    out = _unwrap(framework_sr.backbone).image_size if size is None else size
    if not isinstance(out, numbers.Integral) or isinstance(out, bool) or out <= 0:
        raise ValueError(f"the super-resolved size must be a positive integer, got {out!r}")
    out = int(out)
    if out % S != 0 or out // S < 2:
        raise ValueError(f"the super-resolved size {out} must be an integer multiple s >= 2 of the view size {S}")
    if replace is not None:
        if not isinstance(replace, (tuple, list)) or len(replace) != 2:
            raise ValueError(f"replace must be None or (rgb weight, depth weight), got {replace!r}")
        for w in replace:
            if not (isinstance(w, numbers.Real) and not isinstance(w, bool) and 0.0 <= w <= 1.0):
                raise ValueError(f"replace weights must lie in [0, 1], got {replace!r}")
    return out, out // S


def _per_sample(modelviews):
    return isinstance(modelviews[0], (list, tuple))


@torch.no_grad()
def superresolve_views(framework_sr, views, modelviews, steps=50, size=None, classes=None, guidance=3.0, seeds=None,
                       replace=(0.1, 0.2), fov=45, near=0.6, far=5, atol=0.03, rtol=0.03, erode_rgb=3, rng="philox",
                       solver="ddim", precision="fp16", guidance_interval=None, cache_interval=None, cache_branch=0,
                       dynamic_threshold=None, pag_scale=None, pag_layers=None, apg=None, cache=None):
    """views [B, V, 4, S, S] in [-1, 1] (model space), in the order they were generated; modelviews as sample_all takes them:
    one list of V cameras shared by the batch, or B lists of V -> [B, V, 4, S', S'] on the SR network's device.

    S' = size or framework_sr.backbone.image_size, an integer multiple s >= 2 of S.  Every view runs the ODE sampler of
    `solver` (DdimSampler, DpmSolverSampler, with sde=True for 'dpmpp_sde', or UniPcSampler) for `steps` steps with y = the
    low-res view, classes and guidance as SuperResCFG takes them (without classes, one null-class forward).  View j >= 1 adds
    the replace guidance of the conditional stage, replace_rgb = (replace[0], colour, mask_rgb) and replace_depth =
    (replace[1], depth, mask), from DeviceWarp(B, image_size=S', ssaa=3, max_views=V).aggregate of the super-resolved views
    0 .. j-1.  There is no constrain_depth: the low-res depth is known everywhere.  The default weights are the conditional
    stage's 0.1 and 0.2, not tuned for super-resolution.  replace=None runs every view on its own, without the warp.
    The warp takes the pipeline's fov, near, far, atol and rtol as given and erode_rgb * s, so that the eroded band covers
    the same angle at S'.

    With seeds (one per sample), the x_T of view v of the sample seeded sd is row v of torch.randn(V, 4, S', S',
    generator=torch.Generator().manual_seed(sd)): a scene's result does not depend on its batch.  Without seeds the samplers
    draw x_T at S' from the torch RNG, as they draw it elsewhere.  precision is applied to the SR backbone (set_precision); the other options are the samplers' (guidance
    interval, feature reuse, dynamic thresholding, PAG, APG).  `cache` (a dict the caller keeps across calls) holds the
    samplers and one DeviceWarp per batch size."""
    assert torch.is_tensor(views) and views.dim() == 5 and views.shape[2] == 4 and views.shape[3] == views.shape[4], \
        f"views must be [B,V,4,S,S], got {tuple(views.shape) if torch.is_tensor(views) else type(views).__name__}"
    B, V, _, S, _ = views.shape
    S2, s = check_superres(framework_sr, S, size, replace)
    if _per_sample(modelviews):
        assert len(modelviews) == B and all(len(m) == V for m in modelviews), \
            f"modelviews must be {B} lists of {V} cameras (or one list of {V})"
    else:
        assert len(modelviews) == V, f"modelviews must hold {V} cameras, got {len(modelviews)}"
    assert isinstance(steps, numbers.Integral) and steps >= 1, f"steps must be an integer >= 1, got {steps!r}"
    assert seeds is None or len(seeds) == B, f"seeds must hold one seed per sample ({B}), got {len(seeds)}"
    assert classes is None or len(classes) == B, f"classes must hold one class per sample ({B}), got {len(classes)}"
    ode, sde = solver_sampler(solver)
    opts = SamplerOptions(guidance_interval, cache_interval, cache_branch, dynamic_threshold, pag_scale, pag_layers, apg)
    opts.resolve(framework_sr, classes, guidance)
    net = _unwrap(framework_sr.backbone)
    if net.precision != precision:
        net.set_precision(precision)
    dev = net.device
    cache = {} if cache is None else cache
    key = ("sampler", id(framework_sr), ode)
    if key not in cache:
        cache[key] = ode(framework_sr)
    sampler = cache[key]
    kw = dict(steps=steps, verbose=False, rng=rng, **opts.sampler_kwargs(framework_sr, guidance))
    if sde:
        kw["sde"] = True
    b_classes = None
    if classes is not None:
        b_classes = (classes if torch.is_tensor(classes) else torch.tensor(list(classes))).to(device=dev, dtype=torch.int64)
    noise = None
    if seeds is not None:
        noise = torch.stack([torch.randn(V, 4, S2, S2, generator=torch.Generator().manual_seed(int(sd))) for sd in seeds], 0).to(dev)
    wparams = dict(fov=fov, near=near, far=far, atol=atol, rtol=rtol, erode_rgb=erode_rgb * s)
    warp = None
    if replace is not None and V > 1:
        wkey = ("warp", B, S2, V, dev.index)
        if wkey not in cache:
            cache[wkey] = DeviceWarp(B, image_size=S2, ssaa=3, max_views=V, device=dev.index)
        warp = cache[wkey]
        warp.reset()
    out = []
    for j in range(V):
        mv_j = [modelviews[k][j] for k in range(B)] if _per_sample(modelviews) else modelviews[j]
        args = {}
        if warp is not None and j > 0:
            c = warp.aggregate(mv_j, **wparams)                             # [B,7,S',S'] in [0,1]
            mask, mask_rgb = c[:, 4:5], c[:, 5:6]
            args = dict(replace_rgb=(replace[0], c[:, :3] * 2 - 1, mask_rgb), replace_depth=(replace[1], c[:, 3:4] * 2 - 1, mask))
        # x_T: the seeded rows, or drawn by the sampler at S' (without image_size it would draw at the backbone's own size)
        x_kw = dict(noise=noise[:, j]) if noise is not None else dict(noise=None, image_size=S2)
        res = sampler.sample(B, y=views[:, j], classes=b_classes, **x_kw, **args, **kw)
        out.append(res.samples)
        if warp is not None and j < V - 1:
            warp.add_view(res.samples, mv_j, **wparams)
    return torch.stack(out, dim=1)

"""What a sampler run is configured with beyond the reference's own arguments (guidance interval, feature reuse, dynamic
thresholding, PAG, APG), from the command-line flags to the step arguments, and the solvers of the pipeline's DDIM-step
views.  SamplerOptions holds the options as the samplers take them; resolve checks them into ResolvedOptions."""
from __future__ import annotations

import argparse
import math
from dataclasses import dataclass, fields

from ..backbones.adm import PAG_DEFAULT_LAYERS
from ..frameworks.gaussian_diffusion import ClassifierFreeGuidance, InpaintCFG, SuperResCFG, check_pag

__all__ = ["SamplerOptions", "ResolvedOptions", "SOLVERS", "solver_sampler", "add_arguments", "check_arguments"]

SOLVERS = ("ddim", "dpmpp", "dpmpp_sde", "unipc")


def solver_sampler(solver):
    """(sampler class, sde) of a solver name; 'dpmpp_sde' is DpmSolverSampler with sde=True."""
    from . import DdimSampler, DpmSolverSampler, UniPcSampler      # the package's; samplers.py imports this module
    assert solver in SOLVERS, f"solver must be one of {SOLVERS}, got {solver!r}"
    return {"ddim": (DdimSampler, False), "dpmpp": (DpmSolverSampler, False), "dpmpp_sde": (DpmSolverSampler, True),
            "unipc": (UniPcSampler, False)}[solver]


@dataclass(frozen=True)
class ResolvedOptions:
    """Checked options: interval (t_lo, t_hi) or None, cache_interval an int (0: no reuse), cache_branch, threshold
    (p, s_max) or None, pag (scale, layer indices) or None, apg (eta, r, beta) or None."""
    interval: tuple | None = None
    cache_interval: int = 0
    cache_branch: int = 0
    threshold: tuple | None = None
    pag: tuple | None = None
    apg: tuple | None = None

    def step_kwargs(self, reuse=None):
        """The option keywords of the samplers' step arguments: for a run (reuse None), which reuses the cached features
        every cache_interval steps, or for one step, which reuses them if `reuse`."""
        cache = (self.cache_interval, self.cache_branch, 0) if reuse is None else (0, self.cache_branch, bool(reuse))
        return dict(interval=self.interval, cache=cache, threshold=self.threshold, pag=self.pag, apg=self.apg)


@dataclass(frozen=True)
class SamplerOptions:
    """The options of every sampler's sample / sample_once and of sample_all; the samplers' docstrings give their meaning."""
    guidance_interval: tuple | None = None
    cache_interval: int | None = None
    cache_branch: int = 0
    dynamic_threshold: float | tuple | None = None
    pag_scale: float | None = None
    pag_layers: tuple | None = None
    apg: float | tuple | None = None

    def resolve(self, framework, classes, strength, clip_denoised=False) -> ResolvedOptions:
        """The options checked against `framework`, its classes and guidance strength (AssertionError), normalised."""
        from .samplers import _check_apg, _check_cache, _check_interval, _check_threshold   # samplers.py imports this module
        net = framework.backbone
        return ResolvedOptions(
            interval=_check_interval(self.guidance_interval, len(framework.betas)),
            cache_interval=_check_cache(self.cache_interval, self.cache_branch, getattr(net, "module", net).num_res_blocks),
            cache_branch=self.cache_branch,
            threshold=_check_threshold(self.dynamic_threshold, clip_denoised),
            pag=check_pag(self.pag_scale, self.pag_layers, net),
            apg=_check_apg(self.apg, framework, classes, strength))

    def sampler_kwargs(self, framework, strength):
        """The keywords of `framework`'s sampler, each only when set.  A framework with classifier-free guidance takes
        `strength` and the guidance interval; one without takes the interval only to gate perturbed-attention guidance."""
        cfg = isinstance(framework, (ClassifierFreeGuidance, InpaintCFG, SuperResCFG))
        kw = dict(strength=strength) if cfg else {}
        if self.guidance_interval is not None and (cfg or self.pag_scale is not None):
            kw["guidance_interval"] = tuple(self.guidance_interval)
        if self.cache_interval is not None:
            kw.update(cache_interval=self.cache_interval, cache_branch=self.cache_branch)
        if self.dynamic_threshold is not None:
            kw["dynamic_threshold"] = self.dynamic_threshold
        if self.pag_scale is not None:
            kw.update(pag_scale=self.pag_scale, pag_layers=self.pag_layers)
        if self.apg is not None:
            kw["apg"] = self.apg
        return kw

    @classmethod
    def from_args(cls, opt):
        """The options of a parsed command line (add_arguments); an attribute it lacks takes the field's default."""
        return cls(**{f.name: getattr(opt, f.name, f.default) for f in fields(cls)})

    def dir_suffixes(self):
        """The parts of an output directory name these options add: (interval, cache and threshold parts; PAG and APG parts)."""
        dt, layers, apg = self.dynamic_threshold, self.pag_layers, self.apg
        head = (("" if self.guidance_interval is None else f"_interval{self.guidance_interval[0]}-{self.guidance_interval[1]}")
                + ("" if self.cache_interval is None else f"_cache{self.cache_interval}b{self.cache_branch}")
                + ("" if dt is None else f"_dthresh{dt}" if not isinstance(dt, tuple) else f"_dthresh{dt[0]}-{dt[1]}"))
        # _pag{W}, plus the layers ('+'-joined) when they are not the default; _apg{ETA}, then ,{R} and ,{BETA} as given
        tail = (("" if self.pag_scale is None else f"_pag{self.pag_scale}"
                 + ("" if layers is None or tuple(layers) == PAG_DEFAULT_LAYERS else "-" + "+".join(layers)))
                + ("" if apg is None else "_apg" + ",".join(str(v) for v in (apg if isinstance(apg, tuple) else (apg,)))))
        return head, tail


def check_arguments(ap, opt):
    """The check between the option flags: --pag_layers needs --pag_scale (ap.error)."""
    if opt.pag_layers is not None and opt.pag_scale is None:
        ap.error("--pag_layers needs --pag_scale")


def int_at_least(lo):
    def parse(s):
        try:
            v = int(s)
        except ValueError:
            raise argparse.ArgumentTypeError(f"expected an integer, got {s!r}") from None
        if v < lo:
            raise argparse.ArgumentTypeError(f"expected an integer >= {lo}, got {s!r}")
        return v
    return parse


def parse_interval(s):
    """'LO,HI' -> (LO, HI), the inclusive model-time bounds of --guidance_interval."""
    parts = s.split(",")
    if len(parts) != 2:
        raise argparse.ArgumentTypeError(f"expected LO,HI, got {s!r}")
    try:
        lo, hi = int(parts[0]), int(parts[1])
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected two integers LO,HI, got {s!r}") from None
    if not 0 <= lo <= hi:
        raise argparse.ArgumentTypeError(f"expected 0 <= LO <= HI, got {s!r}")
    return lo, hi


def parse_threshold(s):
    """'P' or 'P,MAX' -> P or (P, MAX) of --dynamic_threshold: the quantile ratio 0 < P <= 1 and the bound MAX >= 1."""
    parts = s.split(",")
    if len(parts) not in (1, 2):
        raise argparse.ArgumentTypeError(f"expected P or P,MAX, got {s!r}")
    try:
        vals = [float(v) for v in parts]
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected numbers P[,MAX], got {s!r}") from None
    if not 0.0 < vals[0] <= 1.0:
        raise argparse.ArgumentTypeError(f"expected 0 < P <= 1, got {s!r}")
    if len(vals) == 2 and not vals[1] >= 1.0:
        raise argparse.ArgumentTypeError(f"expected MAX >= 1, got {s!r}")
    return vals[0] if len(vals) == 1 else (vals[0], vals[1])


def parse_apg(s):
    """'ETA', 'ETA,R' or 'ETA,R,BETA' -> ETA or the tuple of --apg: ETA >= 0, the norm bound R >= 0 (0: none) and the
    momentum -1 < BETA < 1, all finite."""
    parts = s.split(",")
    if len(parts) not in (1, 2, 3):
        raise argparse.ArgumentTypeError(f"expected ETA[,R[,BETA]], got {s!r}")
    try:
        vals = [float(v) for v in parts]
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected numbers ETA[,R[,BETA]], got {s!r}") from None
    if not all(math.isfinite(v) for v in vals):
        raise argparse.ArgumentTypeError(f"expected finite numbers, got {s!r}")
    if vals[0] < 0.0 or (len(vals) > 1 and vals[1] < 0.0):
        raise argparse.ArgumentTypeError(f"expected ETA >= 0 and R >= 0, got {s!r}")
    if len(vals) == 3 and not -1.0 < vals[2] < 1.0:
        raise argparse.ArgumentTypeError(f"expected -1 < BETA < 1, got {s!r}")
    return vals[0] if len(vals) == 1 else tuple(vals)


def parse_pag_scale(s):
    """'W' -> W of --pag_scale, a finite number >= 0."""
    try:
        v = float(s)
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected a number, got {s!r}") from None
    if not (math.isfinite(v) and v >= 0.0):
        raise argparse.ArgumentTypeError(f"expected a finite W >= 0, got {s!r}")
    return v


def parse_pag_layers(s):
    """'NAME[,NAME...]' -> the tuple of attention-layer names of --pag_layers (checked against the network when it is built)."""
    names = tuple(n.strip() for n in s.split(","))
    if not names or any(not n for n in names):
        raise argparse.ArgumentTypeError(f"expected NAME[,NAME...], got {s!r}")
    return names


def add_arguments(ap):
    """The flags of the solver, the network precision and every SamplerOptions field (from_args reads the latter)."""
    ap.add_argument("--solver", choices=SOLVERS, default="ddim",
                    help="sampler of the DDIM-step views: 'ddim' as the reference, 'dpmpp' DPM-Solver++(2M), which needs fewer "
                         "steps for the same convergence, 'dpmpp_sde' its stochastic variant SDE-DPM-Solver++(2M), 'unipc' the "
                         "UniPC predictor-corrector at order 2 (DDPM at --steps_uncond >= 1000 is unchanged)")
    ap.add_argument("--precision", choices=["fp16", "fp8"], default="fp16",
                    help="operands of the ResBlock convs: 'fp16' (default) or 'fp8' (e4m3, faster, changes the numbers; DESIGN.md §2)")
    ap.add_argument("--guidance_interval", type=parse_interval, default=None, metavar="LO,HI",
                    help="apply classifier-free guidance only at the steps whose model time t (0 <= t < T, the t the network "
                         "receives) lies in [LO, HI]; the other steps run unguided with half the network work (default: every step)")
    ap.add_argument("--cache_interval", type=int_at_least(1), default=None, metavar="N",
                    help="reuse the deep UNet features between denoising steps (DeepCache): a full forward every N steps, shallow "
                         "forwards in between; approximates the samples (default: every forward in full)")
    ap.add_argument("--cache_branch", type=int_at_least(0), default=0, metavar="B",
                    help="with --cache_interval: the shallow forwards recompute input blocks 0..B and the last B+1 output blocks, "
                         "0 <= B <= num_res_blocks (default 0, the cheapest)")
    ap.add_argument("--dynamic_threshold", type=parse_threshold, default=None, metavar="P[,MAX]",
                    help="dynamic thresholding of the predicted x_0 (Imagen): clamp each sample's x_0 to [-s, s] and divide by s, "
                         "s = min(max(P-quantile of |x_0|, 1), MAX); e.g. 0.995 (default: off; MAX defaults to no bound)")
    ap.add_argument("--pag_scale", type=parse_pag_scale, default=None, metavar="W",
                    help="perturbed-attention guidance of both networks at scale W >= 0: adds W * (eps - eps with identity "
                         "attention maps) at every guided step; works without classes (default: off)")
    ap.add_argument("--pag_layers", type=parse_pag_layers, default=None, metavar="NAME[,NAME...]",
                    help="with --pag_scale: the attention layers to perturb, by state-dict name (default: middle_block.1)")
    ap.add_argument("--apg", type=parse_apg, default=None, metavar="ETA[,R[,BETA]]",
                    help="adaptive projected guidance of both networks: the guidance update split into its parts parallel and "
                         "orthogonal to the conditional x_0, the parallel part weighted by ETA, the update's norm bounded by R "
                         "(0: no bound) and a momentum BETA across steps; e.g. 0,0,-0.5 (default: plain classifier-free guidance)")

"""CPU: the UniPC sampler's arithmetic (float64 oracle, tests/unipc_ref.py), its convergence order on data with a closed-form
probability-flow ODE, its per-step order pattern, and the host-side error contracts of UniPcSampler, sample_all, the CLI and
the C ABI."""
import ctypes
import json

import numpy as np
import pytest

import ivid_b200.samplers as samplers
import unipc_ref
from ivid_b200 import _lib
from ivid_b200.inference import sample as sample_mod
from oracle import dpm_ref, sampler_ref
from test_dpm_solver import ACP, T, TINY, _gaussian_problem, _rel, _tiny_fw


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("stop_at", [200, 0])
def test_predictor_alone_is_dpm_solver(order, stop_at):
    """Without the corrector, UniP at orders 1 and 2 is the DPM-Solver++ update."""
    x_T, eps_fn, _ = _gaussian_problem()
    for steps in (10, 25, 50):
        a = unipc_ref.run(ACP, x_T, eps_fn, steps, order, stop_at=stop_at, corrector=False)
        b = dpm_ref.run(ACP, x_T, eps_fn, steps, order, stop_at=stop_at)
        assert _rel(a, b) < 1e-12, (order, steps, _rel(a, b))


def test_convergence_order_on_gaussian_data():
    """The corrector raises the order by one: doubling the steps from 50 to 100 to 200 divides the error at t = 200 by ~4 at
    order 1, by 6.6-7.3 at order 2 (approaching 8) and by ~16 at order 3."""
    x_T, eps_fn, exact = _gaussian_problem()
    want = exact(x_T, T, 200)
    for order, lo, hi in ((1, 3.5, 4.5), (2, 6.0, 9.0), (3, 14.0, 18.0)):
        err = [_rel(unipc_ref.run(ACP, x_T, eps_fn, n, order, stop_at=200), want) for n in (50, 100, 200)]
        ratios = [err[i] / err[i + 1] for i in range(2)]
        assert all(lo < r < hi for r in ratios), (order, err, ratios)


def test_order2_beats_dpm_solver_2m():
    x_T, eps_fn, exact = _gaussian_problem()
    want = exact(x_T, T, 200)
    for n in (10, 20, 25, 50, 100, 200):
        e_uni = _rel(unipc_ref.run(ACP, x_T, eps_fn, n, 2, stop_at=200), want)
        e_dpm = _rel(dpm_ref.run(ACP, x_T, eps_fn, n, 2, stop_at=200), want)
        assert e_uni < e_dpm, (n, e_uni, e_dpm)


def test_order_pattern_and_final_step():
    """Step i predicts at order min(order, i + 1) and corrects at the previous step's order (none on the first step); the final
    step to t_prev = 0 is first order and returns D0.  The grid is DdimSampler's."""
    for order in (1, 2, 3):
        for steps in (1, 2, 3, 4, 10, 50):
            sch = unipc_ref.schedule(T, steps, order)
            assert [(t, tp) for (t, tp, _, _) in sch] == sampler_ref.ddim_schedule(T, steps)
            want_q = [min(order, i + 1) for i in range(steps - 1)] + [1]
            assert [q for (_, _, q, _) in sch] == want_q, (order, steps)
            assert [qc for (*_, qc) in sch] == [0] + want_q[:-1], (order, steps)
    x_T, eps_fn, _ = _gaussian_problem()
    rng = np.random.default_rng(5)
    d0, x_t, base = rng.standard_normal(64), rng.standard_normal(64), rng.standard_normal(64)
    hist = [(40, rng.standard_normal(64)), (60, rng.standard_normal(64))]
    x_p, x_c = unipc_ref.step(ACP, x_t, d0, 20, 0, 1, 2, hist, base)
    assert np.array_equal(x_p, d0), "the final step returns D0"
    assert not np.array_equal(x_c, x_t), "and still corrects x_t"


def test_python_surface_and_errors(monkeypatch):
    fw = _tiny_fw()
    uni, dpm = samplers.UniPcSampler(fw), samplers.DpmSolverSampler(fw)
    for name in ("alphas_cumprod", "alphas_cumprod_prev", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod"):
        assert np.array_equal(getattr(uni, name), getattr(dpm, name)), name
    for bad in (0, 4, -1):
        with pytest.raises(AssertionError):
            uni.sample(1, order=bad, verbose=False)
        with pytest.raises(AssertionError):
            uni.sample_once(None, None, None, order=bad)
    with pytest.raises(AssertionError):
        uni.sample_once(None, None, None, prev=[(40, None)])              # prev without prev_x
    with pytest.raises(AssertionError):
        uni.sample_once(None, None, None, prev=[(40, None)] * 4, prev_x=0)
    # sample_all: solver="unipc" runs UniPcSampler at order 2 where the reference runs DdimSampler
    calls = []

    class _Stop(Exception):
        pass

    def fake_sample(self, *a, **kw):
        calls.append((type(self).__name__, kw.get("order", 2), kw.get("sde")))
        raise _Stop

    monkeypatch.setattr(samplers.UniPcSampler, "sample", fake_sample)
    monkeypatch.setattr(samplers.DdpmSampler, "sample", fake_sample)
    for steps_uncond, want in ((10, ("UniPcSampler", 2, None)), (1000, ("DdpmSampler", 2, None))):
        with pytest.raises(_Stop):
            next(sample_mod.sample_all(fw, None, 1, steps_uncond, 10, [None], solver="unipc"))
        assert calls[-1] == want, calls
    with pytest.raises(AssertionError):
        next(sample_mod.sample_all(fw, None, 1, 10, 10, [None], solver="unipc3"))
    # the CLI
    opt = sample_mod.build_arg_parser().parse_args(["--solver", "unipc"])
    assert opt.solver == "unipc"
    assert sample_mod.output_dir_name(opt).endswith("_unipc")
    with pytest.raises(SystemExit):
        sample_mod.build_arg_parser().parse_args(["--solver", "unipc3"])


def test_native_error_contract():
    """The C entry points reject a bad UniPC request with IVID_ERR_INVALID_ARGUMENT before any device work; without
    unipc = 1, kind 3 and kind 2 at order 3 stay rejected."""
    L = _lib.lib()
    unet = ctypes.c_void_p()
    _lib.check(L.ivid_unet_create(json.dumps(TINY).encode(), ctypes.byref(unet)))
    s = samplers.UniPcSampler(_tiny_fw())
    fake = ctypes.c_void_p(256)        # never dereferenced: every call below fails its argument checks first

    def args(**fields):
        a = _lib.StepArgsT()
        a.kind, a.unipc, a.order = 2, 1, 2
        for k, v in fields.items():
            setattr(a, k, v)
        return a

    def step(t, tp, **fields):
        return L.ivid_sampler_step(s._handle, unet, fake, fake, None, 1, t, tp, ctypes.byref(args(**fields)), None)

    hist1 = dict(prev_x0_dev=256, t_last=520, prev_xt_dev=256)
    try:
        cases = [
            (dict(unipc=2), "unipc must be 0 or 1"),
            (dict(unipc=-1), "unipc must be 0 or 1"),
            (dict(kind=1), "unipc = 1 needs kind 2"),
            (dict(kind=0), "unipc = 1 needs kind 2"),
            (dict(sde=1), "unipc = 1 needs kind 2 and sde = 0"),
            (dict(order=0), "UniPC order"),
            (dict(order=4), "UniPC order"),
            (dict(kind=3), "sampler kind"),
            (dict(unipc=0, order=3), "DPM-Solver++ order"),
            (dict(prev_x0_dev=256, t_last=520), "prev_xt_dev"),
            (dict(prev2_x0_dev=256, t_last2=540, prev_xt_dev=256), "prev2_x0_dev needs prev_x0_dev"),
            (dict(hist1, prev3_x0_dev=256, t_last3=560, order=3), "prev3_x0_dev needs prev2_x0_dev"),
            (dict(hist1, t_last=500), "above t"),
            (dict(hist1, t_last=1001), "t_last out of range"),
            (dict(hist1, prev2_x0_dev=256, t_last2=520), "above t"),
            (dict(hist1, prev2_x0_dev=256, t_last2=510), "above t"),
            (dict(hist1, prev2_x0_dev=256, t_last2=1001), "t_last out of range"),
            (dict(hist1, prev2_x0_dev=256, t_last2=540, prev3_x0_dev=256, t_last3=530, order=3), "above t"),
        ]
        for fields, msg in cases:
            rc = step(500, 480, **fields)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and msg in _lib.last_error(), (fields, _lib.last_error())
        for fields, msg in ((dict(order=4), "UniPC order"), (dict(sde=1), "sde = 0"), (dict(unipc=3), "unipc")):
            rc = L.ivid_sampler_run(s._handle, unet, fake, 1, 10, ctypes.byref(args(**fields)), None, None, None, None, None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and msg in _lib.last_error(), (fields, _lib.last_error())
    finally:
        L.ivid_unet_destroy(unet)

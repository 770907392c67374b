"""The device samplers through divergent and non-finite trajectories against the oracle: the case table of
tests/test_divergence_host.py (overflowing static steps, a NaN region, adapted mass matrices containing 0.0) on the thread- and
warp-per-chain kernels, the streamed shapes (rows across lanes, DMMA, the scatter-add, placement 1 with and without the tile
pipeline), pooled adaptation, tracked diagnostics over chains that never move, and density_batch at non-finite positions.

Data-free models in parity math are compared bit for bit (equal_nan).  Streamed and DMMA shapes sum in another order: their
decisions, step counts, log-accept classes and RNG states are equal, their samples agree within the tolerance those paths
already use.  Non-finite values are ordinary data here; nothing provokes a device fault."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.binding import OracleModel
from oracle.rainier_py.diagnostics import trace_diagnostics
from rainier_b200 import abi, api

import parity
import pooled_dense as pd
import pooled_step as ps
from test_divergence_host import CASES, MASS_ZERO, classes, nan_model, oracle_run, spread_seeds

pytestmark = pytest.mark.gpu

CHAINS = 64


def _device_run(rir, cols, config, seeds, env=None, track_thin=None):
    """samples [chains][iterations][n], trace, per-chain rn_chain_stats, mass, the return code and message of
    rn_sampler_stats (RN_E_INVALID for a mass matrix containing 0.0, whose stats are still filled in), tracked diagnostics,
    the emitted kernel source"""
    import torch

    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        cfg, keep = api.lower_config(config)
        gm = api.CudaModel(rir, cols, device=0)
        src = gm.emit_source(config)  # the source of the kernels this sampler launches
        s = api.CudaSampler(gm, config, seeds=seeds, trace=True)
        d = torch.empty((max(cfg.iterations, 1), gm.nVars, s.chains), dtype=torch.float64, device="cuda:0")
        s.warmup(-1)
        if track_thin is not None:
            s.track_diagnostics(track_thin)
        s.run(cfg.iterations, d.data_ptr())
        s.sync()
        diag = s.tracked_diagnostics() if track_thin is not None else None
        samples = d[: cfg.iterations].permute(2, 0, 1).contiguous().cpu().numpy()
        n = gm.nVars
        dense = cfg.mass_tuner == abi.RN_MASS_DENSE
        stats = (abi.ChainStats * s.chains)()
        mass = np.empty((s.chains, n * n if dense else n), dtype=np.float64)
        rings = np.zeros((s.chains, 3, cfg.stats_window), dtype=np.float64)
        rc = api.lib().rn_sampler_stats(s.h, C.cast(stats, C.c_void_p), mass.ctypes.data, rings.ctypes.data)
        msg = api.lib().rn_last_error().decode() if rc else ""
        trace = s.read_trace()
        s.close()
        gm.close()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return {"samples": samples, "trace": trace, "stats": stats, "mass": mass, "rc": rc, "msg": msg, "diag": diag, "src": src}


def _same_chain(g, c, ref, rc, exact=True, tol=1e-9, huge=np.inf):
    gt, rt = g["trace"][c], ref["trace"][rc]
    if exact:
        assert np.array_equal(gt, rt, equal_nan=True), "trace of chain %d differs" % c
        assert np.array_equal(g["samples"][c], ref["samples"][rc], equal_nan=True), "samples of chain %d differ" % c
        assert np.array_equal(g["mass"][c], ref["mass"][rc], equal_nan=True), "mass of chain %d differs" % c
    else:
        for col in (1, 3):  # decisions, leapfrog steps
            assert np.array_equal(gt[:, col], rt[:, col]), "chain %d: trace column %d differs" % (c, col)
        # -inf or finite per iteration; 0 and a finite negative value differ only by the rounding of a deltaH near 0.0, so
        # finite values are compared within tol.  huge: where either side's log-accept is beyond -huge (-inf included), the
        # energies of the trajectory are near the overflow threshold, and fast math's contracted products change the
        # log-accept's class and value there (never the decision, which is compared above)
        la_g, la_r = gt[:, 0], rt[:, 0]
        sure = ~((np.abs(la_r) > huge) | (np.abs(la_g) > huge))
        assert np.array_equal(np.isneginf(la_g)[sure], np.isneginf(la_r)[sure]), "chain %d: log-accept classes differ" % c
        fin = np.isfinite(la_r) & np.isfinite(la_g) & sure
        assert (np.abs(la_g[fin] - la_r[fin]) <= tol * np.maximum(1.0, np.abs(la_r[fin]))).all(), "chain %d: log-accepts" % c
        assert parity.rel_err(gt[:, 2], rt[:, 2]) < tol
        assert parity.rel_err(g["samples"][c], ref["samples"][rc], 1e-9) < tol, "samples of chain %d" % c
    o, s = ref["stats"][rc], g["stats"][c]
    assert s.gradient_evaluations == o.gradient_evaluations and s.leapfrog_steps == o.leapfrog_steps
    assert s.accepted == o.accepted and s.iterations == o.iterations
    assert s.rng.seed48 == o.rng.seed48, "RNG streams of chain %d diverged" % c


def _check_case(case, backend, env=None):
    rir, cols, config, cfg, seeds, ref = oracle_run(case, CHAINS)
    config.backend = backend
    g = _device_run(rir, cols, config, seeds, env)
    if isinstance(ref, tuple):  # adapted mass containing 0.0 on some chains
        zero, per_chain = ref
        assert g["rc"] == abi.RN_E_INVALID and g["msg"] == MASS_ZERO, (g["rc"], g["msg"])
        bits = np.array([(s.error_flags & 2) != 0 for s in g["stats"]])
        assert np.array_equal(bits, zero), "chains with error bit 2: %s, oracle: %s" % (np.nonzero(bits)[0], np.nonzero(zero)[0])
        for c, r in enumerate(per_chain):
            if r is not None:
                _same_chain(g, c, r, 0)
    else:
        assert g["rc"] == 0, g["msg"]
        assert not any(s.error_flags for s in g["stats"])
        for c in range(CHAINS):
            _same_chain(g, c, ref, c)


@pytest.mark.parametrize("backend", [abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP], ids=["tpc", "wpc"])
@pytest.mark.parametrize("case", list(CASES))
def test_divergent_cases_bit_identical_on_the_device(case, backend):
    _check_case(case, backend)


@pytest.mark.parametrize("env", [{"RN_WPC_K": "2"}, {"RN_WPC_PLACE": "1"}], ids=["k2", "place1"])
@pytest.mark.parametrize("case", ["static_funnel_ehmc_40", "nan_region_ehmc_dualavg", "zero_mass_dense_schools"])
def test_divergent_cases_other_warp_shapes(case, env):
    _check_case(case, abi.RN_BACKEND_WARP, env)


# ---- streamed shapes: the same regimes, summation order of the row sums differs from the oracle's ----
# name -> (model, environment, chains, text the emitted source must contain, text it must not contain).  The regression keeps
# its rows streamed (RN_INLINE=0): device-side inlining would turn it into a data-free polynomial and no row path would run.
_DMMA = "rn_dmma(z"
STREAMED = {
    "logreg_rows": (lambda: configs.logreg(300, 3), {"RN_MMA": "0"}, CHAINS, ["#define RN_WPC_PLACE 0\n"], [_DMMA]),
    "logreg_dmma": (lambda: configs.logreg(1500, 6), {}, CHAINS, [_DMMA], []),
    "logreg_dmma_ragged": (lambda: configs.logreg(1500, 6), {}, 13, [_DMMA], []),
    "linreg5_dmma": (lambda: configs.linreg(900, covariates=5), {"RN_INLINE": "0"}, CHAINS, [_DMMA], []),
    "poisson_glmm_scatter": (lambda: configs.poisson_glm(20, 2000), {}, CHAINS, ["rn_scatter_add("], []),
    "logreg_place1_tma0": (lambda: configs.logreg(300, 3), {"RN_MMA": "0", "RN_WPC_PLACE": "1", "RN_TMA": "0"}, CHAINS,
                           ["#define RN_WPC_PLACE 1\n", "#define RN_TMA_STAGES 0\n"], [_DMMA]),
    "logreg_place1_tma2": (lambda: configs.logreg(300, 3), {"RN_MMA": "0", "RN_WPC_PLACE": "1", "RN_TMA": "2"}, CHAINS,
                           ["#define RN_WPC_PLACE 1\n", "#define RN_TMA_STAGES 2\n"], [_DMMA]),
}


@pytest.mark.parametrize("regime", ["static_3", "static_40", "dualavg"])
@pytest.mark.parametrize("name", list(STREAMED))
def test_streamed_shapes_in_divergent_regimes(name, regime):
    build, env, chains, must, must_not = STREAMED[name]
    model = build()
    rir, cols = model.compile(True)
    prir, pcols = model.compile(False)
    if regime == "dualavg":  # some chains diverge during the step-size search and the first iterations
        config = api.make_config(6, 10, sampler=api.HMCSampler(4), stepSizeTuner=api.DualAvgTuner(0.3),
                                 massMatrixTuner=api.IdentityMassMatrixTuner(), backend=abi.RN_BACKEND_WARP)
    else:
        config = api.make_config(6, 0, sampler=api.HMCSampler(4), stepSizeTuner=api.StaticStepSize(float(regime[7:])),
                                 massMatrixTuner=api.IdentityMassMatrixTuner(), backend=abi.RN_BACKEND_WARP)
    cfg, keep = api.lower_config(config)
    seeds = spread_seeds(chains, 3)
    ref = OracleModel(rir, cols).sample(cfg, seeds=seeds, trace=True)
    got = classes(ref["trace"])
    assert {"-inf", "stuck"} <= got if regime != "dualavg" else "-inf" in got, got
    g = _device_run(prir, pcols, config, seeds, env)
    assert g["rc"] == 0, g["msg"]
    assert all(t in g["src"] for t in must) and not any(t in g["src"] for t in must_not), "%s: not the path named" % name
    for c in range(chains):
        _same_chain(g, c, ref, c, exact=False, tol=1e-6 if regime == "dualavg" else 1e-9)


def test_fast_math_in_divergent_regimes():
    """RN_MATH_FAST (FMA contraction, CUDA libm): same decisions, step counts and RNG states as the oracle; log-accepts only
    where the energies stay far from overflow"""
    for case in ("static_funnel_hmc_3", "static_schools_ehmc_40", "nan_region_ehmc_dualavg"):
        rir, cols, config, cfg, seeds, ref = oracle_run(case, CHAINS)
        config.mathMode = abi.RN_MATH_FAST
        g = _device_run(rir, cols, config, seeds)
        assert g["rc"] == 0, g["msg"]
        for c in range(CHAINS):
            _same_chain(g, c, ref, c, exact=False, tol=1e-6, huge=1e30)


# ---- pooled adaptation with chains whose step-size search collapsed to 0.0 and that never accept ----
@pytest.mark.parametrize("mass", ["identity", "diagonal", "dense"])
@pytest.mark.parametrize("backend", [abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP], ids=["tpc", "wpc"])
def test_pooled_adaptation_with_stuck_chains(backend, mass):
    tuner = {"identity": api.IdentityMassMatrixTuner(), "diagonal": api.DiagonalMassMatrixTuner(8, 1.5, 2, 2),
             "dense": api.DenseMassMatrixTuner(8, 1.5, 2, 2)}[mass]
    config = api.make_config(6, 24, sampler=api.HMCSampler(3), stepSizeTuner=api.DualAvgTuner(0.8), massMatrixTuner=tuner,
                             backend=backend)
    config.stepAdaptation = abi.RN_ADAPT_POOLED
    if mass != "identity":
        config.adaptation = abi.RN_ADAPT_POOLED
    rir, cols = nan_model().compile(True)
    cfg, keep = api.lower_config(config)
    seeds = spread_seeds(CHAINS, 1)
    ref = (pd if mass == "dense" else ps).oracle_sample(rir, cols, cfg, seeds, **({} if mass == "dense" else {"dense_mass": False}))
    got = classes(ref["trace"])
    assert {"-inf", "stuck", "moving"} <= got, got
    # the edges: chains whose findReasonableStepSize ends at 0.0 enter the pooled initial step with log2Step at the bottom of
    # its range, which pulls the shared step far below any a finite start gives; and warmup iterations with log-accepts of
    # -inf add the acceptance quantum of p = 0 to the pooled sum
    assert 0.0 < ref["trace"][0, 0, 2] < 1e-100, ref["trace"][0, 0, 2]
    assert np.isneginf(ref["trace"][:, : cfg.warmup_iterations, 0]).any()
    g = _device_run(rir, cols, config, seeds)
    assert g["rc"] == 0, g["msg"]
    for c in range(CHAINS):
        _same_chain(g, c, ref, c)


# ---- tracked diagnostics over runs with chains that never move (zero within-chain variance) ----
@pytest.mark.parametrize("thin", [1, 3])
@pytest.mark.parametrize("case", ["nan_region_hmc_dualavg", "nan_region_ehmc_dualavg", "static_funnel_hmc_40"])
def test_tracked_diagnostics_over_stuck_chains(case, thin):
    """Equal to the restatement of Trace.diagnostics over the drawn samples, with one agreed difference: a parameter that no
    chain moves has a within-chain variance of exactly 0.0, which the device's Welford sums keep exactly (rHat = sqrt(v / 0)
    = +inf), while the restatement's two-pass variance around sum / n is rounding noise (rHat ~1e15).  Where every chain is
    constant the device's rHat is +inf and the restatement's is beyond 1e12; the effective sample size is the restatement's
    there too (the variograms are exactly 0.0 either way)."""
    rir, cols, config, cfg, seeds, ref = oracle_run(case, CHAINS)
    config.iterations = 30
    cfg, keep = api.lower_config(config)
    g = _device_run(rir, cols, config, seeds, track_thin=thin)
    draws = g["samples"][:, ::thin]
    constant = (np.ptp(draws, axis=1) == 0)  # [chains][n]
    assert constant.any(axis=1).any(), "some chains must never move"
    want = np.array(trace_diagnostics(draws))
    got = g["diag"]
    frozen = constant.all(axis=0)  # parameters that no chain moves
    if case.startswith("static_"):
        assert frozen.all(), "no chain moves at this step size"
    assert (got[frozen, 0] == np.inf).all() and (want[frozen, 0] > 1e12).all(), (got[frozen], want[frozen])
    want[frozen, 0] = np.inf
    for cls in (np.isnan, np.isposinf, np.isneginf, np.isfinite):
        assert np.array_equal(cls(got), cls(want)), (got, want)
    fin = np.isfinite(want)
    assert parity.rel_err(got[fin], want[fin], 1e-9) < 1e-9, (got, want)


# ---- density_batch at the positions these trajectories reach ----
def _nonfinite_inputs(n, rng):
    """rows whose value / gradient class does not depend on the order of summation: one infinite or NaN coordinate among
    finite ones, opposite infinities, coordinates of +-1e200 that overflow products, and plain finite rows"""
    rows = [rng.normal(size=n) * 0.3 for _ in range(4)]
    for v in (np.inf, -np.inf, np.nan, 1e200, -1e200):
        for i in (0, n - 1):
            r = rng.normal(size=n) * 0.3
            r[i] = v
            rows.append(r)
    r = rng.normal(size=n) * 0.3
    r[0], r[n - 1] = np.inf, -np.inf
    rows.append(r)
    return np.array(rows)


def _sigma_underflow(q):
    """(d/dq0 at rows where exp(q0) == 0.0) of the regression, whose sigma = exp(q0): the reference's algebra multiplies the
    chain rule's factors as one product of powers, sigma^-3 * sigma = sigma^-2 = +inf, while the adjoint of the primal program
    (what the device differentiates) takes the chain rule factor by factor, sigma^-3 = +inf times d sigma / d q0 = 0.0, which
    is NaN.  Both are the same derivative; only at sigma == 0.0 do the two evaluation orders differ in class."""
    out = np.zeros((q.shape[0], q.shape[1] + 1), dtype=bool)
    with np.errstate(over="ignore"):
        out[:, 1] = np.exp(q[:, 0]) == 0.0
    return out


# path -> (model, environment, differentiate the primal program on the device, entries left out).  density_batch runs
# rn_k_density: the thread-per-chain kernel or the per-warp rows of the warp-per-chain kernel -- also for a model whose sampler
# takes the chain-batched DMMA path, which only the sampler launches (the DMMA path at non-finite positions is reached through
# test_streamed_shapes_in_divergent_regimes).  The regression keeps its rows streamed (RN_INLINE=0); inlined, its density is a
# data-free polynomial of expanded sums (sum y^2 - 2 beta sum x y + ...), which is NaN where the streamed form is -inf.
DENSITY_PATHS = {
    "tpc_funnel": (lambda: configs.funnel(10), {"RN_BACKEND": "0"}, False, None),
    "wpc_funnel": (lambda: configs.funnel(10), {"RN_BACKEND": "1"}, False, None),
    "wpc_place1_schools": (lambda: configs.eight_schools(), {"RN_BACKEND": "1", "RN_WPC_PLACE": "1"}, False, None),
    "tpc_nan_model": (nan_model, {"RN_BACKEND": "0"}, False, None),
    "wpc_rows_logreg": (lambda: configs.logreg(300, 3), {"RN_BACKEND": "1", "RN_MMA": "0"}, True, None),
    "wpc_rows_logreg_ragged_tile": (lambda: configs.logreg(1501, 6), {"RN_BACKEND": "1"}, True, None),
    "wpc_rows_linreg5_streamed": (lambda: configs.linreg(903, covariates=5), {"RN_BACKEND": "1", "RN_INLINE": "0"}, True,
                                  _sigma_underflow),
    "wpc_poisson_glmm": (lambda: configs.poisson_glm(20, 2000), {"RN_BACKEND": "1"}, True, None),
    "wpc_place1_logreg": (lambda: configs.logreg(300, 3), {"RN_BACKEND": "1", "RN_MMA": "0", "RN_WPC_PLACE": "1"}, True, None),
}


@pytest.mark.parametrize("path", list(DENSITY_PATHS))
def test_density_batch_classes_at_nonfinite_positions(path):
    build, env, primal, left_out = DENSITY_PATHS[path]
    model = build()
    rir, cols = model.compile(True)
    grir, gcols = model.compile(False) if primal else (rir, cols)
    om = OracleModel(rir, cols)
    q = _nonfinite_inputs(om.n, np.random.default_rng(5))
    ref = om.density_batch(q)
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        m = api.CudaModel(grir, gcols, device=0)
        got = m.density_batch(q)
        m.close()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    skip = left_out(q) if left_out is not None else np.zeros(ref.shape, dtype=bool)
    assert skip.sum() <= 2, "only the rows whose sigma underflows are left out"
    assert np.isnan(got[skip]).all() and np.isposinf(ref[skip]).all(), "the evaluation-order difference _sigma_underflow describes"
    for name, cls in (("NaN", np.isnan), ("+inf", np.isposinf), ("-inf", np.isneginf), ("finite", np.isfinite)):
        bad = np.argwhere((cls(got) != cls(ref)) & ~skip)
        assert bad.size == 0, "%s class differs at (row, column) %s: device %s, oracle %s" % (
            name, bad[:4].tolist(), got[tuple(bad[0])], ref[tuple(bad[0])])
    fin = np.isfinite(ref) & ~skip
    assert parity.rel_err(got[fin], ref[fin], 1e-9) < 1e-9
    assert not np.isfinite(ref).all(), "the inputs must reach non-finite values"

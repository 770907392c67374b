"""The sampler source through divergent and non-finite trajectories, on the host (tests/host_emulation.py), bit for bit against
the oracle.  Every other parity test stays in a stable regime; these cases drive the branches LeapFrog.scala defines for the
unstable one:

- logAcceptanceProb (rn_log_accept): a NaN deltaH gives -inf, a deltaH of -inf gives 0;
- isUTurn: a NaN dot product counts as a U-turn;
- findReasonableStepSize halves towards 0.0 from a start point whose density is NaN, and DualAvg carries on from there;
- a rejection restores q, gradient and potential, so that a non-finite proposal never leaks into the next iteration;
- require(!elements.contains(0.0)) on an adapted mass matrix, for the chains that never accept during a window.

The case table is shared with tests/test_gpu_divergence.py.  Each case names the log-accept classes and chain classes it must
produce, so that a case cannot drift back into the stable regime unnoticed."""
import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.binding import OracleError, OracleModel
from oracle.rainier_py.compute import Real
from oracle.rainier_py.core import Model
from rainier_b200 import abi, api

import host_emulation as he

MASS_ZERO = "requirement failed: adapted mass matrix contains 0.0 (MassMatrix.scala:8,16)"


def spread_seeds(count, key=1):
    """Seeds far apart: java.util.Random's first gaussians of consecutive seeds are close, so seeds 1, 2, 3, ... would start
    every chain at nearly the same point."""
    return np.random.default_rng(key).integers(1, 2 ** 47, size=count)


def nan_model():
    """log-density sqrt(t0) + log(t0) - t1^2 / 2: density and gradient are NaN on the half-space t0 < 0 (sqrt's derivative),
    the density is -inf at t0 = 0.  About half of the spread start points lie in the NaN region."""
    return Model.track_(list(Real.parameters(2, lambda t: t[0].pow(0.5) + t[0].log() - t[1] * t[1] * 0.5)))


def _static(sampler, step, iterations=8):
    return api.make_config(iterations, 0, sampler=sampler, stepSizeTuner=api.StaticStepSize(step),
                           massMatrixTuner=api.IdentityMassMatrixTuner())


def _dual_avg(sampler, delta=0.8, warmup=24, iterations=6, mass=None):
    return api.make_config(iterations, warmup, sampler=sampler, stepSizeTuner=api.DualAvgTuner(delta),
                           massMatrixTuner=mass if mass is not None else api.IdentityMassMatrixTuner())


# id -> (model factory, config factory, seeds key, classes the oracle's run must contain, dense mass)
# log-accept classes: "-inf" (NaN or +inf deltaH), "0" (deltaH <= 0), "neg" (finite and negative); chain classes: "stuck" (never
# accepts), "moving" (accepts at least once), "zero_mass" (an adapted mass matrix contains 0.0 on some chains, not all).  No
# chain of the funnel or eight schools accepts at a static step of 3 or more, so the static cases are all-rejected by design;
# divergent chains run beside accepting chains in the same warp or CTA in the NaN-region and zero-mass cases, where the start
# point of each seed decides which kind a chain is.
CASES = {}
for _mname, _model in (("funnel", lambda: configs.funnel(10)), ("schools", configs.eight_schools)):
    for _sname, _sampler in (("hmc", lambda: api.HMCSampler(8)), ("ehmc", lambda: api.EHMCSampler(30, 2))):
        for _step in (3.0, 40.0, 1e3):
            _want = {"stuck"}
            if _sname == "hmc":
                _want.add("-inf")
            if _sname == "ehmc" or (_mname == "funnel" and _step == 3.0):
                _want.add("neg")
            if _mname == "funnel" and _sname == "ehmc" and _step > 3.0:
                _want.add("-inf")
            CASES["static_%s_%s_%g" % (_mname, _sname, _step)] = (
                _model, (lambda s=_sampler, st=_step: _static(s(), st)), 1, _want, False)
CASES["nan_region_hmc_dualavg"] = (nan_model, lambda: _dual_avg(api.HMCSampler(3)), 1, {"-inf", "0", "neg", "stuck", "moving"}, False)
CASES["nan_region_ehmc_dualavg"] = (nan_model, lambda: _dual_avg(api.EHMCSampler(10, 2)), 1, {"-inf", "0", "neg", "stuck", "moving"},
                                    False)
for _mname, _model in (("funnel", lambda: configs.funnel(10)), ("schools", configs.eight_schools)):
    CASES["zero_mass_diag_%s" % _mname] = (
        _model, lambda: _dual_avg(api.HMCSampler(8), 0.2, 24, 4, api.DiagonalMassMatrixTuner(8, 1.5, 2, 2)), 2,
        {"-inf", "neg", "moving", "zero_mass"}, False)
    CASES["zero_mass_dense_%s" % _mname] = (
        _model, lambda: _dual_avg(api.HMCSampler(8), 0.2, 24, 4, api.DenseMassMatrixTuner(8, 1.5, 2, 2)), 2,
        {"-inf", "neg", "moving", "zero_mass"}, True)


def classes(trace, zero_mass=None):
    """The classes a trace [chains][iterations][4] contains (see CASES)."""
    la, acc = trace[:, :, 0], trace[:, :, 1].sum(axis=1)
    out = set()
    if np.isneginf(la).any():
        out.add("-inf")
    if (la == 0.0).any():
        out.add("0")
    if (np.isfinite(la) & (la < 0.0)).any():
        out.add("neg")
    if (acc == 0).any():
        out.add("stuck")
    if (acc > 0).any():
        out.add("moving")
    if zero_mass is not None and zero_mass.any() and not zero_mass.all():
        out.add("zero_mass")
    return out


def oracle_by_chain(rir, cols, cfg, seeds, dense):
    """The oracle run one chain at a time (a failed requirement fails the whole call).  Returns (zero_mass [chains] bool,
    results of every chain, None where the requirement failed)."""
    om = OracleModel(rir, cols)
    failed, results = [], []
    for s in seeds:
        try:
            results.append(om.sample(cfg, seeds=[s], trace=True, dense_mass=dense))
            failed.append(False)
        except OracleError as e:
            assert str(e) == MASS_ZERO
            results.append(None)
            failed.append(True)
    return np.array(failed), results


def oracle_run(case, count):
    """(rir, cols, config, lowered cfg, seeds, reference) of a case; the reference is the oracle's run of all chains, or, for
    the zero-mass cases, (zero_mass, per-chain results)."""
    model_f, config_f, key, want, dense = CASES[case]
    rir, cols = model_f().compile(True)
    config = config_f()
    cfg, keep = api.lower_config(config)
    seeds = spread_seeds(count, key)
    if "zero_mass" in want:
        zero, per_chain = oracle_by_chain(rir, cols, cfg, seeds, dense)
        got = classes(np.concatenate([r["trace"] for r in per_chain if r is not None]), zero)
        assert want <= got, "%s: the oracle's run lacks %s" % (case, sorted(want - got))
        ref = (zero, per_chain)
    else:
        ref = OracleModel(rir, cols).sample(cfg, seeds=seeds, trace=True, dense_mass=dense)
        got = classes(ref["trace"])
        assert want <= got, "%s: the oracle's run lacks %s" % (case, sorted(want - got))
    return rir, cols, config, cfg, seeds, ref


# kernel shapes of the host emulation: thread per chain; warp per chain with 1 or 4 chains per CTA, 1 or 2 warps per chain,
# the chain state in shared memory (placement 0) or in global memory (placement 1)
SHAPES = {
    "tpc": None,
    "wpc_k1_cta1": dict(k="1", cpc=1, place=None),
    "wpc_k2_cta4": dict(k="2", cpc=4, place=None),
    "wpc_k1_cta4_place1": dict(k="1", cpc=4, place="1"),
}


def _emit(monkeypatch, rir, cols, config, shape):
    sh = SHAPES[shape]
    config.backend = abi.RN_BACKEND_THREAD if sh is None else abi.RN_BACKEND_WARP
    if sh is not None:
        monkeypatch.setenv("RN_TMA", "0")
        monkeypatch.setenv("RN_WPC_K", sh["k"])
        if sh["place"] is not None:
            monkeypatch.setenv("RN_WPC_PLACE", sh["place"])
    cm = api.CudaModel(rir, cols, device=-1)
    src = cm.emit_source(config)
    for v in ("RN_TMA", "RN_WPC_K", "RN_WPC_PLACE"):
        monkeypatch.delenv(v, raising=False)
    if sh is not None:
        assert "#define RN_BACKEND 1" in src and ("#define RN_WPC_K %s\n" % sh["k"]) in src
        if sh["place"] is not None:
            assert ("#define RN_WPC_PLACE %s\n" % sh["place"]) in src
    return cm, src, 1 if sh is None else sh["cpc"]


def assert_chain_equal(got, c, ref, rc=0, what=""):
    """chain c of the emulated run equals chain rc of an oracle result bit for bit: trace (log-accept, decision, step size,
    steps), samples, stats, RNG state and mass"""
    assert np.array_equal(got["trace"][c], ref["trace"][rc], equal_nan=True), "%strace of chain %d differs" % (what, c)
    assert np.array_equal(got["samples"][c], ref["samples"][rc], equal_nan=True), "%ssamples of chain %d differ" % (what, c)
    o = ref["stats"][rc]
    assert got["stats"][c, 0] == o.gradient_evaluations and got["stats"][c, 1] == o.leapfrog_steps, "%sstats of chain %d" % (what, c)
    assert got["stats"][c, 2] == o.accepted and got["stats"][c, 3] == o.rng.seed48, "%saccepts / RNG of chain %d" % (what, c)
    assert np.array_equal(got["mass"][c], ref["mass"][rc], equal_nan=True), "%smass of chain %d differs" % (what, c)


# every case on the thread-per-chain source; the warp-per-chain shapes (32 or 64 host threads per chain) run one static step
# of each model and sampler
PAIRS = [(c, s) for c in CASES for s in SHAPES if s == "tpc" or not c.startswith("static_") or c.endswith("_40")]


@pytest.mark.parametrize("case,shape", PAIRS)
def test_divergent_trajectories_match_the_oracle_bit_for_bit(case, shape, monkeypatch):
    count = 8
    rir, cols, config, cfg, seeds, ref = oracle_run(case, count)
    cm, src, cpc = _emit(monkeypatch, rir, cols, config, shape)
    got = he.sample(src, cfg, seeds, cm, chains_per_cta=cpc)
    if isinstance(ref, tuple):
        zero, per_chain = ref
        assert np.array_equal((got["stats"][:, 4] & 2) != 0, zero), "chains with error bit 2: %s, oracle: %s" % (
            np.nonzero(got["stats"][:, 4] & 2)[0], np.nonzero(zero)[0])
        for c, r in enumerate(per_chain):
            if r is not None:
                assert_chain_equal(got, c, r)
    else:
        assert not got["stats"][:, 4].any()
        for c in range(count):
            assert_chain_equal(got, c, ref, c)


def test_nan_region_is_reached_and_step_size_search_collapses():
    """The NaN model's evidence: start points where the density and gradient are NaN, NaN densities at the positions those
    chains hold while sampling, step sizes that findReasonableStepSize halved to exactly 0.0, and, under EHMC, chains at step 0 whose
    counted trajectories stop at l = 1 (the NaN momentum makes isUTurn's dot product NaN) instead of running to maxSteps."""
    rir, cols, config, cfg, seeds, ref = oracle_run("nan_region_ehmc_dualavg", 8)
    om = OracleModel(rir, cols)
    start = om.density_batch(_start_points(rir, cols, seeds))
    nan_start = np.isnan(start[:, 0])
    assert nan_start.any() and not nan_start.all()
    assert np.isnan(start[nan_start, 1]).all()  # d/dt0
    tr = ref["trace"]
    assert np.array_equal(tr[:, 0, 2] == 0.0, nan_start), "exactly the chains that start in the NaN region search down to 0.0"
    assert (tr[nan_start, :, 1] == 0).all()
    # warmup, every trajectory counted: a chain at step 0 turns after one step (NaN dot product), then takes minSteps - 1 = 1
    # more; sampling draws its lengths from the ring of those counts (l = 1)
    warm = cfg.warmup_iterations
    assert (tr[nan_start, :warm, 3] == 2).all() and (tr[nan_start, warm:, 3] == 1).all()
    # the positions the chains hold while sampling: NaN density exactly on the chains that started in the NaN region
    held = om.density_batch(ref["samples"].reshape(-1, 2))[:, 0].reshape(len(seeds), -1)
    assert np.array_equal(np.isnan(held).all(axis=1), nan_start) and np.isfinite(held[~nan_start]).all()


def _start_points(rir, cols, seeds):
    """LeapFrog.initialize's q of each seed: a static step of 0 keeps every chain where it started"""
    cfg, keep = api.lower_config(_static(api.HMCSampler(1), 0.0, iterations=1))
    return OracleModel(rir, cols).sample(cfg, seeds=seeds)["samples"][:, 0, :]

"""Pooled mass-matrix windows (rn_config.adaptation = RN_ADAPT_POOLED) on the host: the lockstep oracle's window masses
against the reduction restated in the kernels' order over the oracle's own warmup draws, against the exact pooled variance
of those draws, and against the per-chain oracle where one chain makes the pooled formula the reference's; the restated
reduction over several emulated ranks.  The device side is tests/test_gpu_pooled_mass.py."""
from fractions import Fraction

import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.binding import OracleModel
from rainier_b200 import abi, api

import pooled_step as ps


def _cfg(it, warm, sampler, step, mass, **kw):
    return api.make_config(iterations=it, warmupIterations=warm, sampler=sampler, stepSizeTuner=step, massMatrixTuner=mass,
                           adaptation=abi.RN_ADAPT_POOLED, **kw)


def _dist(a, b):
    """|a - b| for a float and a Fraction, as a float (exact up to the final rounding)"""
    return abs(float(Fraction(a) - b))


def _check_windows(model, config, seeds):
    """every window the oracle closed: its pooled variance == the restated reduction over its draws, bit for bit, and
    within the first-order bound of the exact pooled variance of those draws"""
    rir, cols = model.compile(True)
    cfg, keep = api.lower_config(config)
    ref = ps.oracle_sample(rir, cols, cfg, seeds)
    wins = ps.windows(cfg)
    assert len(wins) >= 2 and len(ref["window_mass"]) == len(wins)
    for w, idx in enumerate(wins):
        draws = ref["warm_draws"][:, idx, :]
        mean, m2 = ps.welford_restated(draws)
        _, var, _ = ps.pool_reduce_restated(mean, m2, len(idx))
        assert np.array_equal(var, ref["window_mass"][w]), "window %d: oracle's pooled variance differs from the restatement" % w
        bound = ps.window_variance_bound(draws)
        exact = ps.pooled_variance_exact(draws)
        for i in range(len(var)):
            assert _dist(var[i], exact[i]) <= bound[i], "window %d, parameter %d: %r vs exact %r (bound %g)" % (w, i, var[i], float(exact[i]), bound[i])
    assert np.all(ref["mass"] == ref["window_mass"][-1]), "chains do not end warmup with the last window's pooled matrix"
    return ref


def test_eight_schools_default_config_per_chain_steps():
    """EHMC + per-chain DualAvg + windows 50/1.5/50/50 (every chain restarts DualAvg from its own logStepSizeBar)"""
    ref = _check_windows(configs.eight_schools(), api.SamplerConfig(iterations=5, warmupIterations=300, adaptation=abi.RN_ADAPT_POOLED),
                         np.arange(20) + 3)
    assert len(set(ref["trace"][:, 0, 2])) > 1, "per-chain steps should start from different step sizes"


def test_funnel_static_step_many_chains():
    """StaticStepSize, 300 chains: the reduction's thread-to-chain stride wraps past 256"""
    _check_windows(configs.funnel(), _cfg(5, 90, api.HMCSampler(5), api.StaticStepSize(0.2), api.DiagonalMassMatrixTuner(15, 1.5, 10, 10)),
                   np.arange(300) + 1)


def test_funnel_pooled_steps_and_pooled_mass():
    config = _cfg(5, 100, api.HMCSampler(5), api.DualAvgTuner(0.8), api.DiagonalMassMatrixTuner(10, 2.0, 5, 5),
                  stepAdaptation=abi.RN_ADAPT_POOLED)
    ref = _check_windows(configs.funnel(), config, np.arange(40) + 17)
    assert np.all(ref["trace"][:, :, 2] == ref["trace"][:1, :, 2])


def test_first_window_of_one_length():
    """a first window of one draw per chain: no within-chain term, the variance is the spread of the chains' positions"""
    _check_windows(configs.funnel(), _cfg(5, 40, api.HMCSampler(5), api.DualAvgTuner(0.8), api.DiagonalMassMatrixTuner(1, 2.0, 0, 0)),
                   np.arange(33) + 2)


def test_one_chain_equals_the_per_chain_oracle():
    """with one chain and one window the pooled variance is raw / L, the reference's VarianceEstimator.variance: the lockstep
    oracle's whole run equals the per-chain oracle's bit for bit"""
    config = _cfg(30, 60, api.HMCSampler(5), api.DualAvgTuner(0.8), api.DiagonalMassMatrixTuner(30, 1.5, 10, 20))
    cfg, keep = api.lower_config(config)
    assert len(ps.window_closes(cfg)) == 1
    rir, cols = configs.funnel().compile(True)
    seeds = np.array([77], dtype=np.int64)
    ref = ps.oracle_sample(rir, cols, cfg, seeds)
    per_chain_cfg, keep2 = api.lower_config(config)
    per_chain_cfg.adaptation = abi.RN_ADAPT_PER_CHAIN
    one = OracleModel(rir, cols).sample(per_chain_cfg, seeds=seeds, trace=True)
    assert np.array_equal(ref["mass"], one["mass"])
    assert np.array_equal(ref["window_mass"][0], one["mass"][0])
    assert np.array_equal(ref["samples"], one["samples"])
    assert np.array_equal(ref["trace"], one["trace"])


def _stats(rng, chains, n, L, mean_scale=1.0, spread=1.0):
    mean = mean_scale + rng.normal(size=(chains, n)) * spread
    m2 = rng.gamma(max(L - 1, 1) / 2.0, 2.0, size=(chains, n)) if L > 1 else np.zeros((chains, n))
    return mean, m2


@pytest.mark.parametrize("chains,L", [(7, 3), (300, 50), (1029, 1), (4099, 1687)])
def test_rank_split_stays_within_the_bound(chains, L):
    """R emulated ranks change the summation order only: each split is within its bound of the exact value"""
    mean, m2 = _stats(np.random.default_rng(chains), chains, 3, L, mean_scale=4.0)
    exact = ps.pooled_variance_exact_stats(mean, m2, L)
    _, one, _ = ps.pool_reduce_restated(mean, m2, L, 1)
    for ranks in (1, 2, 3, 8):
        pool, var, _ = ps.pool_reduce_restated(mean, m2, L, ranks)
        assert pool[0] == chains
        bound = ps.pool_error_bound(mean, m2, L, ranks)
        bound1 = ps.pool_error_bound(mean, m2, L, 1)
        for i in range(3):
            assert _dist(var[i], exact[i]) <= bound[i]
            assert abs(var[i] - one[i]) <= bound[i] + bound1[i]


def test_rank_split_is_exact_where_order_does_not_matter():
    """small integer statistics with an integer pooled mean: every sum is exact, so every split gives the same bits"""
    rng = np.random.default_rng(5)
    chains = 1000
    mean = rng.integers(-50, 50, size=(chains, 2)).astype(np.float64)
    mean[0] -= mean.sum(axis=0) - 3 * chains  # pooled mean exactly 3
    m2 = rng.integers(0, 1000, size=(chains, 2)).astype(np.float64)
    _, one, _ = ps.pool_reduce_restated(mean, m2, 9, 1)
    for ranks in (2, 3, 8):
        _, var, _ = ps.pool_reduce_restated(mean, m2, 9, ranks)
        assert np.array_equal(var, one)
    # the sums are exact, so the one rounding left is the final division: the correctly rounded exact variance
    assert list(one) == [float(e) for e in ps.pooled_variance_exact_stats(mean, m2, 9)]


def test_bound_separates_the_textbook_form():
    """|mean| >> sd: the two-pass form stays within the bound, sum q^2 / N - mean^2 does not"""
    rng = np.random.default_rng(8)
    chains, L = 4099, 50
    mean, m2 = _stats(rng, chains, 2, L, mean_scale=1e8)
    exact = ps.pooled_variance_exact_stats(mean, m2, L)
    _, var, _ = ps.pool_reduce_restated(mean, m2, L)
    bound = ps.pool_error_bound(mean, m2, L)
    s1, s2 = (L * mean).sum(axis=0), (m2 + L * mean * mean).sum(axis=0)
    tb = ps.textbook_variance(s1, s2, float(chains * L))
    for i in range(2):
        assert _dist(var[i], exact[i]) <= bound[i]
        assert _dist(tb[i], exact[i]) > bound[i], "the bound cannot tell the textbook form apart"


def test_exact_variance_of_draws():
    """pooled_variance_exact against the exact statistics of the same draws, and the bound of the kernels' Welford path"""
    rng = np.random.default_rng(3)
    draws = 1e6 + rng.normal(size=(9, 40, 2))
    exact = ps.pooled_variance_exact(draws)
    ref = np.var(draws.reshape(-1, 2).astype(np.longdouble) - np.longdouble(1e6), axis=0)
    for i in range(2):
        assert abs(float(exact[i]) - float(ref[i])) <= 1e-12 * float(ref[i])
    mean, m2 = ps.welford_restated(draws)
    _, var, _ = ps.pool_reduce_restated(mean, m2, 40)
    bound = ps.window_variance_bound(draws)
    for i in range(2):
        assert _dist(var[i], exact[i]) <= bound[i]

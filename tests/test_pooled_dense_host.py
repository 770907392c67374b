"""Pooled dense mass-matrix windows (DenseMassMatrixTuner with rn_config.adaptation = RN_ADAPT_POOLED) on the host: the
lockstep oracle's window covariances against the reduction restated in the kernels' order over the oracle's own warmup draws
and against the exact pooled covariance of those draws, its factor against the restated Cholesky, the restated reduction
over several emulated ranks, and the host mirror dist.combine_welford_dense.  The device side is
tests/test_gpu_pooled_dense.py."""
from fractions import Fraction

import numpy as np
import pytest

from oracle.rainier_py import configs
from rainier_b200 import abi, api, dist

import pooled_dense as pd
import pooled_step as ps


def _check_windows(model, config, seeds):
    """every window the oracle closed: its pooled covariance == the restated reduction over its draws, bit for bit, and
    every entry within the first-order bound of the exact pooled covariance of those draws"""
    rir, cols = model.compile(True)
    cfg, keep = api.lower_config(config)
    assert cfg.mass_tuner == abi.RN_MASS_DENSE and cfg.adaptation == abi.RN_ADAPT_POOLED
    ref = pd.oracle_sample(rir, cols, cfg, seeds)
    wins = ps.windows(cfg)
    n = ref["warm_draws"].shape[2]
    assert len(wins) >= 2 and len(ref["window_mass"]) == len(wins)
    for w, idx in enumerate(wins):
        draws = ref["warm_draws"][:, idx, :]
        mean, cov = pd.welford_dense_restated(draws)
        _, M, _ = pd.pool_reduce_dense_restated(mean, cov, len(idx))
        assert np.array_equal(M.reshape(-1), ref["window_mass"][w]), "window %d: oracle's pooled covariance differs from the restatement" % w
        bound = pd.window_covariance_bound(draws)
        exact = pd.pooled_covariance_exact(draws)
        for j in range(n):
            for k in range(n):
                assert abs(float(Fraction(M[j, k]) - exact[j][k])) <= bound[j, k], "window %d, entry (%d, %d) outside the bound" % (w, j, k)
    assert np.all(ref["mass"] == ref["window_mass"][-1]), "chains do not end warmup with the last window's pooled matrix"
    return ref


def test_eight_schools_default_config_dense():
    """DefaultConfig (EHMC, per-chain DualAvg, windows 50/1.5/50/50) with the dense tuner"""
    config = api.SamplerConfig(iterations=5, warmupIterations=300, adaptation=abi.RN_ADAPT_POOLED)
    config._massMatrixTuner = api.DenseMassMatrixTuner(50, 1.5, 50, 50)
    _check_windows(configs.eight_schools(), config, np.arange(20) + 3)


def test_funnel_300_chains_dense():
    """StaticStepSize, 300 chains: the reduction's thread-to-chain stride wraps past 256"""
    config = api.make_config(5, 90, sampler=api.HMCSampler(5), stepSizeTuner=api.StaticStepSize(0.2),
                             massMatrixTuner=api.DenseMassMatrixTuner(15, 1.5, 10, 10), adaptation=abi.RN_ADAPT_POOLED)
    _check_windows(configs.funnel(), config, np.arange(300) + 1)


def test_funnel_dense_with_pooled_steps():
    config = api.make_config(5, 100, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.DenseMassMatrixTuner(10, 2.0, 5, 5), adaptation=abi.RN_ADAPT_POOLED,
                             stepAdaptation=abi.RN_ADAPT_POOLED)
    ref = _check_windows(configs.funnel(), config, np.arange(40) + 17)
    assert np.all(ref["trace"][:, :, 2] == ref["trace"][:1, :, 2])


def test_oracle_factor_equals_the_restated_cholesky():
    """the factor the oracle gives every chain at each window end of a run equals cholesky_restated's, bit for bit, flag
    included; so do crafted matrices: random SPD ones, a singular one, one with an element 0.0"""
    config = api.make_config(5, 60, sampler=api.HMCSampler(5), stepSizeTuner=api.StaticStepSize(0.2),
                             massMatrixTuner=api.DenseMassMatrixTuner(10, 1.5, 5, 5), adaptation=abi.RN_ADAPT_POOLED)
    rir, cols = configs.funnel().compile(True)
    cfg, keep = api.lower_config(config)
    ref = pd.oracle_sample(rir, cols, cfg, np.arange(30) + 5)
    n = ref["warm_draws"].shape[2]
    mats = [w.reshape(n, n) for w in ref["window_mass"]]
    rng = np.random.default_rng(9)
    for m in (1, 2, 10, 40):
        X = rng.normal(size=(2 * m, m))
        mats.append(X.T @ X / (2 * m) + 0.01 * np.eye(m))
    mats += [np.ones((3, 3)), np.array([[1.0, 0.0], [0.0, 2.0]])]
    for k, M in enumerate(mats):
        upper, bad = pd.oracle_factor(M)
        _, want, want_bad = pd.cholesky_restated(M)
        assert np.array_equal(upper, want, equal_nan=True) and bad == want_bad, "matrix %d" % k
    assert pd.oracle_factor(mats[-2])[1] and pd.oracle_factor(mats[-1])[1]
    assert not any(pd.oracle_factor(M)[1] for M in mats[:-2])


def test_restated_cholesky_matches_the_textbook_factor():
    rng = np.random.default_rng(4)
    for n in (1, 2, 10, 33):
        X = rng.normal(size=(3 * n, n))
        M = X.T @ X / (3 * n) + 0.1 * np.eye(n)
        lower, upper, bad = pd.cholesky_restated(M)
        assert not bad
        Lnp = np.linalg.cholesky(M)
        assert np.allclose(lower, Lnp[np.tril_indices(n)], rtol=1e-12, atol=1e-13)
    Z = np.ones((3, 3))  # rank one: the second pivot is 0 (or rounds below it)
    assert pd.cholesky_restated(Z)[2]
    Y = np.eye(3)
    Y[0, 1] = 0.0
    assert pd.cholesky_restated(Y)[2], "an element 0.0 must set the flag (MassMatrix.scala:16)"


def _stats(rng, chains, n, L, mean_scale=1.0):
    mean = mean_scale + rng.normal(size=(chains, n))
    X = rng.normal(size=(chains, max(L, 1), n))
    cov = np.einsum("cti,ctj->cij", X, X) if L > 1 else np.zeros((chains, n, n))
    return mean, cov


@pytest.mark.parametrize("ranks", [1, 2, 3, 5, 8])
def test_rank_split_matches_the_restatement_where_sums_are_exact(ranks):
    """small integer statistics and an integer pooled mean: every partial sum is exact, so every split over 1-8 emulated
    ranks gives the restatement's bits, and the one rounding left is the final division"""
    rng = np.random.default_rng(11)
    chains, n, L = 777, 4, 9
    mean = rng.integers(-50, 50, size=(chains, n)).astype(np.float64)
    mean[0] -= mean.sum(axis=0) - 2 * chains  # pooled mean exactly 2
    cov = rng.integers(-300, 300, size=(chains, n, n)).astype(np.float64)
    _, one, _ = pd.pool_reduce_dense_restated(mean, cov, L, 1)
    pool, M, local = pd.pool_reduce_dense_restated(mean, cov, L, ranks)
    assert pool[0] == chains and len(local) == ranks
    assert np.array_equal(M, one)
    exact = (cov.sum(axis=0) + L * np.einsum("ci,cj->ij", mean - 2.0, mean - 2.0)) / (chains * L)
    assert np.array_equal(M, exact)


@pytest.mark.parametrize("chains,L", [(7, 3), (300, 50), (1029, 1), (4099, 20)])
def test_rank_split_stays_within_the_bound(chains, L):
    rng = np.random.default_rng(chains)
    mean, cov = _stats(rng, chains, 3, L, mean_scale=4.0)
    _, one, _ = pd.pool_reduce_dense_restated(mean, cov, L, 1)
    b1 = pd.pool_dense_error_bound(mean, cov, L, 1)
    for ranks in (2, 3, 8):
        _, M, _ = pd.pool_reduce_dense_restated(mean, cov, L, ranks)
        b = pd.pool_dense_error_bound(mean, cov, L, ranks)
        assert np.all(np.abs(M - one) <= b + b1)


def test_diagonal_of_the_dense_reduction_is_the_diagonal_reduction():
    """the diagonal of M is bit for bit the pooled diagonal tuner's variance for the same statistics"""
    rng = np.random.default_rng(2)
    draws = 3.0 + rng.normal(size=(513, 17, 5))
    mean, cov = pd.welford_dense_restated(draws)
    m, m2 = ps.welford_restated(draws)
    assert np.array_equal(mean, m) and np.array_equal(np.einsum("cii->ci", cov), m2)
    for ranks in (1, 3):
        _, M, _ = pd.pool_reduce_dense_restated(mean, cov, 17, ranks)
        _, var, _ = ps.pool_reduce_restated(m, m2, 17, ranks)
        assert np.array_equal(np.diag(M), var)


def test_exact_covariance_of_draws_and_the_bound():
    rng = np.random.default_rng(3)
    draws = 1e6 + rng.normal(size=(9, 40, 3)) @ np.array([[1.0, 0.5, 0.0], [0.0, 1.0, 0.3], [0.0, 0.0, 2.0]])
    exact = pd.pooled_covariance_exact(draws)
    x = draws.reshape(-1, 3).astype(np.longdouble) - np.longdouble(1e6)
    ref = np.cov(x.T.astype(np.float64), bias=True)
    for j in range(3):
        for k in range(3):
            assert abs(float(exact[j][k]) - ref[j, k]) <= 1e-9 * abs(ref[j, j])
    mean, cov = pd.welford_dense_restated(draws)
    _, M, _ = pd.pool_reduce_dense_restated(mean, cov, 40)
    bound = pd.window_covariance_bound(draws)
    for j in range(3):
        for k in range(3):
            assert abs(float(Fraction(M[j, k]) - exact[j][k])) <= bound[j, k]


def test_combine_welford_dense_is_the_pooled_covariance():
    rng = np.random.default_rng(6)
    draws = rng.normal(size=(12, 25, 4))
    mean, cov = pd.welford_dense_restated(draws)
    M = dist.combine_welford_dense(25, mean, cov)
    assert np.allclose(M, np.cov(draws.reshape(-1, 4).T, bias=True), rtol=1e-12, atol=1e-14)
    assert np.allclose(np.diag(M), dist.combine_welford(25, mean, np.einsum("cii->ci", cov)), rtol=1e-14)

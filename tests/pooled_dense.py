"""
Test infrastructure for pooled dense mass windows (DenseMassMatrixTuner with rn_config.adaptation == RN_ADAPT_POOLED): the
dense lockstep oracle (tests/pooled_dense_oracle.cpp, built on tests/pooled_step_oracle.cpp and the per-chain oracle) and the
pooled window covariance three ways: the kernels' summation order restated in float64 (`pool_reduce_dense_restated`,
`cholesky_restated` for the factor), exactly in rationals (`pooled_covariance_exact`), and a first-order bound on the
distance between the two (`pool_dense_error_bound`, `welford_dense_error_bound`).  Shares the diagonal mode's helpers in
tests/pooled_step.py.  None of it is part of the product.
"""
import ctypes as C
import hashlib
import os
import subprocess
from fractions import Fraction

import numpy as np

from oracle.rainier_py.cachedir import private_dir
from rainier_b200.abi import ChainStats, Config

from pooled_step import POOL_THREADS, U, _block_sum, _dyadic, _scale, window_closes

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_ORACLE = None


def _oracle_lib():
    global _ORACLE
    if _ORACLE is None:
        srcs = [os.path.join(_HERE, "pooled_dense_oracle.cpp"), os.path.join(_HERE, "pooled_step_oracle.cpp"),
                os.path.join(_ROOT, "oracle", "rainier_oracle.cpp"), os.path.join(_ROOT, "oracle", "jmath.h"),
                os.path.join(_ROOT, "include", "rainier_cuda.h"), os.path.join(_ROOT, "include", "rainier_rir.h")]
        key = hashlib.sha1(b"".join(open(p, "rb").read() for p in srcs)).hexdigest()[:16]
        so = os.path.join(private_dir("rno_pooled_dense"), key + ".so")
        if not os.path.exists(so):
            tmp = so + ".tmp%d" % os.getpid()
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread", "-w", "-shared",
                            "-o", tmp, srcs[0], "-ldl"], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.rno_last_error.restype = C.c_char_p
        L.rno_model_create.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int, C.c_int,
                                       C.POINTER(C.c_void_p)]
        L.rno_model_destroy.argtypes = [C.c_void_p]
        L.rno_model_nvars.argtypes = [C.c_void_p]
        L.rno_sample_pooled_dense.argtypes = [C.c_void_p, C.POINTER(Config), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p]
        L.rno_pooled_dense_factor.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _ORACLE = L
    return _ORACLE


def oracle_sample(rir, cols, cfg, seeds):
    """the dense lockstep oracle: dict(samples [chains][iters][n], mass [chains][n * n], stats (rn_chain_stats), trace
    [chains][warm+iters][4], warm_draws [chains][warmup][n] = the position after every warmup iteration, window_mass
    [windows][n * n] = the pooled covariance of every closed window)"""
    L = _oracle_lib()
    cols = [np.ascontiguousarray(c, dtype=np.float64) for c in cols]
    ptrs = (C.c_void_p * max(len(cols), 1))(*[c.ctypes.data for c in cols])
    rows = (C.c_int64 * max(len(cols), 1))(*[len(c) for c in cols])
    h = C.c_void_p()
    rir = bytes(rir)
    if L.rno_model_create(rir, len(rir), ptrs, rows, len(cols), 0, C.byref(h)) != 0:
        raise RuntimeError(L.rno_last_error().decode())
    try:
        n = L.rno_model_nvars(h)
        seeds = np.ascontiguousarray(seeds, dtype=np.int64)
        chains = len(seeds)
        samples = np.zeros((chains, cfg.iterations, n))
        mass = np.zeros((chains, n * n))
        stats = (ChainStats * chains)()
        trace = np.zeros((chains, cfg.warmup_iterations + cfg.iterations, 4))
        warm = np.zeros((chains, cfg.warmup_iterations, n))
        win = np.zeros((max(len(window_closes(cfg)), 1), n * n))
        cfg.rng_states = None
        if L.rno_sample_pooled_dense(h, C.byref(cfg), seeds.ctypes.data, chains, samples.ctypes.data, mass.ctypes.data,
                                     C.cast(stats, C.c_void_p), trace.ctypes.data, warm.ctypes.data, win.ctypes.data) != 0:
            raise RuntimeError(L.rno_last_error().decode())
    finally:
        L.rno_model_destroy(h)
    return {"samples": samples, "mass": mass, "stats": stats, "trace": trace, "warm_draws": warm,
            "window_mass": win[:len(window_closes(cfg))]}


def oracle_factor(M):
    """the factor the dense lockstep oracle gives every chain for the pooled matrix M [n][n]: (upper [n(n+1)/2], flag)"""
    L = _oracle_lib()
    M = np.ascontiguousarray(M, dtype=np.float64)
    n = M.shape[0]
    upper = np.zeros(n * (n + 1) // 2)
    bad = L.rno_pooled_dense_factor(M.ctypes.data, n, upper.ctypes.data)
    return upper, bool(bad)


# ---------------------------------------------------------------------------------------------------------------------
# The pooled window covariance of RN_ADAPT_POOLED with the dense tuner (rn_k_pool_reduce pass 0, rn_k_pool_reduce_dense,
# rn_k_pool_factor, rn_k_pool_apply_dense)
# ---------------------------------------------------------------------------------------------------------------------
def welford_dense_restated(draws):
    """the kernels' per-chain window statistics over draws [chains][L][n] with the co-moment: mean += od / k,
    cov[j][k] += nd[j] * od[k] (nd = q - the updated mean).  Returns (mean [chains][n], cov [chains][n][n])."""
    draws = np.asarray(draws, dtype=np.float64)
    C_, n = draws.shape[0], draws.shape[2]
    mean, cov = np.zeros((C_, n)), np.zeros((C_, n, n))
    for k in range(draws.shape[1]):
        q = draws[:, k]
        od = q - mean
        mean = mean + od / float(k + 1)
        nd = q - mean
        cov = cov + nd[:, :, None] * od[:, None, :]
    return mean, cov


def pool_reduce_dense_restated(mean, cov, L, ranks=1):
    """rn_k_pool_reduce (pass 0) and rn_k_pool_reduce_dense (pass 1) in float64, in the kernels' order, over chains split as
    dist.chain_block splits them, the two all-reduces summing the ranks' buffers in rank order.  mean [chains][n], cov
    [chains][n][n].  Returns (pool [1 + n + n^2] after the second all-reduce, M [n][n] = S / (C L), the ranks' own buffers
    after pass 1 before it)."""
    from rainier_b200 import dist

    mean, cov = np.asarray(mean, dtype=np.float64), np.asarray(cov, dtype=np.float64)
    chains, n = mean.shape
    blocks = [dist.chain_block(chains, r, ranks) for r in range(ranks)]
    pools = []
    for lo, hi in blocks:
        p = np.zeros(1 + n + n * n)
        p[0], p[1:n + 1] = float(hi - lo), _block_sum(mean[lo:hi])
        pools.append(p)
    tot = pools[0][:n + 1].copy()
    for p in pools[1:]:
        tot = tot + p[:n + 1]
    g = tot[1:] / tot[0]
    for p, (lo, hi) in zip(pools, blocks):
        p[:n + 1] = tot
        d = mean[lo:hi] - g
        t = cov[lo:hi] + float(L) * d[:, :, None] * d[:, None, :]
        p[n + 1:] = _block_sum(t.reshape(hi - lo, n * n))
    s = pools[0][n + 1:].copy()
    for p in pools[1:]:
        s = s + p[n + 1:]
    pool = np.concatenate([tot, s])
    return pool, (s / (pool[0] * float(L))).reshape(n, n), [p.copy() for p in pools]


def cholesky_restated(M):
    """choleskyUpperTriangular (MassMatrix.scala:76-117) in float64, the reference's loop order.  Returns (lower, upper, bad):
    the packed lower and upper factors and whether M has an element 0.0 or a pivot is not > 0 (error flag 2)."""
    M = np.asarray(M, dtype=np.float64)
    n = M.shape[0]
    tri = lambda k: (k * (k + 1)) // 2  # noqa: E731
    lower = [np.float64(0.0)] * tri(n)
    bad = bool(np.any(M == 0.0))
    l = 0
    with np.errstate(all="ignore"):  # IEEE semantics: a zero pivot divides to inf / nan as on the device
        for i in range(n):
            for k in range(i + 1):
                s = np.float64(0.0)
                for j in range(k):
                    s += lower[tri(i) + j] * lower[tri(k) + j]
                x = M[i, k] - s
                if i == k:
                    lower[l] = np.sqrt(x)
                    bad = bad or not (lower[l] > 0.0)
                else:
                    lower[l] = np.float64(1.0) / lower[tri(k + 1) - 1] * x
                l += 1
    upper = [lower[tri(k + i) + i] for i in range(n) for k in range(n - i)]
    return np.array(lower), np.array(upper), bad


def pooled_covariance_exact(draws):
    """the population covariance of all draws [chains][L][n] of a window in exact rational arithmetic around the exact mean,
    (N sum q_j q_k - sum q_j sum q_k) / N^2.  Returns an n x n list of Fractions."""
    draws = np.asarray(draws, dtype=np.float64)
    n = draws.shape[2]
    a, e = _dyadic(draws.reshape(-1, n).T)  # one exponent for all entries
    N = draws.shape[0] * draws.shape[1]
    cols = [a[i * N:(i + 1) * N] for i in range(n)]
    sums = [sum(c) for c in cols]
    out = [[None] * n for _ in range(n)]
    for j in range(n):
        for k in range(j, n):
            v = Fraction(N * sum(x * y for x, y in zip(cols[j], cols[k])) - sums[j] * sums[k], N * N) * _scale(2 * e)
            out[j][k] = out[k][j] = v
    return out


def pool_dense_error_bound(mean, cov, L, ranks=1, e_mean=0.0, e_cov=0.0):
    """First-order bound on |M[j][k] - M_exact[j][k]|, [n][n]: M = pool_reduce_dense_restated(mean, cov, L, ranks)[1],
    M_exact the pooled population covariance of draws whose exact per-chain window means and co-moments lie within e_mean
    ([chains][n] or scalar) and e_cov ([chains][n][n] or scalar) of `mean`, `cov`.  Rounding error u = 2^-53 per operation,
    products of two error terms dropped; h = ceil(C_r / 256) + 8 + (R - 1) as in pool_error_bound.
      pooled mean g_j:              |dg_j| <= mean_c(e_mean) + h u mean_c |m_cj| + u |g_j|;
      d_cj = m_cj - g_j:            |dd_cj| <= e_mean_cj + |dg_j| + u |d_cj|;
      t_c = cov_c + (L d_cj) d_ck:  |dt_c| <= e_cov_c + L (|d_cj| |dd_ck| + |d_ck| |dd_cj|) + 2 u L |d_cj d_ck| + u |t_c|;
      M = sum_c t_c / (C L):        |dM| <= (sum_c |dt_c| + h u sum_c |t_c|) / (C L) + u |M|.
    sum_c C2_c[j][k] + L sum_c (mu_cj - g*_j)(mu_ck - g*_k) is exactly C L times the pooled covariance for the exact chain
    means mu_c, their exact mean g* and the exact co-moments C2_c, so this bounds the distance to M_exact."""
    mean, cov = np.asarray(mean, dtype=np.float64), np.asarray(cov, dtype=np.float64)
    chains, n = mean.shape
    e_mean, e_cov = np.broadcast_to(e_mean, mean.shape), np.broadcast_to(e_cov, cov.shape)
    per_rank = -(-chains // ranks)
    h = -(-per_rank // POOL_THREADS) + 8 + (ranks - 1)
    pool, M, _ = pool_reduce_dense_restated(mean, cov, L, ranks)
    g = pool[1:n + 1] / pool[0]
    dg = e_mean.mean(axis=0) + h * U * np.abs(mean).mean(axis=0) + U * np.abs(g)
    d = mean - g
    dd = e_mean + dg + U * np.abs(d)
    dj, dk, ddj, ddk = d[:, :, None], d[:, None, :], dd[:, :, None], dd[:, None, :]
    t = cov + float(L) * dj * dk
    dt = e_cov + L * (np.abs(dj) * ddk + np.abs(dk) * ddj) + 2.0 * U * L * np.abs(dj * dk) + U * np.abs(t)
    return (dt.sum(axis=0) + h * U * np.abs(t).sum(axis=0)) / (chains * float(L)) + U * np.abs(M)


def welford_dense_error_bound(draws):
    """First-order bounds (e_mean [chains][n], e_cov [chains][n][n]) on the distance between welford_dense_restated(draws)
    and the exact per-chain window means and co-moments.  E_i, R_i as in welford_error_bound.  Both factors of a product
    nd_j od_k are <= R and err by <= E + u R each; the product adds u R_j R_k; the running sum's partial sums are <= t R_j R_k
    after t draws, so its L roundings add <= u R_j R_k L (L + 1) / 2:
      |dC2[j][k]| <= L (R_k E_j + R_j E_k + 3 u R_j R_k) + u R_j R_k L (L + 1) / 2."""
    draws = np.asarray(draws, dtype=np.float64)
    L = draws.shape[1]
    A, R = np.abs(draws).max(axis=1), draws.max(axis=1) - draws.min(axis=1)
    E = U * (L * A + 2.0 * R * sum(1.0 / k for k in range(1, L + 1)))
    Rj, Rk, Ej, Ek = R[:, :, None], R[:, None, :], E[:, :, None], E[:, None, :]
    return E, L * (Rk * Ej + Rj * Ek + 3.0 * U * Rj * Rk) + U * Rj * Rk * L * (L + 1) / 2.0


def window_covariance_bound(draws, ranks=1):
    """first-order bound on |pooled window covariance as the kernels compute it from draws [chains][L][n] - the exact one|"""
    mean, cov = welford_dense_restated(draws)
    e_mean, e_cov = welford_dense_error_bound(draws)
    return pool_dense_error_bound(mean, cov, np.asarray(draws).shape[1], ranks, e_mean, e_cov)

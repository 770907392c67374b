"""
Pooled dense mass-matrix windows on the device (DenseMassMatrixTuner with rn_config.adaptation = RN_ADAPT_POOLED): the
shared covariance matrix and its factor are checked as values, at three levels.
  * The kernels on crafted statistics: tests/pool_dense_probe.cu launches rn_k_pool_reduce (pass 0), rn_k_pool_reduce_dense,
    rn_k_pool_factor and rn_k_pool_apply_dense of the module the runtime emits, with pool_window_dense's launch shapes, over
    R emulated ranks whose pool buffers are summed on the host in rank order.  Pool, matrix, factor, error flags and DualAvg
    restart are bit-equal to pooled_dense.pool_reduce_dense_restated / cholesky_restated and the oracle's exp / log.
  * Whole runs against the dense lockstep oracle (tests/pooled_dense_oracle.cpp) with parity.assert_parity, masses bit for bit
    where the model has no data; every window of a staged warmup; chunked against one-call runs.
  * The diagonal of the first pooled dense window against the pooled diagonal tuner, and funnel(60) with windows of 50
    draws, where each chain's own window covariance is rank-deficient.
"""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.cachedir import private_dir
from rainier_b200 import abi, api, dist

import parity
import pooled_dense as pd
import pooled_step as ps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# the kernels on crafted statistics
# ---------------------------------------------------------------------------------------------------------------------
def build_probe():
    src = os.path.join(ROOT, "tests", "pool_dense_probe.cu")
    hdr = os.path.join(ROOT, "rainier_b200", "csrc", "rn_args.h")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    key = hashlib.sha1(open(src, "rb").read() + open(hdr, "rb").read()).hexdigest()[:16]
    so = os.path.join(private_dir("rn_pool_dense_probe"), key + ".so")
    if not os.path.exists(so):
        tmp = so + ".tmp%d" % os.getpid()
        stubs = os.path.join(os.path.dirname(os.path.dirname(nvcc)), "lib64", "stubs")
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-w", "-shared", "-Xcompiler", "-fPIC", src,
                        "-L" + stubs, "-lcuda", "-o", tmp], check=True)
        os.replace(tmp, so)
    return so


NS = {abi.RN_BACKEND_THREAD: (1, 2, 10, 64), abi.RN_BACKEND_WARP: (1, 2, 10, 64, 200, 512)}


class _Modules(dict):
    """the emitted module of (n, backend, math mode), compiled on first use"""

    def __init__(self, lib):
        super().__init__()
        self.lib = lib

    def __missing__(self, key):
        n, backend, math = key
        rir, cols = configs.funnel(n).compile(True)
        m = api.CudaModel(rir, cols, device=-1)
        config = api.make_config(10, 10, sampler=api.HMCSampler(3), massMatrixTuner=api.DenseMassMatrixTuner(5, 1.5, 2, 2),
                                 adaptation=abi.RN_ADAPT_POOLED, backend=backend, mathMode=math, gradientMode=abi.RN_GRAD_ADJOINT)
        h = C.c_void_p()
        assert self.lib.pool_dense_probe_load(m.emit_cubin(config), 0, C.byref(h)) == 0
        m.close()
        self[key] = h
        return h


@pytest.fixture(scope="module")
def probe():
    import torch
    torch.zeros(1, device="cuda:0")  # the primary context, current on this thread
    L = C.CDLL(build_probe())
    L.pool_dense_probe_load.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]
    L.pool_dense_probe_unload.argtypes = [C.c_void_p, C.c_int]
    L.pool_dense_probe_launch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 8 + [C.c_int, C.c_void_p, C.c_int]
    mods = _Modules(L)
    yield L, mods
    for h in mods.values():
        L.pool_dense_probe_unload(h, 0)


def _tri(n):
    return n * (n + 1) // 2


def allreduce_in_rank_order(pools, lo, hi):
    import torch
    s = pools[0][lo:hi].cpu().numpy().copy()
    for p in pools[1:]:
        s = s + p[lo:hi].cpu().numpy()
    for p in pools:
        p[lo:hi] = torch.from_numpy(s).to(p.device)


def _pool_on_device(probe, key, mean, cov, L, ranks, da, da_iter, st_err, step_tuner):
    """pool_window_dense on R emulated ranks: pass 0, all-reduce of pool[0..n], pass 1, all-reduce of the n^2 sums, factor,
    apply"""
    import torch
    lib, mods = probe
    mod = mods[key]
    chains, n = mean.shape
    dev = lambda a, t=torch.float64: torch.tensor(np.ascontiguousarray(a), dtype=t, device="cuda:0")  # noqa: E731
    rk = []
    for r in range(ranks):
        lo, hi = dist.chain_block(chains, r, ranks)
        c = hi - lo
        rk.append({"lo": lo, "hi": hi, "mean": dev(mean[lo:hi].T), "raw": torch.full((n, c), 7.0, dtype=torch.float64, device="cuda:0"),
                   "cov": dev(cov[lo:hi].reshape(c, n * n).T), "mass": torch.full((n * n, c), -1.0, dtype=torch.float64, device="cuda:0"),
                   "chol": torch.full((_tri(n), c), -1.0, dtype=torch.float64, device="cuda:0"), "da": dev(da[lo:hi].T),
                   "da_iter": dev(da_iter[lo:hi], torch.int32), "st_err": dev(st_err[lo:hi], torch.int32),
                   "pool": torch.zeros(1 + n + n * n + 2 * _tri(n) + 1, dtype=torch.float64, device="cuda:0")})
    torch.cuda.synchronize()

    def launch(x, which):
        rc = lib.pool_dense_probe_launch(mod, which, n, x["hi"] - x["lo"], x["mean"].data_ptr(), x["raw"].data_ptr(), x["cov"].data_ptr(),
                                         x["mass"].data_ptr(), x["chol"].data_ptr(), x["da"].data_ptr(), x["da_iter"].data_ptr(),
                                         x["st_err"].data_ptr(), step_tuner, x["pool"].data_ptr(), L)
        assert rc == 0, "CUresult %d" % rc

    pools = [x["pool"] for x in rk]
    for x in rk:
        launch(x, 0)
    allreduce_in_rank_order(pools, 0, n + 1)
    for x in rk:
        launch(x, 1)
    local = [p[:1 + n + n * n].cpu().numpy().copy() for p in pools]
    allreduce_in_rank_order(pools, n + 1, 1 + n + n * n)
    for x in rk:
        launch(x, 2)
        launch(x, 3)
    cat = lambda k: np.concatenate([x[k].cpu().numpy() for x in rk], axis=-1)  # noqa: E731
    return {"local": local, "pools": [p.cpu().numpy() for p in pools], "mass": cat("mass").T, "chol": cat("chol").T, "mean": cat("mean").T,
            "raw": cat("raw").T, "cov": cat("cov").T, "da": cat("da").T, "da_iter": cat("da_iter"), "st_err": cat("st_err")}


def _crafted(kind, chains, L, n, seed):
    rng = np.random.default_rng(seed)
    mu = np.arange(n) * 0.5 - 2.0
    B = rng.normal(size=(n, n)) / np.sqrt(n)
    S = B @ B.T + np.eye(n)
    mean = mu + rng.normal(size=(chains, n))
    noise = rng.normal(size=(chains, n, n)) * 0.05
    cov = max(L - 1, 0) * (S + noise + noise.transpose(0, 2, 1))
    if kind == "between":  # within-chain co-moments all zero
        cov[:] = 0.0
    elif kind == "within":  # every chain has the same mean
        mean[:] = mu + 0.3
    elif kind == "big_mean":  # |mean| ~ 1e8 >> sd ~ 1
        mean = 1e8 + rng.normal(size=(chains, n))
    elif kind == "singular":  # M = v v^T exactly (v = 1, 2, ..., n): the second pivot is exactly 0
        v = np.arange(1.0, n + 1.0)
        mean[:] = 1.25
        cov[:] = float(L) * np.outer(v, v)
    elif kind == "nan":
        mean[rng.integers(chains), n - 1] = np.nan
    da = rng.normal(size=(chains, 5))
    da[:, 2] = rng.normal(-2.0, 1.0, size=chains)  # logStepSizeBar
    return mean, cov, da, rng.integers(1, 500, size=chains), rng.integers(0, 2, size=chains)


T, W = abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP
CASES = [  # (kind, chains, L, ranks, n, backend)
    ("general", 1, 1, 1, 1, T), ("general", 257, 50, 3, 2, T), ("general", 300, 7, 8, 10, T), ("general", 1029, 50, 2, 10, W),
    ("general", 257, 50, 1, 64, T), ("general", 257, 50, 5, 64, W), ("general", 257, 20, 2, 200, W), ("general", 40, 50, 3, 512, W),
    ("general", 4099, 2, 8, 2, W), ("between", 300, 50, 3, 10, T), ("between", 513, 1, 8, 10, W), ("within", 257, 50, 2, 10, W),
    ("within", 2, 50, 1, 2, T), ("big_mean", 4099, 50, 3, 10, T), ("big_mean", 257, 50, 2, 64, W), ("singular", 257, 3, 2, 10, T),
    ("singular", 40, 2, 1, 200, W), ("nan", 257, 50, 2, 10, W), ("nan", 300, 50, 3, 2, T)]


@pytest.mark.parametrize("kind,chains,L,ranks,n,backend", CASES, ids=["%s-C%d-L%d-R%d-n%d-b%d" % c for c in CASES])
def test_pool_dense_kernels_on_crafted_statistics(probe, kind, chains, L, ranks, n, backend):
    mean, cov, da, da_iter, st_err = _crafted(kind, chains, L, n, seed=chains * 31 + L * 7 + ranks + n)
    pool, M, local = pd.pool_reduce_dense_restated(mean, cov, L, ranks)
    _, upper, bad = pd.cholesky_restated(M)
    if kind in ("singular", "nan"):
        assert bad
    elif chains * L > n:
        assert not bad, "crafted matrix should be positive definite"
    ss = ps._vec(0, da[:, 2])
    da_want = np.stack([ss, ps._vec(1, ss), np.zeros(chains), np.zeros(chains), ps._vec(1, 10 * ss)], axis=1)
    for step_tuner in (0, 1):
        g = _pool_on_device(probe, (n, backend, abi.RN_MATH_PARITY), mean, cov, L, ranks, da, da_iter, st_err, step_tuner)
        for r in range(ranks):
            assert np.array_equal(g["local"][r], local[r], equal_nan=True), "rank %d: pool after pass 1 differs from the restatement" % r
            assert np.array_equal(g["pools"][r][:1 + n + n * n], pool, equal_nan=True), "rank %d: all-reduced pool differs" % r
        assert np.array_equal(g["mass"], np.broadcast_to(M.reshape(-1), (chains, n * n)), equal_nan=True), "mass differs on some chain"
        assert np.array_equal(g["chol"], np.broadcast_to(upper, (chains, _tri(n))), equal_nan=True), "factor differs on some chain"
        assert np.all(g["mean"] == 0.0) and np.all(g["raw"] == 0.0) and np.all(g["cov"] == 0.0), "window statistics not cleared"
        assert np.array_equal(g["st_err"], st_err | (2 if bad else 0))
        if step_tuner == 0:
            assert np.array_equal(g["da"], da_want) and np.all(g["da_iter"] == 0), "DualAvg restart differs"
        else:
            assert np.array_equal(g["da"], da) and np.array_equal(g["da_iter"], da_iter), "a static step size must leave DualAvg alone"


@pytest.mark.parametrize("n,backend", [(n, b) for b, ns in NS.items() for n in ns])
def test_factor_kernel_on_random_spd_matrices(probe, n, backend):
    """rn_k_pool_factor alone (C = 1, L = 1: M is the pool's sums): bit for bit the reference's loop in parity modules, within
    rounding in fast ones"""
    import torch
    lib, _ = probe
    rng = np.random.default_rng(n)
    X = rng.normal(size=(2 * n + 3, n))
    M = X.T @ X / (2 * n + 3) + 0.05 * np.eye(n)
    lower, upper, bad = pd.cholesky_restated(M)
    assert not bad
    for math in (abi.RN_MATH_PARITY, abi.RN_MATH_FAST):
        pool = np.zeros(1 + n + n * n + 2 * _tri(n) + 1)
        pool[0] = 1.0
        pool[1 + n:1 + n + n * n] = M.reshape(-1)
        p = torch.tensor(pool, device="cuda:0")
        z = torch.zeros(1, dtype=torch.float64, device="cuda:0")
        zi = torch.zeros(1, dtype=torch.int32, device="cuda:0")
        rc = lib.pool_dense_probe_launch(probe[1][(n, backend, math)], 2, n, 1, z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(),
                                         z.data_ptr(), z.data_ptr(), zi.data_ptr(), zi.data_ptr(), 1, p.data_ptr(), 1)
        assert rc == 0
        out = p.cpu().numpy()
        off = 1 + n + n * n
        got_lower, got_upper, flag = out[off:off + _tri(n)], out[off + _tri(n):off + 2 * _tri(n)], out[off + 2 * _tri(n)]
        assert flag == 0.0
        if math == abi.RN_MATH_PARITY:
            assert np.array_equal(got_lower, lower) and np.array_equal(got_upper, upper)
        else:
            assert np.allclose(got_upper, upper, rtol=1e-12, atol=1e-14)


# ---------------------------------------------------------------------------------------------------------------------
# whole runs against the lockstep oracle
# ---------------------------------------------------------------------------------------------------------------------
_ORACLE = {}


def _oracle(key, rir, cols, cfg, seeds):
    if key not in _ORACLE:
        _ORACLE[key] = pd.oracle_sample(rir, cols, cfg, seeds)
    return _ORACLE[key]


def _gpu(rir, cols, config, seeds, chunk=None, closes=None):
    """staged run: warmup(-1), or chunks of `chunk` iterations, or up to each of `closes` reading the mass after each"""
    import torch
    cfg, keep = api.lower_config(config)
    gm = api.CudaModel(rir, cols, device=0)
    s = api.CudaSampler(gm, config, seeds=seeds, trace=True)
    window_mass = []
    if closes is not None:
        done = 0
        for t in sorted(closes):
            s.warmup(t + 1 - done)
            done = t + 1
            window_mass.append(s.stats()[1])
        s.warmup(-1)
    elif chunk:
        for _ in range(0, cfg.warmup_iterations, chunk):
            s.warmup(chunk)
    else:
        s.warmup(-1)
    d = torch.empty((max(cfg.iterations, 1), gm.nVars, s.chains), dtype=torch.float64, device="cuda:0")
    s.run(cfg.iterations, d.data_ptr())
    s.sync()
    out = {"samples": d[: cfg.iterations].permute(2, 0, 1).contiguous().cpu().numpy(), "trace": s.read_trace(), "window_mass": window_mass}
    out["stats"], out["mass"] = s.stats()
    s.close()
    gm.close()
    return out


def _vs_oracle(key, model, config, seeds, exact_mass=True, tol=1e-9, primal=False):
    rir, cols = model.compile(not primal)
    cfg, keep = api.lower_config(config)
    g = _gpu(rir, cols, config, seeds)
    ref = _oracle(key, rir, cols, cfg, seeds)
    r = {"gpu": g["samples"], "ref": ref["samples"], "gpu_trace": g["trace"], "ref_trace": ref["trace"], "gpu_stats": g["stats"],
         "ref_stats": ref["stats"], "gpu_mass": g["mass"], "ref_mass": ref["mass"]}
    parity.assert_parity(r, tol=tol)
    assert np.all(g["mass"] == g["mass"][:1]), "chains ended warmup with different mass matrices"
    if exact_mass:
        assert np.array_equal(g["mass"], ref["mass"]), "pooled mass differs from the oracle's"
    else:
        assert parity.rel_err(g["mass"], ref["mass"]) < tol
    return g, ref


def _schools_config(**kw):
    c = api.SamplerConfig(**dict({"iterations": 30, "warmupIterations": 300, "adaptation": abi.RN_ADAPT_POOLED}, **kw))
    c._massMatrixTuner = api.DenseMassMatrixTuner(50, 1.5, 50, 50)
    return c


def test_eight_schools_default_config_thread_backend():
    """DefaultConfig (EHMC, per-chain DualAvg, windows 50/1.5/50/50) with the dense tuner, 256 chains"""
    _vs_oracle("schools", configs.eight_schools(), _schools_config(backend=abi.RN_BACKEND_THREAD), np.arange(256) + 11)


def test_eight_schools_default_config_warp_backend():
    _vs_oracle("schools", configs.eight_schools(), _schools_config(backend=abi.RN_BACKEND_WARP), np.arange(256) + 11)


def test_eight_schools_default_config_two_warps_per_chain(monkeypatch):
    monkeypatch.setenv("RN_WPC_K", "2")
    _vs_oracle("schools", configs.eight_schools(), _schools_config(backend=abi.RN_BACKEND_WARP), np.arange(256) + 11)


def test_funnel_hmc_ragged_chain_count():
    """1029 chains: several strides of 256 in the reduction and a ragged last block of the apply grid"""
    config = api.make_config(iterations=20, warmupIterations=150, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.DenseMassMatrixTuner(20, 1.5, 10, 10), adaptation=abi.RN_ADAPT_POOLED,
                             backend=abi.RN_BACKEND_THREAD)
    assert len(ps.window_closes(api.lower_config(config)[0])) >= 3
    _vs_oracle("funnel1029", configs.funnel(), config, np.arange(1029) + 5)


def test_pooled_dense_and_pooled_steps_together():
    _vs_oracle("schools-step", configs.eight_schools(), _schools_config(stepAdaptation=abi.RN_ADAPT_POOLED), np.arange(256) + 1)


def test_streamed_model_warp_backend():
    """streamed logistic regression on the warp shape: row sums are trees here, so samples and mass agree to 1e-8"""
    model = configs.logreg(1500, 6)
    config = api.make_config(iterations=10, warmupIterations=60, sampler=api.HMCSampler(4), stepSizeTuner=api.StaticStepSize(0.01),
                             massMatrixTuner=api.DenseMassMatrixTuner(8, 2.0, 5, 5), adaptation=abi.RN_ADAPT_POOLED,
                             backend=abi.RN_BACKEND_WARP)
    assert len(ps.window_closes(api.lower_config(config)[0])) >= 2
    _vs_oracle("logreg", model, config, np.arange(67) + 3, exact_mass=False, tol=1e-8, primal=True)


def test_every_window_of_a_staged_warmup():
    rir, cols = configs.eight_schools().compile(True)
    config = _schools_config(iterations=5)
    cfg, keep = api.lower_config(config)
    seeds = np.arange(300) + 2
    ref = _oracle("schools-windows", rir, cols, cfg, seeds)
    closes, wins = sorted(ps.window_closes(cfg)), ps.windows(cfg)
    assert len(wins) >= 2
    g = _gpu(rir, cols, config, seeds, closes=closes)
    for w, idx in enumerate(wins):
        m = g["window_mass"][w]
        assert np.array_equal(m, np.broadcast_to(ref["window_mass"][w], m.shape)), "window %d: device mass differs from the oracle's" % w


def test_chunked_warmup_and_one_call_sample_are_invisible():
    """warmup in chunks of 7 with launchIterations = 5 equals warmup(-1) bit for bit; rn_sample equals the staged sampler"""
    rir, cols = configs.eight_schools().compile(True)
    seeds = np.arange(200) + 4
    whole = _gpu(rir, cols, _schools_config(), seeds)
    chunked = _gpu(rir, cols, _schools_config(launchIterations=5), seeds, chunk=7)
    for k in ("samples", "trace", "mass"):
        assert np.array_equal(whole[k], chunked[k]), k
    assert [s.stepSize for s in whole["stats"]] == [s.stepSize for s in chunked["stats"]]
    m = api.CudaModel(rir, cols, device=0)
    tr = m.sample(_schools_config(), seeds=seeds)
    m.close()
    assert np.array_equal(np.asarray(tr.chains), whole["samples"])
    assert np.array_equal(tr.mass, whole["mass"])


@pytest.mark.parametrize("backend", [abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP])
def test_first_window_diagonal_equals_the_pooled_diagonal_tuner(backend):
    """same seeds and config, parity math, a data-free model: up to the first window end both runs carry the identity, and
    the diagonal co-moment products are the diagonal M2 products, so the first dense window's diagonal is the diagonal
    tuner's first window bit for bit"""
    rir, cols = configs.eight_schools().compile(True)
    seeds = np.arange(300) + 21
    dense = _schools_config(iterations=1, backend=backend)
    diag = api.SamplerConfig(iterations=1, warmupIterations=300, adaptation=abi.RN_ADAPT_POOLED, backend=backend)
    first = min(ps.window_closes(api.lower_config(dense)[0]))
    assert first == min(ps.window_closes(api.lower_config(diag)[0]))
    a = _gpu(rir, cols, dense, seeds, closes=[first])["window_mass"][0]
    b = _gpu(rir, cols, diag, seeds, closes=[first])["window_mass"][0]
    n = b.shape[1]
    assert a.shape == (len(seeds), n * n)
    assert np.array_equal(np.einsum("cii->ci", a.reshape(-1, n, n)), b)


def test_funnel60_windows_of_50_draws():
    """n = 60 > L = 50: every chain's own window covariance is rank-deficient, the pooled one over 1024 chains is not.
    Warmup finishes with no error flag and finite samples, and the returned matrix is positive definite."""
    rir, cols = configs.funnel(60).compile(True)
    config = api.SamplerConfig(iterations=50, warmupIterations=400, adaptation=abi.RN_ADAPT_POOLED, backend=abi.RN_BACKEND_WARP)
    config._massMatrixTuner = api.DenseMassMatrixTuner(50, 1.5, 50, 50)
    assert len(ps.window_closes(api.lower_config(config)[0])) >= 2
    g = _gpu(rir, cols, config, np.arange(1024) + 1)  # (error flag 2 on any chain raises RN_E_INVALID when stats are read)
    assert np.all(np.isfinite(g["samples"]))
    M = g["mass"][0].reshape(60, 60)
    assert np.all(g["mass"] == g["mass"][:1])
    np.linalg.cholesky(M)

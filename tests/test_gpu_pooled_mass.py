"""
Pooled mass-matrix windows on the device (rn_config.adaptation = RN_ADAPT_POOLED): the shared diagonal mass matrix is
checked as a value, at three levels.
  * The kernels on crafted statistics: tests/pool_probe.cu launches rn_k_pool_reduce and rn_k_pool_apply of the module the
    runtime emits, with pool_window's launch shapes, over R emulated ranks whose pool buffers are summed on the host in
    rank order.  Pool, mass, error flags and DualAvg restart are bit-equal to the restated reduction
    (pooled_step.pool_reduce_restated) and the oracle's exp / log; the variance is within a first-order bound
    (pooled_step.pool_error_bound, derivation there) of the exact pooled variance.
  * Whole runs against the lockstep oracle (tests/pooled_step_oracle.cpp) with parity.assert_parity, masses bit for bit
    where the model has no data.
  * Every window of a staged warmup against the oracle's window masses and the exact variance of that window's draws.
"""
import ctypes as C
import hashlib
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.binding import OracleModel
from oracle.rainier_py.cachedir import private_dir
from rainier_b200 import abi, api, dist

import parity
import pooled_step as ps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# the kernels on crafted statistics
# ---------------------------------------------------------------------------------------------------------------------
def build_probe():
    src = os.path.join(ROOT, "tests", "pool_probe.cu")
    hdr = os.path.join(ROOT, "rainier_b200", "csrc", "rn_args.h")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    key = hashlib.sha1(open(src, "rb").read() + open(hdr, "rb").read()).hexdigest()[:16]
    so = os.path.join(private_dir("rn_pool_probe"), key + ".so")
    if not os.path.exists(so):
        tmp = so + ".tmp%d" % os.getpid()
        stubs = os.path.join(os.path.dirname(os.path.dirname(nvcc)), "lib64", "stubs")
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-w", "-shared", "-Xcompiler", "-fPIC", src,
                        "-L" + stubs, "-lcuda", "-o", tmp], check=True)
        os.replace(tmp, so)
    return so


@pytest.fixture(scope="module")
def probe():
    import torch
    torch.zeros(1, device="cuda:0")  # the primary context, current on this thread
    L = C.CDLL(build_probe())
    L.pool_probe_load.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]
    L.pool_probe_unload.argtypes = [C.c_void_p, C.c_int]
    L.pool_probe_launch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_void_p, C.c_int, C.c_int]
    mods = {}
    for n in (1, 10):
        rir, cols = configs.funnel(n).compile(True)
        m = api.CudaModel(rir, cols, device=-1)
        for backend in (abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP):
            cubin = m.emit_cubin(api.SamplerConfig(adaptation=abi.RN_ADAPT_POOLED, backend=backend))
            h = C.c_void_p()
            assert L.pool_probe_load(cubin, 0, C.byref(h)) == 0
            mods[(n, backend)] = h
        m.close()
    yield L, mods
    for h in mods.values():
        L.pool_probe_unload(h, 0)


def allreduce_in_rank_order(pools, lo, hi):
    """the emulated ncclAllReduce(sum) of pools[r][lo:hi]: summed on the host in rank order, written back to every rank"""
    import torch
    s = pools[0][lo:hi].cpu().numpy().copy()
    for p in pools[1:]:
        s = s + p[lo:hi].cpu().numpy()
    for p in pools:
        p[lo:hi] = torch.from_numpy(s).to(p.device)


def _pool_on_device(probe, n, backend, mean, m2, L, ranks, da, da_iter, st_err, step_tuner):
    """pool_window on R emulated ranks: pass 0, all-reduce of pool[0..n], pass 1, all-reduce of pool[n+1..2n], apply"""
    import torch
    lib, mods = probe
    mod = mods[(n, backend)]
    chains = mean.shape[0]
    dev = lambda a, t=torch.float64: torch.tensor(np.ascontiguousarray(a), dtype=t, device="cuda:0")  # noqa: E731
    ranks_ = []
    for r in range(ranks):
        lo, hi = dist.chain_block(chains, r, ranks)
        ranks_.append({"lo": lo, "hi": hi, "mean": dev(mean[lo:hi].T), "m2": dev(m2[lo:hi].T), "mass": torch.full((n, hi - lo), -1.0, dtype=torch.float64, device="cuda:0"),
                       "da": dev(da[lo:hi].T), "da_iter": dev(da_iter[lo:hi], torch.int32), "st_err": dev(st_err[lo:hi], torch.int32),
                       "pool": torch.zeros(2 * n + 1, dtype=torch.float64, device="cuda:0")})
    torch.cuda.synchronize()

    def launch(x, which, pass_):
        rc = lib.pool_probe_launch(mod, which, n, x["hi"] - x["lo"], x["mean"].data_ptr(), x["m2"].data_ptr(), x["mass"].data_ptr(),
                                   x["da"].data_ptr(), x["da_iter"].data_ptr(), x["st_err"].data_ptr(), step_tuner, x["pool"].data_ptr(), L, pass_)
        assert rc == 0, "CUresult %d" % rc

    pools = [x["pool"] for x in ranks_]
    for x in ranks_:
        launch(x, 0, 0)
    allreduce_in_rank_order(pools, 0, n + 1)
    for x in ranks_:
        launch(x, 0, 1)
    local = [p.cpu().numpy().copy() for p in pools]
    allreduce_in_rank_order(pools, n + 1, 2 * n + 1)
    for x in ranks_:
        launch(x, 1, 0)
    cat = lambda k: np.concatenate([x[k].cpu().numpy() for x in ranks_], axis=-1)  # noqa: E731
    return {"local": local, "pools": [p.cpu().numpy() for p in pools], "mass": cat("mass").T, "mean": cat("mean").T, "m2": cat("m2").T,
            "da": cat("da").T, "da_iter": cat("da_iter"), "st_err": cat("st_err")}


def _crafted(kind, chains, L, n, seed):
    rng = np.random.default_rng(seed)
    mu, sd = np.arange(n) * 3.0 - 5.0, 0.5 + np.arange(n) * 0.25
    mean = mu + rng.normal(size=(chains, n)) * sd
    m2 = rng.gamma(max(L - 1, 1) / 2.0, 2.0, size=(chains, n)) * sd * sd if L > 1 else np.zeros((chains, n))
    if kind == "between":  # within-chain statistics all zero
        m2[:] = 0.0
    elif kind == "within":  # every chain has the same mean
        mean[:] = mu + 0.3
    elif kind == "big_mean":  # |mean| ~ 1e8 >> sd ~ 1
        mean = 1e8 + rng.normal(size=(chains, n))
    elif kind == "zero":  # no variance at all: every chain gets error flag 2, the matrix is still written
        mean[:], m2[:] = 1.25, 0.0
    elif kind == "nan":
        mean[rng.integers(chains), n - 1] = np.nan
    da = rng.normal(size=(chains, 5))
    da[:, 2] = rng.normal(-2.0, 1.0, size=chains)  # logStepSizeBar
    return mean, m2, da, rng.integers(1, 500, size=chains), rng.integers(0, 2, size=chains)


SHAPES = [  # (chains, L, ranks, n): every chain count, window length, rank count and n of the issue's grid
    (1, 1, 1, 1), (1, 1687, 1, 10), (2, 2, 2, 1), (2, 50, 1, 10), (255, 50, 3, 10), (255, 1, 8, 1), (256, 2, 8, 10),
    (256, 1687, 1, 1), (257, 50, 2, 10), (257, 1, 3, 1), (4099, 1687, 8, 10), (4099, 2, 3, 1), (135168, 50, 8, 10),
    (135168, 1687, 1, 1), (135168, 1, 3, 10)]
CASES = ([("general", s, 0) for s in SHAPES] + [("general", (257, 2, 1, 10), 1)] +
         [("between", (257, 50, 3, 10), 0), ("between", (4099, 1, 8, 1), 0), ("within", (256, 1687, 2, 10), 0), ("within", (2, 50, 1, 1), 0),
          ("big_mean", (4099, 50, 3, 10), 0), ("big_mean", (135168, 1687, 8, 1), 0), ("zero", (255, 2, 2, 10), 0), ("zero", (1, 1, 1, 1), 0),
          ("nan", (257, 50, 2, 10), 0), ("nan", (135168, 50, 3, 1), 0)])


@pytest.mark.parametrize("kind,shape,step_tuner", CASES, ids=["%s-C%d-L%d-R%d-n%d-st%d" % ((k,) + s + (t,)) for k, s, t in CASES])
def test_pool_kernels_on_crafted_statistics(probe, kind, shape, step_tuner):
    chains, L, ranks, n = shape
    mean, m2, da, da_iter, st_err = _crafted(kind, chains, L, n, seed=chains * 31 + L * 7 + ranks + n)
    pool, var, local = ps.pool_reduce_restated(mean, m2, L, ranks)
    bad = not np.all(var > 0.0)
    assert bad == (kind in ("zero", "nan") or chains * L == 1)  # (one draw in all: no variance either)
    ss = ps._vec(0, da[:, 2])
    da_want = np.stack([ss, ps._vec(1, ss), np.zeros(chains), np.zeros(chains), ps._vec(1, 10 * ss)], axis=1)
    finite = [i for i in range(n) if np.isfinite(var[i])]
    exact = ps.pooled_variance_exact_stats(mean[:, finite], m2[:, finite], L)
    bound = ps.pool_error_bound(mean[:, finite], m2[:, finite], L, ranks)
    for k, i in enumerate(finite):
        assert abs(float(Fraction(var[i]) - exact[k])) <= bound[k], "parameter %d: restated variance outside the bound" % i
    if kind == "big_mean":  # the bound tells the two-pass form from sum q^2 / N - mean^2 (which cancels here)
        tb = ps.textbook_variance((L * mean).sum(axis=0), (m2 + L * mean * mean).sum(axis=0), float(chains * L))
        for k, i in enumerate(finite):
            assert abs(float(Fraction(tb[i]) - exact[k])) > bound[k]
    for backend in (abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP):
        g = _pool_on_device(probe, n, backend, mean, m2, L, ranks, da, da_iter, st_err, step_tuner)
        for r in range(ranks):
            assert np.array_equal(g["local"][r], local[r], equal_nan=True), "rank %d: pool after pass 1 differs from the restatement" % r
            assert np.array_equal(g["pools"][r], pool, equal_nan=True), "rank %d: all-reduced pool differs" % r
        assert np.array_equal(g["mass"], np.broadcast_to(var, (chains, n)), equal_nan=True), "mass differs on some chain"
        assert np.all(g["mean"] == 0.0) and np.all(g["m2"] == 0.0), "window statistics not cleared on every chain"
        assert np.array_equal(g["st_err"], st_err | (2 if bad else 0))
        if step_tuner == 0:
            assert np.array_equal(g["da"], da_want) and np.all(g["da_iter"] == 0), "DualAvg restart differs"
        else:
            assert np.array_equal(g["da"], da) and np.array_equal(g["da_iter"], da_iter), "a static step size must leave DualAvg alone"


# ---------------------------------------------------------------------------------------------------------------------
# whole runs against the lockstep oracle
# ---------------------------------------------------------------------------------------------------------------------
_ORACLE = {}


def _oracle(key, rir, cols, cfg, seeds):
    if key not in _ORACLE:
        _ORACLE[key] = ps.oracle_sample(rir, cols, cfg, seeds)
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
    return api.SamplerConfig(**dict({"iterations": 30, "warmupIterations": 300, "adaptation": abi.RN_ADAPT_POOLED}, **kw))


def test_eight_schools_default_config_thread_backend():
    """DefaultConfig (EHMC, per-chain DualAvg, windows 50/1.5/50/50), 256 chains"""
    _vs_oracle("schools", configs.eight_schools(), _schools_config(backend=abi.RN_BACKEND_THREAD), np.arange(256) + 11)


def test_eight_schools_default_config_warp_backend():
    _vs_oracle("schools", configs.eight_schools(), _schools_config(backend=abi.RN_BACKEND_WARP), np.arange(256) + 11)


def test_eight_schools_default_config_two_warps_per_chain(monkeypatch):
    monkeypatch.setenv("RN_WPC_K", "2")
    _vs_oracle("schools", configs.eight_schools(), _schools_config(backend=abi.RN_BACKEND_WARP), np.arange(256) + 11)


def test_funnel_hmc_ragged_chain_count():
    """1029 chains: several strides of 256 in the reduction and a ragged last block of the apply grid"""
    config = api.make_config(iterations=20, warmupIterations=150, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.DiagonalMassMatrixTuner(20, 1.5, 10, 10), adaptation=abi.RN_ADAPT_POOLED,
                             backend=abi.RN_BACKEND_THREAD)
    assert len(ps.window_closes(api.lower_config(config)[0])) >= 3
    _vs_oracle("funnel1029", configs.funnel(), config, np.arange(1029) + 5)


def test_pooled_mass_and_pooled_steps_together():
    _vs_oracle("schools-step", configs.eight_schools(), _schools_config(stepAdaptation=abi.RN_ADAPT_POOLED), np.arange(256) + 1)


def test_dmma_path_with_ragged_tail():
    """streamed logistic regression on the chain-batched DMMA path: 67 chains = four CTAs of 16 and a per-warp tail, whose
    Welford statistics feed the same reduction; row sums are trees here, so samples and mass agree to 1e-8"""
    model = configs.logreg(1500, 6)
    prir, pcols = model.compile(False)
    config = api.make_config(iterations=10, warmupIterations=60, sampler=api.HMCSampler(4), stepSizeTuner=api.StaticStepSize(0.01),
                             massMatrixTuner=api.DiagonalMassMatrixTuner(8, 2.0, 5, 5), adaptation=abi.RN_ADAPT_POOLED,
                             backend=abi.RN_BACKEND_WARP)
    assert "rn_dmma(z" in api.CudaModel(prir, pcols, device=-1).emit_source(config), "the model should take the DMMA path"
    assert len(ps.window_closes(api.lower_config(config)[0])) >= 2
    _vs_oracle("dmma", model, config, np.arange(67) + 3, exact_mass=False, tol=1e-8, primal=True)


def _window_checks(key, model, config, seeds):
    rir, cols = model.compile(True)
    cfg, keep = api.lower_config(config)
    ref = _oracle(key, rir, cols, cfg, seeds)
    closes, wins = sorted(ps.window_closes(cfg)), ps.windows(cfg)
    g = _gpu(rir, cols, config, seeds, closes=closes)
    for w, idx in enumerate(wins):
        m = g["window_mass"][w]
        assert np.array_equal(m, np.broadcast_to(ref["window_mass"][w], m.shape)), "window %d: device mass differs from the oracle's" % w
        draws = ref["warm_draws"][:, idx, :]  # the device's draws too: the runs are bit-identical
        exact, bound = ps.pooled_variance_exact(draws), ps.window_variance_bound(draws)
        for i in range(m.shape[1]):
            assert abs(float(Fraction(m[0, i]) - exact[i])) <= bound[i], "window %d, parameter %d outside the bound" % (w, i)
    return g, ref, wins


def test_every_window_of_a_staged_warmup():
    g, ref, wins = _window_checks("schools-windows", configs.eight_schools(), _schools_config(iterations=5), np.arange(300) + 2)
    assert len(wins) >= 2


def test_every_window_first_window_of_one_draw():
    config = api.make_config(iterations=5, warmupIterations=60, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.DiagonalMassMatrixTuner(1, 2.0, 3, 5), adaptation=abi.RN_ADAPT_POOLED)
    g, ref, wins = _window_checks("funnel-L1", configs.funnel(), config, np.arange(300) + 9)
    assert len(wins[0]) == 1 and len(wins) >= 4


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


def test_one_chain_equals_the_per_chain_oracle():
    """C = 1 and one window: the pooled variance reduces to the reference's raw / samples, so the device run equals the
    per-chain oracle's bit for bit in the mass"""
    config = api.make_config(iterations=30, warmupIterations=60, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.DiagonalMassMatrixTuner(30, 1.5, 10, 20), adaptation=abi.RN_ADAPT_POOLED)
    cfg, keep = api.lower_config(config)
    assert len(ps.window_closes(cfg)) == 1
    rir, cols = configs.funnel().compile(True)
    seeds = np.array([77], dtype=np.int64)
    g = _gpu(rir, cols, config, seeds)
    per_chain, keep2 = api.lower_config(config)
    per_chain.adaptation = abi.RN_ADAPT_PER_CHAIN
    ref = OracleModel(rir, cols).sample(per_chain, seeds=seeds, trace=True)
    assert np.array_equal(g["mass"], ref["mass"])
    r = {"gpu": g["samples"], "ref": ref["samples"], "gpu_trace": g["trace"], "ref_trace": ref["trace"], "gpu_stats": g["stats"],
         "ref_stats": ref["stats"], "gpu_mass": g["mass"], "ref_mass": ref["mass"]}
    parity.assert_parity(r, tol=1e-9)

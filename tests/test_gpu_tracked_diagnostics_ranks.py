"""Tracked diagnostics pooled over ranks, on one GPU: tests/diag_probe.cu launches the emitted module's rn_k_diag_accum,
rn_k_diag_terms and rn_k_diag_reduce over each emulated rank's chain block, with the launch shapes of rn_runtime.cpp's
track_accumulate and rn_sampler_tracked_diagnostics, and the rank buffers are summed on the host in rank order between the
two passes (the emulated ncclAllReduce).  200 chains span several CTAs of both kernels.  The result over R in {1, 2, 3, 8}
ranks must agree with the one-rank result to rounding and with the restatement of Trace.thin(thin).diagnostics to 1e-9."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.cachedir import private_dir
from oracle.rainier_py.diagnostics import trace_diagnostics
from rainier_b200 import api
from rainier_b200 import dist as rdist

import parity

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
LAGS = rdist.DIAG_LAGS
TERM_ROWS = 8  # rn_runtime.cpp: kTermRows


def build_probe():
    src = os.path.join(ROOT, "tests", "diag_probe.cu")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    key = hashlib.sha1(open(src, "rb").read()).hexdigest()[:16]
    so = os.path.join(private_dir("rn_diag_probe"), key + ".so")
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
    L.diag_probe_load.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]
    L.diag_probe_unload.argtypes = [C.c_void_p, C.c_int]
    L.diag_probe_accum.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 5 + [C.c_longlong, C.c_int, C.c_void_p, C.c_int]
    L.diag_probe_terms.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.diag_probe_reduce.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    rir, cols = configs.eight_schools().compile(True)
    m = api.CudaModel(rir, cols, device=-1)
    cubin = m.emit_cubin(api.SamplerConfig())
    m.close()
    h = C.c_void_p()
    assert L.diag_probe_load(cubin, 0, C.byref(h)) == 0
    yield L, h
    L.diag_probe_unload(h, 0)


def series(chains, iterations, n, seed):
    """AR(1) draws [chains][iterations][n] (phi 0.7, a chain-dependent offset): autocorrelated, so the ESS loop runs
    several lags, and the chains disagree a little, so rHat > 1"""
    rng = np.random.default_rng(seed)
    x = np.zeros((chains, iterations, n))
    e = rng.normal(size=(chains, iterations, n))
    for t in range(1, iterations):
        x[:, t] = 0.7 * x[:, t - 1] + e[:, t]
    return x + 0.05 * rng.normal(size=(chains, 1, n)) + 3.0


def track_rank(L, mod, draws, chunks, thin, threads=64, sub=99):
    """one rank: track_accumulate's launches over its chain block draws [chains_r][iterations][n] -> (state, kept)"""
    import torch
    Cr, I, n = draws.shape
    state = torch.zeros((3 + 2 * LAGS, n, Cr), dtype=torch.float64, device="cuda")
    seen = kept = 0
    for k in chunks:
        d = torch.tensor(np.ascontiguousarray(draws[:, seen:seen + k, :].transpose(1, 2, 0)), device="cuda")  # [k][n][C_r]
        j0 = (thin - seen % thin) % thin
        m = (k - 1 - j0) // thin + 1 if j0 < k else 0
        if m:
            assert L.diag_probe_accum(mod, d.data_ptr(), n, Cr, j0, thin, m, kept, min(sub, m), state.data_ptr(), threads) == 0
        seen, kept = seen + k, kept + m
    return state, kept


def pooled(L, mod, states, kept):
    """rn_sampler_tracked_diagnostics' two passes over the ranks' states, rank buffers summed on the host in rank order"""
    import torch
    n = states[0].shape[1]
    Lg = min(LAGS, kept - 1)
    nq = 2 + Lg
    terms = [torch.zeros((TERM_ROWS, n, s.shape[2]), dtype=torch.float64, device="cuda") for s in states]
    p0 = None
    for s, tm in zip(states, terms):
        Cr = s.shape[2]
        buf = torch.zeros(n, dtype=torch.float64, device="cuda")
        assert L.diag_probe_terms(mod, s.data_ptr(), n, Cr, kept, Lg, 0, 1, tm.data_ptr()) == 0
        assert L.diag_probe_reduce(mod, tm.data_ptr(), n, Cr, None, buf.data_ptr()) == 0
        v = np.concatenate([[0.0, 0.0, Cr, kept, float(kept) * kept], buf.cpu().numpy()])
        p0 = v if p0 is None else p0 + v
    assert rdist.equal_kept_counts(len(states), p0)
    shift = torch.tensor(p0[5:] / p0[2], device="cuda")
    p1 = None
    for s, tm in zip(states, terms):
        Cr = s.shape[2]
        out = torch.zeros(nq * n, dtype=torch.float64, device="cuda")
        assert L.diag_probe_reduce(mod, tm.data_ptr(), n, Cr, shift.data_ptr(), out.data_ptr()) == 0  # means left by pass 0
        for q0 in range(1, nq, TERM_ROWS):
            rows = min(TERM_ROWS, nq - q0)
            assert L.diag_probe_terms(mod, s.data_ptr(), n, Cr, kept, Lg, q0, rows, tm.data_ptr()) == 0
            assert L.diag_probe_reduce(mod, tm.data_ptr(), rows * n, Cr, None, out[q0 * n:].data_ptr()) == 0
        v = out.cpu().numpy()
        p1 = v if p1 is None else p1 + v
    return rdist.diagnostics_finish(kept, p0, p1)


@pytest.mark.parametrize("thin,chunks", [(1, [1, 120, 99, 80]), (3, [37] * 16 + [8])])
def test_ranks_agree_with_one_rank_and_restatement(probe, thin, chunks):
    L, mod = probe
    total = 200
    x = series(total, sum(chunks), 3, seed=thin)
    ref = np.array(trace_diagnostics(x[:, ::thin]))
    results = {}
    for R in (1, 2, 3, 8):
        states, kept = [], None
        for r in range(R):
            lo, hi = rdist.chain_block(total, r, R)
            st, kept = track_rank(L, mod, x[lo:hi], chunks, thin)
            states.append(st)
        results[R] = pooled(L, mod, states, kept)
        assert parity.rel_err(results[R], ref, 1e-9) < 1e-9, (R, results[R], ref)
        assert parity.rel_err(results[R], results[1], 1e-12) < 1e-12, R
    assert np.all(results[1][:, 0] > 1.0) and np.all(results[1][:, 1] < total * x[:, ::thin].shape[1])


def test_block_shapes_do_not_change_the_state(probe):
    """the state does not depend on the CTA size or the stage length: 200 chains over CTAs of 32, 64 and 128 threads"""
    L, mod = probe
    x = series(200, 300, 2, seed=9)
    base, _ = track_rank(L, mod, x, [300], 2)
    for threads, sub in ((32, 5), (64, 1), (128, 60)):
        st, _ = track_rank(L, mod, x, [100, 200], 2, threads=threads, sub=sub)
        assert st.cpu().numpy().tobytes() == base.cpu().numpy().tobytes(), (threads, sub)

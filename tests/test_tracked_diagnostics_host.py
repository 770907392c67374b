"""Tracked diagnostics (rn_sampler_track_diagnostics) on the CPU.  The emitted module's rn_k_diag_accum and rn_k_diag_terms
run under RN_HOST_EMULATION over oracle samples cut into random launch-sized chunks; their state must equal a sequential
float64 restatement bit for bit, and the host mirror of the two-pass finish (dist.combine_diagnostics) must reproduce the
restatement of Trace.thin(thin).diagnostics."""
import ctypes as C
import os
import socket

import numpy as np
import pytest

import host_emulation
from oracle.rainier_py.binding import OracleModel, default_config
from oracle.rainier_py.diagnostics import trace_diagnostics
from rainier_b200 import abi, api
from rainier_b200 import dist as rdist

import parity

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAGS = rdist.DIAG_LAGS

_SHIM = r"""
#include <vector>
// one launch of rn_k_diag_accum / rn_k_diag_terms, every emulated thread in turn (each owns its shared-memory column)
extern "C" void emu_diag_accum(const double* s, int n, int C, int j0, int thin, int m, long long T0, int sub, double* state,
                               int block) {
  std::vector<double> smem((size_t)(RN_DIAG_LAGS + sub) * block);
  rn_diag_accum_smem = smem.data();
  blockDim.x = (unsigned)block; gridDim.x = (unsigned)((C + block - 1) / block); gridDim.y = (unsigned)n;
  for (int y = 0; y < n; y++)
    for (unsigned b = 0; b < gridDim.x; b++)
      for (int t = 0; t < block; t++) {
        blockIdx.x = b; blockIdx.y = (unsigned)y; threadIdx.x = (unsigned)t;
        rn_k_diag_accum(s, n, C, j0, thin, m, T0, sub, state);
      }
}
extern "C" void emu_diag_terms(const double* state, int n, int C, long long T, int L, int q0, int nq, double* out) {
  blockDim.x = 128; gridDim.x = (unsigned)((C + 127) / 128); gridDim.y = (unsigned)n;
  for (int y = 0; y < n; y++)
    for (unsigned b = 0; b < gridDim.x; b++)
      for (int t = 0; t < 128; t++) {
        blockIdx.x = b; blockIdx.y = (unsigned)y; threadIdx.x = (unsigned)t;
        rn_k_diag_terms(state, n, C, T, L, q0, nq, out);
      }
}
"""


@pytest.fixture(scope="module")
def kernels():
    rir = open(os.path.join(ROOT, "rainier_b200", "models", "eight_schools.rir"), "rb").read()
    m = api.CudaModel(rir, [], device=-1)
    src = m.emit_source(api.SamplerConfig(backend=abi.RN_BACKEND_THREAD))
    m.close()
    L = host_emulation.compile_source(src + _SHIM)
    L.emu_diag_accum.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_int, C.c_void_p, C.c_int]
    L.emu_diag_terms.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_void_p]
    return L


def oracle_samples(model, iterations, chains=5, seed=11):
    rir = open(os.path.join(ROOT, "rainier_b200", "models", model + ".rir"), "rb").read()
    cfg = default_config()
    cfg.sampler, cfg.n_steps = abi.RN_SAMPLER_HMC, 4
    cfg.mass_tuner = abi.RN_MASS_IDENTITY
    cfg.warmup_iterations, cfg.iterations = 60, iterations
    return OracleModel(rir, []).sample(cfg, seeds=np.arange(chains) + seed)["samples"]  # [chains][iterations][n]


def track(L, chains, chunks, thin, sub=99, block=64):
    """drives rn_k_diag_accum like rn_runtime.cpp's track_accumulate over launches of the given sizes -> state [201][n][C]"""
    Cn, I, n = chains.shape
    state = np.zeros((3 + 2 * LAGS, n, Cn))
    seen = kept = 0
    for k in chunks:
        draws = np.ascontiguousarray(chains[:, seen:seen + k, :].transpose(1, 2, 0))  # [k][n][C], as rn_sampler_run writes
        j0 = (thin - seen % thin) % thin
        m = (k - 1 - j0) // thin + 1 if j0 < k else 0
        if m:
            L.emu_diag_accum(draws.ctypes.data, n, Cn, j0, thin, m, kept, min(sub, m), state.ctypes.data, block)
        seen, kept = seen + k, kept + m
    return state, kept


def restated(x):
    """sequential float64 restatement of one chain's series: sum, Welford mean and M2, variogram sums of lags 1..99"""
    s, mean, m2 = 0.0, 0.0, 0.0
    for t, v in enumerate(x):
        s += v
        d = v - mean
        mean += d / float(t + 1)
        m2 += d * (v - mean)
    vg = []
    for lag in range(1, LAGS + 1):
        a = 0.0
        for t in range(lag, len(x)):
            d = x[t] - x[t - lag]
            a += d * d
        vg.append(a)
    return s, mean, m2, vg


def random_chunks(rng, total):
    out = []
    while sum(out) < total:
        out.append(int(min(total - sum(out), rng.choice([1, 2, 3, 17, 98, 99, 100, 250]))))
    return out


@pytest.mark.parametrize("model", ["eight_schools", "funnel10"])
@pytest.mark.parametrize("thin", [1, 2, 3, 7])
def test_accumulated_state_is_the_sequential_sums(kernels, model, thin):
    chains = oracle_samples(model, 260)
    rng = np.random.default_rng(thin)
    state, kept = track(kernels, chains, random_chunks(rng, chains.shape[1]), thin)
    kept_draws = chains[:, ::thin, :]
    assert kept == kept_draws.shape[1]
    for c in range(chains.shape[0]):
        for i in range(chains.shape[2]):
            s, mean, m2, vg = restated([float(v) for v in kept_draws[c, :, i]])
            assert state[0, i, c] == s and state[1, i, c] == mean and state[2, i, c] == m2
            assert np.array_equal(state[3 + LAGS:, i, c], vg)
            ring = state[3:3 + LAGS, i, c]
            for t in range(max(0, kept - LAGS), kept):
                assert ring[t % LAGS] == kept_draws[c, t, i]
    # the same run in one launch, and with a stage of 5 draws and 32 threads per block: the same bits
    whole, _ = track(kernels, chains, [chains.shape[1]], thin)
    small, _ = track(kernels, chains, [chains.shape[1]], thin, sub=5, block=32)
    assert np.array_equal(whole, state) and np.array_equal(small, state)


def test_several_ctas_match_the_vectorised_restatement(kernels):
    """200 chains: several CTAs of 32 and 64 threads, stages of 1, 5 and 99 draws, thin 1, 3 and 7; the state equals a
    sequential float64 restatement (vectorised over pairs, each element still summed in order) bit for bit"""
    rng = np.random.default_rng(4)
    x = np.cumsum(rng.normal(size=(200, 230, 2)), axis=1) * 0.1 + rng.normal(size=(200, 230, 2))
    for thin in (1, 3, 7):
        kept_draws = x[:, ::thin, :]
        T = kept_draws.shape[1]
        s, mean, m2 = np.zeros((200, 2)), np.zeros((200, 2)), np.zeros((200, 2))
        for t in range(T):
            v = kept_draws[:, t]
            s = s + v
            d = v - mean
            mean = mean + d / float(t + 1)
            m2 = m2 + d * (v - mean)
        vg = np.zeros((LAGS, 200, 2))
        for lag in range(1, LAGS + 1):
            for t in range(lag, T):
                d = kept_draws[:, t] - kept_draws[:, t - lag]
                vg[lag - 1] = vg[lag - 1] + d * d
        for block, sub in ((32, 5), (64, 1), (64, 99)):
            state, kept = track(kernels, x, random_chunks(np.random.default_rng(block + sub + thin), 230), thin, sub=sub, block=block)
            assert kept == T
            assert np.array_equal(state[0], s.T) and np.array_equal(state[1], mean.T) and np.array_equal(state[2], m2.T)
            assert np.array_equal(state[3 + LAGS:], vg.transpose(0, 2, 1))


def blocks_of(kernels, state, kept, bounds):
    """per emulated rank: (T, sums, M2, variogram sums) of its chain block, read from the state (field-major, chain fastest)"""
    out = []
    for lo, hi in bounds:
        st = state[:, :, lo:hi]
        out.append((kept, st[0].T, st[2].T, st[3 + LAGS:].transpose(2, 0, 1)))
    return out


@pytest.mark.parametrize("kept_target", [2, 3, 50, 99, 100, 101, 1000])
@pytest.mark.parametrize("model", ["eight_schools", "funnel10"])
def test_finish_matches_trace_restatement(kernels, model, kept_target):
    thin = 3 if kept_target in (3, 101) else 1
    chains = oracle_samples(model, kept_target * thin, chains=4, seed=5)
    rng = np.random.default_rng(kept_target)
    state, kept = track(kernels, chains, random_chunks(rng, chains.shape[1]), thin)
    assert kept == kept_target
    ref = np.array(trace_diagnostics(chains[:, ::thin]))
    got = rdist.combine_diagnostics(blocks_of(kernels, state, kept, [(0, chains.shape[0])]))
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    assert parity.rel_err(got, ref, 1e-9) < 1e-9, (got, ref)
    # the device's per-chain terms (rn_k_diag_terms) are the mirror's
    n, Cn, L = chains.shape[2], chains.shape[0], min(LAGS, kept - 1)
    terms = np.zeros((2 + L, n, Cn))
    for q0 in range(0, 2 + L, 8):  # in the runtime's batches of 8 quantities
        kernels.emu_diag_terms(state.ctypes.data, n, Cn, kept, L, q0, 8, terms[q0:].ctypes.data)
    assert np.array_equal(terms[0], state[0] / kept) and np.array_equal(terms[1], state[2] / (kept - 1))
    for lag in range(1, L + 1):
        assert np.array_equal(terms[1 + lag], state[3 + LAGS + lag - 1] / (kept - lag))


def test_rank_split_agrees_with_one_block(kernels):
    chains = oracle_samples("funnel10", 300, chains=11, seed=3)
    state, kept = track(kernels, chains, [300], 2)
    one = rdist.combine_diagnostics(blocks_of(kernels, state, kept, [(0, 11)]))
    ref = np.array(trace_diagnostics(chains[:, ::2]))
    assert parity.rel_err(one, ref, 1e-9) < 1e-9
    for world in range(1, 9):
        split = rdist.combine_diagnostics(blocks_of(kernels, state, kept, [rdist.chain_block(11, r, world) for r in range(world)]))
        assert parity.rel_err(split, one, 1e-12) < 1e-12, world


def test_errors_and_equal_count_verdict():
    rng = np.random.default_rng(0)
    blk = lambda T, C: (T, rng.normal(size=(C, 2)), rng.random((C, 2)), rng.random((C, LAGS, 2)))
    with pytest.raises(ValueError, match="Trace.scala:12"):
        rdist.combine_diagnostics([blk(10, 1)])
    rdist.combine_diagnostics([blk(10, 1), blk(10, 1)])  # one chain per rank, two in total
    with pytest.raises(ValueError, match="at least 2"):
        rdist.combine_diagnostics([blk(1, 3)])
    # every rank sums the pass-0 vectors in its own order (here: starting from itself); the counts are integers, exact in
    # fp64, so every rank reaches the same verdict, and it is the true one
    for counts in ([5, 5, 5], [5, 6, 5], [1, 1], [7, 3], [1000000, 999999], [3, 3, 3, 3, 3, 3, 3, 4]):
        vecs = [rdist.diagnostics_pass0(T, np.full((2, 1), 0.1 * (r + 1))) for r, T in enumerate(counts)]
        verdicts = set()
        for r in range(len(counts)):
            total = vecs[r].copy()
            for v in vecs[r + 1:] + vecs[:r]:
                total = total + v
            verdicts.add(rdist.equal_kept_counts(len(counts), total))
        assert verdicts == {len(set(counts)) == 1}
        if len(set(counts)) > 1:
            with pytest.raises(ValueError, match="different numbers"):
                rdist.combine_diagnostics([blk(T, 2) for T in counts])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_dir, blocks):
    import sys
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    T, sums, m2, vg = blocks[rank]
    p0 = torch.tensor(rdist.diagnostics_pass0(T, sums))
    dist.all_reduce(p0)
    p0 = p0.numpy()
    assert rdist.equal_kept_counts(world, p0)
    p1 = torch.tensor(rdist.diagnostics_pass1(T, sums, m2, vg, p0))
    dist.all_reduce(p1)
    np.save(os.path.join(out_dir, "diag%d.npy" % rank), rdist.diagnostics_finish(T, p0, p1.numpy()))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_gloo(kernels, tmp_path):
    import torch.multiprocessing as mp
    chains = oracle_samples("eight_schools", 150, chains=7, seed=9)
    state, kept = track(kernels, chains, [40, 60, 50], 1)
    blocks = blocks_of(kernels, state, kept, [rdist.chain_block(7, r, 2) for r in range(2)])
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path), blocks), nprocs=2, join=True)
    d0, d1 = np.load(tmp_path / "diag0.npy"), np.load(tmp_path / "diag1.npy")
    assert np.array_equal(d0, d1)
    assert parity.rel_err(d0, rdist.combine_diagnostics(blocks), 1e-12) < 1e-12
    assert parity.rel_err(d0, np.array(trace_diagnostics(chains)), 1e-9) < 1e-9

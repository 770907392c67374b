"""Pooled EHMC trajectory lengths (rn_config.trajectory_adaptation = RN_ADAPT_POOLED) on this box: the ABI field, config
validation, the emitted source, the library's draw L_t against an independent restatement (tests/pooled_traj.py) and the
distribution it samples, and the kernels compiled for sm_90a.  The GPU tests (tests/test_zz_gpu_pooled_trajectory.py) run them."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle.rainier_py import configs
from rainier_b200 import abi, api

import pooled_traj as pt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_config_layout_keeps_the_reserved_slot():
    """trajectory_adaptation takes the int32 after static_matrix (formerly reserved2): size and every other offset unchanged"""
    sizes = (C.c_int32 * 4)()
    api.lib().rn_abi_sizes(sizes)
    assert sizes[0] == C.sizeof(abi.Config) == 152
    assert abi.Config.static_matrix.offset == 96 and abi.Config.trajectory_adaptation.offset == 100
    assert abi.Config.static_matrix_elements.offset == 104 and abi.Config.adaptation.offset == 112
    assert abi.Config.step_adaptation.offset == 52 and abi.Config.diagnostics.offset == 144
    c = abi.Config()
    c.trajectory_adaptation = 7
    api.lib().rn_config_default(C.byref(c))
    assert c.trajectory_adaptation == abi.RN_ADAPT_PER_CHAIN
    assert api.lower_config(api.SamplerConfig())[0].trajectory_adaptation == abi.RN_ADAPT_PER_CHAIN
    pooled = api.lower_config(api.SamplerConfig(trajectoryAdaptation=abi.RN_ADAPT_POOLED))[0]
    assert pooled.trajectory_adaptation == abi.RN_ADAPT_POOLED


def _create_rc(config, mutate=None):
    rir = open(os.path.join(ROOT, "rainier_b200", "models", "eight_schools.rir"), "rb").read()
    m = api.CudaModel(rir, [], device=-1)
    cfg, keep = api.lower_config(config)
    if mutate:
        mutate(cfg)
    seeds = np.arange(4, dtype=np.int64)
    h = C.c_void_p()
    return api.lib().rn_sampler_create(m.h, C.byref(cfg), seeds.ctypes.data, 4, C.byref(h))


def test_config_validation():
    hmc = api.make_config(10, 10, sampler=api.HMCSampler(3), trajectoryAdaptation=abi.RN_ADAPT_POOLED)
    assert _create_rc(hmc) == abi.RN_E_UNSUPPORTED  # nothing to pool
    too_long = api.make_config(10, 10, sampler=api.EHMCSampler(65537), trajectoryAdaptation=abi.RN_ADAPT_POOLED)
    assert _create_rc(too_long) == abi.RN_E_UNSUPPORTED
    assert _create_rc(api.SamplerConfig(), lambda c: setattr(c, "trajectory_adaptation", 2)) == abi.RN_E_INVALID
    assert _create_rc(api.SamplerConfig(), lambda c: setattr(c, "trajectory_adaptation", -1)) == abi.RN_E_INVALID
    # valid configurations get past validation to the missing device (no CPU fallback)
    assert _create_rc(api.SamplerConfig(trajectoryAdaptation=abi.RN_ADAPT_POOLED)) == abi.RN_E_CUDA
    longest = api.make_config(10, 10, sampler=api.EHMCSampler(65536), trajectoryAdaptation=abi.RN_ADAPT_POOLED)
    assert _create_rc(longest) == abi.RN_E_CUDA
    both = api.SamplerConfig(trajectoryAdaptation=abi.RN_ADAPT_POOLED, stepAdaptation=abi.RN_ADAPT_POOLED,
                             adaptation=abi.RN_ADAPT_POOLED)
    assert _create_rc(both) == abi.RN_E_CUDA


def test_per_chain_source_has_no_pooled_code():
    rir = open(os.path.join(ROOT, "rainier_b200", "models", "eight_schools.rir"), "rb").read()
    m = api.CudaModel(rir, [], device=-1)
    for backend in (abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP):
        assert "RN_TRAJ_POOL 1" not in m.emit_source(api.SamplerConfig(backend=backend))
        assert "#define RN_TRAJ_POOL 1" in m.emit_source(api.SamplerConfig(trajectoryAdaptation=abi.RN_ADAPT_POOLED, backend=backend))
    # HMC has no trajectory lengths to pool: never in its modules
    hmc = api.make_config(10, 10, sampler=api.HMCSampler(3))
    assert "#define RN_TRAJ_POOL 1" not in m.emit_source(hmc)


def _crafted():
    single = np.zeros(11, dtype=np.int64)
    single[7] = 5
    zero = np.zeros(1025, dtype=np.int64)
    zero[0] = 8192
    big = np.zeros(300, dtype=np.int64)
    big[[1, 17, 299]] = [(1 << 40) - 12345, 3, 1 << 39]
    rng = np.random.default_rng(5)
    wide = rng.integers(0, 4, size=65537).astype(np.int64)
    wide[65536] = 9
    skewed = np.zeros(1025, dtype=np.int64)
    skewed[[0, 1, 2, 3, 40, 1024]] = [3, 700, 2000, 5, 90, 1]
    return {"single bin": single, "all mass in bin 0": zero, "T near 2^40": big, "max_steps = 65536": wide, "skewed": skewed}


@pytest.mark.parametrize("name", list(_crafted()))
def test_library_draw_equals_the_restatement(name):
    h = _crafted()[name]
    for t0 in (0, 1, 12345678901):
        got = api.trajectory_lengths_sequence(h, t0, 300)
        assert np.array_equal(got, pt.lengths(h, t0, 300)), name
    assert np.all(h[api.trajectory_lengths_sequence(h, 0, 2000)] > 0)  # only lengths that occur are drawn


def test_draw_frequencies_match_the_histogram():
    """over 10^6 values of t the observed frequency of every length is h/T within 5 binomial standard deviations"""
    h = _crafted()["skewed"]
    n = 1_000_000
    got = api.trajectory_lengths_sequence(h, 0, n)
    obs = np.bincount(got, minlength=len(h))
    p = h / h.sum()
    sd = np.sqrt(n * p * (1 - p))
    assert np.all(np.abs(obs - n * p) <= 5 * sd + 1e-9), (obs[h > 0], (n * p)[h > 0])
    big = _crafted()["T near 2^40"]
    got = api.trajectory_lengths_sequence(big, 0, n)
    p = big / big.sum()
    obs = np.bincount(got, minlength=len(big))
    assert np.all(np.abs(obs - n * p) <= 5 * np.sqrt(n * p * (1 - p)) + 1e-9)


def test_tooling_refuses_bad_histograms():
    for h in (np.zeros(5, dtype=np.int64), np.array([1, -1, 3], dtype=np.int64), np.ones(65538, dtype=np.int64)):
        with pytest.raises(api.RainierCudaError) as e:
            api.trajectory_lengths_sequence(h, 0, 4)
        assert e.value.code == abi.RN_E_INVALID


def test_ring_histogram_keeps_the_unfilled_slot_zero():
    """a ring that never filled offers indices [0, ring_i + 1): slot 0 holds 0 (the reference's pre-increment)"""
    ring = np.array([[0, 4, 6, 0], [3, 2, 5, 1], [0, 0, 0, 0]], dtype=np.float64)
    h = pt.ring_histogram(ring, ring_i=np.array([2, 1, 0]), ring_full=np.array([0, 1, 0]), max_steps=6)
    assert h.tolist() == [2, 1, 1, 1, 1, 1, 1]
    assert h.sum() == 3 + 4 + 1


@pytest.mark.parametrize("backend", [abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP])
def test_pooled_kernels_compile_for_sm90a_without_device(backend):
    rir = open(os.path.join(ROOT, "rainier_b200", "models", "eight_schools.rir"), "rb").read()
    m = api.CudaModel(rir, [], device=-1)
    cfg = api.SamplerConfig(trajectoryAdaptation=abi.RN_ADAPT_POOLED, stepAdaptation=abi.RN_ADAPT_POOLED, backend=backend)
    cubin = m.emit_cubin(cfg)
    assert cubin[:4] == b"\x7fELF"
    _report(cubin, "eight schools, backend %d" % backend)


def test_dmma_module_admits_pooled_ehmc():
    """streamed logistic regression: per-chain EHMC keeps the per-warp path, pooled EHMC compiles the chain-batched DMMA path"""
    model = configs.logreg(1500, 6)
    prir, pcols = model.compile(False)
    m = api.CudaModel(prir, pcols, device=-1)
    per_chain = api.SamplerConfig(backend=abi.RN_BACKEND_WARP, _massMatrixTuner=api.IdentityMassMatrixTuner())
    pooled = api.SamplerConfig(backend=abi.RN_BACKEND_WARP, trajectoryAdaptation=abi.RN_ADAPT_POOLED,
                               _massMatrixTuner=api.IdentityMassMatrixTuner())
    assert "rn_dmma(z" not in m.emit_source(per_chain)
    src = m.emit_source(pooled)
    assert "rn_dmma(z" in src and "#define RN_TRAJ_POOL 1" in src
    cubin = m.emit_cubin(pooled)
    assert cubin[:4] == b"\x7fELF"
    _report(cubin, "logistic regression, DMMA")


def _report(cubin, what):
    """registers and spills of the sampling kernels as ptxas reports them (printed for the record)"""
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        return
    with tempfile.NamedTemporaryFile(suffix=".cubin") as f:
        f.write(cubin)
        f.flush()
        out = subprocess.run([cuobjdump, "-res-usage", f.name], capture_output=True, text=True).stdout
    print(what)
    for line in out.splitlines():
        if "Function" in line or "REG" in line:
            print("  " + line.strip())


# ---- the emitted kernels under host emulation against the oracle's restatement (tests/pooled_traj_oracle.cpp) -------------
def _emulated_vs_oracle(config, seeds, backend=abi.RN_BACKEND_THREAD, chains_per_cta=1, ranks=1, split=None):
    rir, cols = configs.eight_schools().compile(True)
    config.trajectoryAdaptation = abi.RN_ADAPT_POOLED
    config.backend = backend
    cfg, keep = api.lower_config(config)
    cm = api.CudaModel(rir, cols, device=-1)
    got = pt.emulate(cm.emit_source(config), cfg, seeds, cm, chains_per_cta=chains_per_cta, ranks=ranks, split=split)
    ref = pt.oracle_sample(rir, cols, cfg, seeds)
    assert np.array_equal(got["hist"], ref["hist"]), "pooled histograms differ"
    assert np.array_equal(got["rank_hists"].sum(axis=0), got["hist"])
    for k, what in ((1, "accept decisions"), (3, "leapfrog step counts"), (2, "step sizes"), (0, "log acceptance probabilities")):
        assert np.array_equal(got["trace"][:, :, k], ref["trace"][:, :, k]), what + " differ"
    assert np.array_equal(got["samples"], ref["samples"]), "samples are not bit-identical"
    for k, o in enumerate(ref["stats"]):
        assert got["stats"][k, 0] == o.gradient_evaluations and got["stats"][k, 1] == o.leapfrog_steps
        assert got["stats"][k, 2] == o.accepted and got["stats"][k, 3] == o.rng.seed48 and got["stats"][k, 4] == 0
    assert np.array_equal(got["mass"], ref["mass"])
    w = cfg.warmup_iterations
    L = pt.lengths(ref["hist"], 0, cfg.iterations)
    assert np.all(got["trace"][:, w:, 3] == L[None, :]), "a chain's sampling length differs from L_t"
    return got, ref


def test_thread_shape_matches_the_oracle_on_host():
    """eight schools, DefaultConfig (EHMC + DualAvg + diagonal windows), 40 chains, sampling split over two launches"""
    _emulated_vs_oracle(api.SamplerConfig(iterations=30, warmupIterations=160), np.arange(40) + 11, split=11)


def test_warp_shape_several_chains_per_cta_matches_the_oracle_on_host():
    """warp-per-chain source, 3 emulated chains per CTA and a ragged last CTA"""
    _emulated_vs_oracle(api.SamplerConfig(iterations=10, warmupIterations=80), np.arange(7) + 3, backend=abi.RN_BACKEND_WARP,
                        chains_per_cta=3)


def test_reversed_seeds_give_the_same_histogram_on_host():
    seeds = np.array([3, 17, 5, 99, 42, 8, 61, 23], dtype=np.int64)
    a, _ = _emulated_vs_oracle(api.SamplerConfig(iterations=20, warmupIterations=120), seeds)
    b, _ = _emulated_vs_oracle(api.SamplerConfig(iterations=20, warmupIterations=120), seeds[::-1].copy())
    assert np.array_equal(a["hist"], b["hist"])
    assert np.array_equal(a["samples"], b["samples"][::-1]) and np.array_equal(a["trace"], b["trace"][::-1])


def test_no_warmup_gives_zero_lengths_on_host():
    got, ref = _emulated_vs_oracle(api.SamplerConfig(iterations=12, warmupIterations=0), np.arange(9) + 1)
    assert got["hist"][0] == 9 and got["hist"][1:].sum() == 0
    assert np.all(got["trace"][:, :, 3] == 0)


@pytest.mark.parametrize("ranks", [2, 3])
def test_rank_histograms_sum_to_the_histogram_of_all_chains_on_host(ranks):
    """the chains split over emulated ranks as dist.chain_block splits them: each rank's rn_k_traj_hist counts its own chains,
    and their sum (the all-reduce) is the histogram of all chains, whatever the split"""
    seeds = np.arange(11, dtype=np.int64) + 5
    one, _ = _emulated_vs_oracle(api.SamplerConfig(iterations=15, warmupIterations=120), seeds)
    got, _ = _emulated_vs_oracle(api.SamplerConfig(iterations=15, warmupIterations=120), seeds, ranks=ranks)
    assert np.all(got["rank_hists"].sum(axis=1) > 0)
    assert np.array_equal(got["hist"], one["hist"]) and np.array_equal(got["samples"], one["samples"])

"""Pooled step-size adaptation (rn_config.step_adaptation = RN_ADAPT_POOLED) on this box: the ABI field, config validation,
and the kernel source with RN_STEP_POOL run under host emulation against the oracle's lockstep restatement, bit for bit
(tests/pooled_step.py).  The GPU tests (tests/test_gpu_pooled_step.py) check the device against the same oracle."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle.rainier_py import configs
from rainier_b200 import abi, api

import pooled_step as ps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_config_layout_keeps_the_reserved_slot():
    """step_adaptation takes the int32 after step_size_tuner (formerly reserved1): size and every other offset unchanged"""
    sizes = (C.c_int32 * 4)()
    api.lib().rn_abi_sizes(sizes)
    assert sizes[0] == C.sizeof(abi.Config) == 152
    assert abi.Config.step_size_tuner.offset == 48 and abi.Config.step_adaptation.offset == 52 and abi.Config.delta.offset == 56
    assert abi.Config.adaptation.offset == 112 and abi.Config.diagnostics.offset == 144
    c = abi.Config()
    c.step_adaptation = 7
    api.lib().rn_config_default(C.byref(c))
    assert c.step_adaptation == abi.RN_ADAPT_PER_CHAIN
    assert api.lower_config(api.SamplerConfig())[0].step_adaptation == abi.RN_ADAPT_PER_CHAIN
    assert api.lower_config(api.SamplerConfig(stepAdaptation=abi.RN_ADAPT_POOLED))[0].step_adaptation == abi.RN_ADAPT_POOLED


def _create_rc(config, mutate=None):
    rir = open(os.path.join(ROOT, "rainier_b200", "models", "funnel10.rir"), "rb").read()
    m = api.CudaModel(rir, [], device=-1)
    cfg, keep = api.lower_config(config)
    if mutate:
        mutate(cfg)
    seeds = np.arange(4, dtype=np.int64)
    h = C.c_void_p()
    return api.lib().rn_sampler_create(m.h, C.byref(cfg), seeds.ctypes.data, 4, C.byref(h))


def test_config_validation():
    static = api.make_config(10, 10, sampler=api.HMCSampler(3), stepSizeTuner=api.StaticStepSize(0.1),
                             massMatrixTuner=api.IdentityMassMatrixTuner(), stepAdaptation=abi.RN_ADAPT_POOLED)
    assert _create_rc(static) == abi.RN_E_UNSUPPORTED  # nothing to pool
    assert _create_rc(api.SamplerConfig(), lambda c: setattr(c, "step_adaptation", 2)) == abi.RN_E_INVALID
    assert _create_rc(api.SamplerConfig(), lambda c: setattr(c, "step_adaptation", -1)) == abi.RN_E_INVALID
    # valid configurations get past validation to the missing device (no CPU fallback)
    assert _create_rc(api.SamplerConfig(stepAdaptation=abi.RN_ADAPT_POOLED)) == abi.RN_E_CUDA
    assert _create_rc(api.SamplerConfig(stepAdaptation=abi.RN_ADAPT_POOLED, adaptation=abi.RN_ADAPT_POOLED)) == abi.RN_E_CUDA


def test_per_chain_source_has_no_pooled_code():
    rir = open(os.path.join(ROOT, "rainier_b200", "models", "eight_schools.rir"), "rb").read()
    m = api.CudaModel(rir, [], device=-1)
    assert "#define RN_STEP_POOL 1" not in m.emit_source(api.SamplerConfig())
    assert "#define RN_STEP_POOL 1" in m.emit_source(api.SamplerConfig(stepAdaptation=abi.RN_ADAPT_POOLED))


def _run(model, config, seeds, dense=False, backend=abi.RN_BACKEND_THREAD, chains_per_cta=1):
    rir, cols = model.compile(True)
    config.stepAdaptation = abi.RN_ADAPT_POOLED
    config.backend = backend
    cfg, keep = api.lower_config(config)
    cm = api.CudaModel(rir, cols, device=-1)
    got = ps.emulate(cm.emit_source(config), cfg, seeds, cm, chains_per_cta=chains_per_cta)
    ref = ps.oracle_sample(rir, cols, cfg, seeds, dense_mass=dense)
    assert np.array_equal(got["trace"][:, :, 1], ref["trace"][:, :, 1]), "accept decisions differ"
    assert np.array_equal(got["trace"][:, :, 3], ref["trace"][:, :, 3]), "leapfrog step counts differ"
    assert np.array_equal(got["trace"][:, :, 2], ref["trace"][:, :, 2]), "step sizes differ"
    assert np.array_equal(got["trace"][:, :, 0], ref["trace"][:, :, 0]), "log acceptance probabilities differ"
    assert np.all(got["trace"][:, :, 2] == got["trace"][:1, :, 2]), "chains ran different step sizes"
    assert np.array_equal(got["samples"], ref["samples"]), "samples are not bit-identical"
    for k, o in enumerate(ref["stats"]):
        assert got["stats"][k, 0] == o.gradient_evaluations and got["stats"][k, 1] == o.leapfrog_steps
        assert got["stats"][k, 2] == o.accepted and got["stats"][k, 3] == o.rng.seed48 and got["stats"][k, 4] == 0
    assert np.array_equal(got["mass"], ref["mass"])
    # every chain's copy of the DualAvg state is the same, and sampling used exp(logStepSizeBar) = the oracle's final step
    assert np.all(got["da"] == got["da"][:1]) and ref["stats"][0].step_size == got["trace"][0, -1, 2]
    return got, ref


def _cfg(it, warm, sampler, step, mass):
    return api.make_config(iterations=it, warmupIterations=warm, sampler=sampler, stepSizeTuner=step, massMatrixTuner=mass)


def test_funnel_hmc_dualavg_identity_on_host():
    _run(configs.funnel(), _cfg(30, 120, api.HMCSampler(5), api.DualAvgTuner(0.8), api.IdentityMassMatrixTuner()), np.arange(6) + 7)


def test_default_config_eight_schools_on_host():
    """EHMC + DualAvg + windowed diagonal mass: the pooled step is reset at every window end"""
    cfg = api.SamplerConfig(iterations=40, warmupIterations=260)
    assert len(ps.window_closes(api.lower_config(cfg)[0])) >= 2
    _run(configs.eight_schools(), cfg, np.arange(5) + 11)


def test_dense_mass_tuner_on_host():
    cfg = _cfg(20, 200, api.EHMCSampler(32, 1, 10, 0.1), api.DualAvgTuner(0.8), api.DenseMassMatrixTuner(40, 1.5, 20, 20))
    _run(configs.eight_schools(), cfg, np.arange(3) + 5, dense=True)


def test_wpc_source_several_chains_per_cta_on_host():
    """warp-per-chain source, 3 emulated chains per CTA (concurrent host threads adding into one slot) and a ragged last CTA"""
    _run(configs.eight_schools(), api.SamplerConfig(iterations=12, warmupIterations=110), np.arange(7) + 3,
         backend=abi.RN_BACKEND_WARP, chains_per_cta=3)


def test_reversed_seeds_reverse_the_outputs_on_host():
    """the pooled sums do not depend on chain order: in the oracle and in emulation, reversed seeds give reversed outputs"""
    seeds = np.array([3, 17, 5, 99, 42, 8], dtype=np.int64)
    cfg = api.SamplerConfig(iterations=15, warmupIterations=160)
    got, ref = _run(configs.eight_schools(), cfg, seeds)
    got_r, ref_r = _run(configs.eight_schools(), api.SamplerConfig(iterations=15, warmupIterations=160), seeds[::-1])
    for a, b in ((got, got_r), (ref, ref_r)):
        assert np.array_equal(a["samples"], b["samples"][::-1])
        assert np.array_equal(a["trace"], b["trace"][::-1])


@pytest.mark.parametrize("backend", [abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP])
def test_pooled_kernels_compile_for_sm90a_without_device(backend):
    rir = open(os.path.join(ROOT, "rainier_b200", "models", "eight_schools.rir"), "rb").read()
    m = api.CudaModel(rir, [], device=-1)
    cfg = api.SamplerConfig(stepAdaptation=abi.RN_ADAPT_POOLED, adaptation=abi.RN_ADAPT_POOLED, backend=backend)
    assert m.emit_cubin(cfg)[:4] == b"\x7fELF"

"""The thread-per-chain sampler's restore point (q, gradient and potential at startIteration) in shared memory, and the emitted
density without accumulations of the literal +0.0 -- both on the host (tests/host_emulation.py), bit-exact against the oracle.

The runtime gives the restore point shared-memory slots only where they cost no CTA per SM (rn_runtime.cpp:
tpc_restore_on_chip); elsewhere the sampler restores from `params` as before.  The emulation has no occupancy to lose, so the
configurations that keep the restore point in `params` on the device also run here with it on chip: EHMC's isUTurn against the
slots, and diagonal / dense mass-matrix window ends, after which the next iteration reads the current momentum from `params`."""
import os

import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.binding import OracleModel
from rainier_b200 import abi, api

import host_emulation as he

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _source(model, config):
    rir, cols = model.compile(True)
    config.backend = abi.RN_BACKEND_THREAD
    cm = api.CudaModel(rir, cols, device=-1)
    return cm, cm.emit_source(config)


def _check(model, config, seeds, src, cm, dense=False):
    rir, cols = model.compile(True)
    cfg, keep = api.lower_config(config)
    got = he.sample(src, cfg, seeds, cm)
    ref = OracleModel(rir, cols).sample(cfg, seeds=seeds, trace=True, dense_mass=dense)
    assert np.array_equal(got["trace"][:, :, 1], ref["trace"][:, :, 1]), "accept decisions differ"
    assert np.array_equal(got["trace"][:, :, 3], ref["trace"][:, :, 3]), "leapfrog step counts differ"
    assert np.array_equal(got["samples"], ref["samples"]), "samples are not bit-identical"
    for k, o in enumerate(ref["stats"]):
        assert got["stats"][k, 0] == o.gradient_evaluations and got["stats"][k, 1] == o.leapfrog_steps
        assert got["stats"][k, 2] == o.accepted and got["stats"][k, 3] == o.rng.seed48 and got["stats"][k, 4] == 0
    assert np.array_equal(got["mass"], ref["mass"])


def test_funnel_density_has_no_zero_accumulations():
    rir = open(os.path.join(ROOT, "rainier_b200", "models", "funnel10.rir"), "rb").read()
    m = api.CudaModel(rir, [], device=-1)
    cfg = api.make_config(iterations=10, warmupIterations=0, sampler=api.HMCSampler(5), stepSizeTuner=api.StaticStepSize(0.1),
                          massMatrixTuner=api.IdentityMassMatrixTuner())
    for backend in (abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP):
        cfg.backend = backend
        src = m.emit_source(cfg)
        dens = src[src.index("// ---- emitted"):]
        assert "+= 0x0p+0" not in dens
        assert "+= " in dens  # the data-free target's other terms are still accumulated


def test_restore_point_selection():
    """on chip for the funnel's HMC (n = 10, identity mass: 41 doubles per thread keep 4 CTAs of 128 per SM); in `params` for
    EHMC with an adapted diagonal matrix at n = 10 (61 doubles: 3 CTAs) and for dense mass at n = 64"""
    hmc = api.make_config(iterations=10, warmupIterations=10, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                          massMatrixTuner=api.IdentityMassMatrixTuner())
    assert "#define RN_TS_RESTORE 1" in _source(configs.funnel(), hmc)[1]
    assert "#define RN_TS_RESTORE 0" in _source(configs.eight_schools(), api.SamplerConfig(iterations=10, warmupIterations=60))[1]
    dense = api.make_config(iterations=2, warmupIterations=30, sampler=api.HMCSampler(2), stepSizeTuner=api.DualAvgTuner(0.8),
                            massMatrixTuner=api.DenseMassMatrixTuner(12, 1.5, 4, 4))
    assert "#define RN_TS_RESTORE 0" in _source(configs.funnel(64), dense)[1]


@pytest.mark.parametrize("case", ["default_eight_schools", "dense_ehmc_eight_schools", "diagonal_hmc_funnel7"])
def test_restore_point_on_chip_is_bit_exact(case):
    """window ends of both adapted matrices (the momentum `params` holds after an accepted or a rejected proposal), EHMC's
    isUTurn against the slots, odd n"""
    dense = False
    if case == "default_eight_schools":
        model, config, seeds = configs.eight_schools(), api.SamplerConfig(iterations=30, warmupIterations=200), np.arange(4) + 11
    elif case == "dense_ehmc_eight_schools":
        model, seeds, dense = configs.eight_schools(), np.arange(3) + 5, True
        config = api.make_config(iterations=20, warmupIterations=200, sampler=api.EHMCSampler(32, 1, 10, 0.1),
                                 stepSizeTuner=api.DualAvgTuner(0.8), massMatrixTuner=api.DenseMassMatrixTuner(40, 1.5, 20, 20))
    else:
        model, seeds = configs.funnel(7), np.arange(4) + 3
        config = api.make_config(iterations=20, warmupIterations=150, sampler=api.HMCSampler(4), stepSizeTuner=api.DualAvgTuner(0.8),
                                 massMatrixTuner=api.DiagonalMassMatrixTuner(30, 1.5, 15, 15))
    cm, src = _source(model, config)
    on = src.replace("#define RN_TS_RESTORE 0", "#define RN_TS_RESTORE 1")
    off = on.replace("#define RN_TS_RESTORE 1", "#define RN_TS_RESTORE 0")
    _check(model, config, seeds, on, cm, dense=dense)
    # the momentum `params` holds enters only the energy recomputed where a launch starts or a window ends (prevH): compare
    # energyVariance / energyTransitions2 after the warmup launch and after the sampling launch with the restore point in `params`
    assert np.array_equal(_energies(on, config, seeds, cm), _energies(off, config, seeds, cm))


# the emulated sampler's Stats energies ([e_mean, e_raw, trans2] x chains) after the warmup launch and after the sampling launch
_PROBE = """// energy probe
static double rn_probe_energy[2][3 * 64];
extern "C" const double* rn_probe_energies() { return &rn_probe_energy[0][0]; }
"""


def _energies(src, config, seeds, cm):
    shim = he._SAMPLER_SHIM
    a, b = "  // lf.resetStats(), Driver.scala:31\n", "  for (size_t k = 0; k < C; k++) {\n    out_stats[k * 5 + 0]"
    assert a in shim and b in shim and len(seeds) <= 64
    probe = shim.replace(a, "  std::memcpy(rn_probe_energy[0], energy.data(), 3 * C * sizeof(double));\n" + a)
    probe = probe.replace(b, "  std::memcpy(rn_probe_energy[1], energy.data(), 3 * C * sizeof(double));\n" + b)
    cfg, keep = api.lower_config(config)
    he._SAMPLER_SHIM = probe
    try:
        he.sample(_PROBE + src, cfg, seeds, cm)
        lib = he.compile_source(_PROBE + src)
    finally:
        he._SAMPLER_SHIM = shim
    lib.rn_probe_energies.restype = np.ctypeslib.ndpointer(np.float64, shape=(2, 3 * 64))
    return lib.rn_probe_energies()[:, : 3 * len(seeds)].copy()

"""Models whose per-chain state does not fit shared memory, on the device (rn_sampler_wpc.cuh / rn_optimizer.cuh:
RN_WPC_PLACE).  cfg 5's Poisson GLMM at 6 000 groups (n = 6 003) gets placement 1 -- chain vectors, L-BFGS history and
density scratch in global memory -- and must agree with the oracle as the warp-per-chain kernels do at any size; small models
forced into placement 1 must give what placement 0 gives."""
import os

import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.binding import OracleModel
from oracle.rainier_py.optimizer import lbfgs
from rainier_b200 import abi, api

import parity

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def glmm_6000():
    return configs.poisson_glm(6000, 12000).compile(False)  # primal RIR: the adjoint is emitted (scatter-add)


def _static(it, nsteps, eps):
    return api.make_config(iterations=it, warmupIterations=0, sampler=api.HMCSampler(nsteps), stepSizeTuner=api.StaticStepSize(eps),
                           massMatrixTuner=api.IdentityMassMatrixTuner())


def test_large_model_takes_placement_1(glmm_6000):
    prir, pcols = glmm_6000
    cm = api.CudaModel(prir, pcols)
    for cfg in (_static(1, 1, 0.1), api.SamplerConfig()):
        assert "#define RN_WPC_PLACE 1\n" in cm.emit_source(cfg)
    cm.close()


def test_large_model_density_batch(glmm_6000):
    prir, pcols = glmm_6000
    cm = api.CudaModel(prir, pcols)
    q = np.random.default_rng(0).normal(size=(5, cm.nVars)) * 0.2
    out = cm.density_batch(q)
    cm.close()
    ref = OracleModel(prir, pcols).density_batch(q)
    assert parity.rel_err(out, ref, 1e-9) < 1e-9


def test_large_model_static_hmc_matches_oracle(glmm_6000):
    prir, pcols = glmm_6000
    r = parity.run_both(prir, pcols, _static(8, 3, 0.002), seeds=np.arange(8) + 1)
    parity.assert_parity(r, tol=1e-7, check_mass=False)


def test_large_model_default_config_matches_oracle(glmm_6000):
    prir, pcols = glmm_6000
    r = parity.run_both(prir, pcols, api.SamplerConfig(iterations=4, warmupIterations=12), seeds=np.arange(4) + 21)
    parity.assert_parity(r, tol=1e-7, check_mass=False)


def test_large_model_optimize_matches_oracle(glmm_6000):
    prir, pcols = glmm_6000
    cm = api.CudaModel(prir, pcols)
    got = cm.optimize()
    cm.close()
    om = OracleModel(prir, pcols)
    ref = lbfgs(om.density_batch, len(got["x"][0]))
    # hundreds of evaluations in 6 003 dimensions: the tree-ordered row sums move the path by rounding, so the two runs stop
    # at different iterates.  Both converge; the device's f is the oracle's density at the device's x, that x meets the
    # stopping rule by the oracle's own gradient, and both minima agree.
    assert got["info"][0] == ref["info"] == 0 and abs(got["evals"][0] - ref["evals"]) <= 0.25 * ref["evals"]
    d = om.density_batch(got["x"][:1])[0]
    assert abs(got["f"][0] + d[0]) <= 1e-9 * abs(d[0])
    assert np.linalg.norm(d[1:]) / max(1.0, np.linalg.norm(got["x"][0])) <= 0.1
    assert abs(got["f"][0] - ref["f"]) <= 5e-3 * abs(ref["f"])


def test_large_model_chain_blocks_do_not_share_slices(glmm_6000, monkeypatch):
    """rn_sample cut into four chain blocks (rn_k_iter offsets by chain_begin): every chain equals the same seed sampled
    alone-ish in a call of four chains.  The scatter-add of the Lookup adjoint sums in no fixed order, so values agree to
    rounding; a shared slice would not agree at all."""
    prir, pcols = glmm_6000
    cfg = _static(6, 3, 0.002)
    seeds = np.arange(64) + 100
    monkeypatch.setenv("RN_SAMPLE_BLOCKS", "4")
    cm = api.CudaModel(prir, pcols)
    big = cm.sample(cfg, nChains=len(seeds), seeds=seeds).chains
    monkeypatch.delenv("RN_SAMPLE_BLOCKS")
    for part in (slice(0, 4), slice(30, 34), slice(60, 64)):
        small = cm.sample(cfg, nChains=4, seeds=seeds[part]).chains
        assert parity.rel_err(big[part], small, 1e-9) < 1e-10
    cm.close()


# ---- forced placements on small models: what placement 0 gives, on the device ------------------------------------------

def _device_run(rir, cols, config, seeds):
    cfg, keep = api.lower_config(config)
    gm = api.CudaModel(rir, cols)
    src = gm.emit_source(config)
    s = api.CudaSampler(gm, config, seeds=seeds, trace=True)
    import torch

    d = torch.empty((max(cfg.iterations, 1), gm.nVars, s.chains), dtype=torch.float64, device="cuda:0")
    s.warmup(-1)
    s.run(cfg.iterations, d.data_ptr())
    s.sync()
    out = {"samples": d[: cfg.iterations].permute(2, 0, 1).contiguous().cpu().numpy(), "trace": s.read_trace(), "src": src}
    stats, mass = s.stats()
    out["stats"] = [(g.gradientEvaluations, g.leapfrogSteps, g.accepted, g.rng[0]) for g in stats]
    out["mass"] = mass
    q = np.random.default_rng(1).normal(size=(7, gm.nVars)) * 0.3
    out["density"] = gm.density_batch(q)
    s.close()
    gm.close()
    return out


def _forced(monkeypatch, rir, cols, config, seeds, tma, scatter=False):
    config.backend = abi.RN_BACKEND_WARP
    monkeypatch.setenv("RN_WPC_K", "1")
    monkeypatch.setenv("RN_TMA", tma)
    monkeypatch.setenv("RN_MMA", "0")  # the chain-batched DMMA path only exists in placement 0
    runs = []
    for place in (0, 1):
        monkeypatch.setenv("RN_WPC_PLACE", str(place))
        r = _device_run(rir, cols, config, seeds)
        assert ("#define RN_WPC_PLACE %d\n" % place) in r["src"]
        runs.append(r)
    r0 = runs[0]
    for r in runs[1:]:
        assert np.array_equal(r["trace"][:, :, 1], r0["trace"][:, :, 1]) and np.array_equal(r["trace"][:, :, 3], r0["trace"][:, :, 3])
        assert r["stats"] == r0["stats"]
        if scatter:  # atomic adds of the Lookup adjoint: no fixed order between lanes
            assert parity.rel_err(r["samples"], r0["samples"], 1e-9) < 1e-11
            assert parity.rel_err(r["density"], r0["density"], 1e-9) < 1e-12
        else:
            assert np.array_equal(r["samples"], r0["samples"]) and np.array_equal(r["trace"], r0["trace"])
            assert np.array_equal(r["density"], r0["density"])
        assert np.array_equal(np.asarray(r["mass"]), np.asarray(r0["mass"]))


@pytest.mark.parametrize("tma", ["0", "2"])
def test_forced_placements_eight_schools_default_config(monkeypatch, tma):
    rir, cols = configs.eight_schools().compile(True)
    _forced(monkeypatch, rir, cols, api.SamplerConfig(iterations=20, warmupIterations=60), np.arange(40) + 3, tma)


@pytest.mark.parametrize("tma", ["0", "2"])
def test_forced_placements_logreg(monkeypatch, tma):
    prir, pcols = configs.logreg(300, 3).compile(False)
    _forced(monkeypatch, prir, pcols, _static(10, 3, 0.02), np.arange(40) + 9, tma)


@pytest.mark.parametrize("tma", ["0", "2"])
def test_forced_placements_poisson_glmm_scatter(monkeypatch, tma):
    prir, pcols = configs.poisson_glm(40, 640).compile(False)
    _forced(monkeypatch, prir, pcols, _static(10, 3, 0.005), np.arange(40) + 5, tma, scatter=True)


def test_forced_placements_optimizer(monkeypatch):
    prir, pcols = configs.logreg(700, 4).compile(False)
    monkeypatch.setenv("RN_WPC_K", "1")
    x0 = np.random.default_rng(2).normal(size=(6, 4)) * 0.3
    got = []
    for place in (0, 1):
        monkeypatch.setenv("RN_WPC_PLACE", str(place))
        cm = api.CudaModel(prir, pcols)
        got.append(cm.optimize(x0=x0, backend=abi.RN_BACKEND_WARP, eps=1e-5))
        cm.close()
    for g in got[1:]:
        for key in ("x", "f", "info", "evals"):
            assert np.array_equal(np.asarray(g[key]), np.asarray(got[0][key])), key

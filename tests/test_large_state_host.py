"""Placement of the warp-per-chain kernels' per-chain state (RN_WPC_PLACE, rn_sampler_wpc.cuh / rn_optimizer.cuh), on the
host emulation: 0 keeps it all in shared memory, 1 moves the chain vectors and the density scratch to global memory (the
cross-warp reduction slots stay in shared memory).  Moving state changes addresses, never arithmetic, so forced placement 1 is
bit-identical to placement 0; a model whose state does not fit shared memory gets placement 1 instead of a refusal."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.binding import OracleModel
from oracle.rainier_py.optimizer import lbfgs
from rainier_b200 import abi, api

import host_emulation as he

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _emit(monkeypatch, rir, cols, config, place, tma="0", k="1"):
    monkeypatch.setenv("RN_TMA", tma)
    monkeypatch.setenv("RN_WPC_K", k)
    if place is None:
        monkeypatch.delenv("RN_WPC_PLACE", raising=False)
    else:
        monkeypatch.setenv("RN_WPC_PLACE", str(place))
    cm = api.CudaModel(rir, cols, device=-1)
    src = cm.emit_source(config) if config is not None else cm.emit_optimizer_source(backend=abi.RN_BACKEND_WARP)
    monkeypatch.delenv("RN_WPC_PLACE", raising=False)
    return cm, src


def _placements_agree(monkeypatch, model, config, seeds, tol, primal=False, tma="0", k="1", scatter=False):
    """P0 and forced P1 give bit-identical densities, samples, accept decisions, step counts, stats and RNG states,
    and the oracle agrees with them as it does with the warp-per-chain kernels (test_sampler_host.py: _run_wpc).  scatter: the
    model's gradient has a Lookup adjoint, whose atomic adds from the lanes land in no fixed order (in any placement, and from
    run to run of one placement), so the values agree to rounding and every decision exactly."""
    rir, cols = model.compile(True)
    grir, gcols = model.compile(False) if primal else (rir, cols)
    config.backend = abi.RN_BACKEND_WARP
    cfg, keep = api.lower_config(config)
    om = OracleModel(rir, cols)
    q = np.random.default_rng(0).normal(size=(2, api.CudaModel(grir, gcols, device=-1).nVars)) * 0.3
    ref = om.sample(cfg, seeds=seeds, trace=True)
    runs = []
    for place in (0, 1):
        cm, src = _emit(monkeypatch, grir, gcols, config, place, tma, k)
        assert ("#define RN_WPC_PLACE %d\n" % place) in src and ("#define RN_WPC_K %s\n" % k) in src
        assert ("#define RN_TMA_STAGES %s\n" % tma) in src
        d, err = he.density(src, q, None, cm)
        assert err == 0
        runs.append((d, he.sample(src, cfg, seeds, cm)))
    d0, r0 = runs[0]
    for d, r in runs[1:]:
        if scatter:
            np.testing.assert_allclose(d, d0, rtol=1e-13, atol=0)
            np.testing.assert_allclose(r["samples"], r0["samples"], rtol=1e-11, atol=1e-13)
            for key in ("stats", "mass"):
                assert np.array_equal(r[key], r0[key]), key
            for col in (1, 3):  # accept decisions, leapfrog steps
                assert np.array_equal(r["trace"][:, :, col], r0["trace"][:, :, col])
        else:
            assert np.array_equal(d, d0)
            for key in ("samples", "trace", "stats", "mass"):
                assert np.array_equal(r[key], r0[key]), key
        assert r["mass_kind"] == r0["mass_kind"]
    assert np.array_equal(r0["trace"][:, :, 1], ref["trace"][:, :, 1]), "accept decisions differ from the oracle"
    assert np.array_equal(r0["trace"][:, :, 3], ref["trace"][:, :, 3]), "leapfrog step counts differ from the oracle"
    assert np.max(np.abs(r0["samples"] - ref["samples"]) / np.maximum(np.abs(ref["samples"]), 1e-9)) < tol
    for c, o in enumerate(ref["stats"]):
        assert r0["stats"][c, 0] == o.gradient_evaluations and r0["stats"][c, 3] == o.rng.seed48


def test_placements_bit_identical_eight_schools_default_config(monkeypatch):
    # DefaultConfig: EHMC, diagonal mass tuner, DualAvg -- every chain vector, the snapshot and the mass move
    _placements_agree(monkeypatch, configs.eight_schools(), api.SamplerConfig(iterations=12, warmupIterations=70), np.arange(2) + 3,
                      tol=1e-300)


def _poisson_cfg():
    return api.make_config(iterations=6, warmupIterations=0, sampler=api.HMCSampler(3), stepSizeTuner=api.StaticStepSize(0.005),
                           massMatrixTuner=api.IdentityMassMatrixTuner())


@pytest.mark.parametrize("k", ["1", "2"])
def test_placements_bit_identical_poisson_glmm_scatter(monkeypatch, k):
    # the Lookup adjoint's scatter-add into shared (P0) and global (P1) accumulators; with two warps per chain the
    # cross-warp reduction slots stay in shared memory while the rest of the scratch is in global memory (P1)
    _placements_agree(monkeypatch, configs.poisson_glm(40, 640), _poisson_cfg(), np.arange(2) + 5, tol=1e-8, primal=True, k=k,
                      scatter=True)


def test_placements_bit_identical_logreg_tile_pipeline(monkeypatch):
    # CTA-shared data tiles (two stages) beside a chain state in global memory
    cfg = api.make_config(iterations=6, warmupIterations=0, sampler=api.HMCSampler(3), stepSizeTuner=api.StaticStepSize(0.02),
                          massMatrixTuner=api.IdentityMassMatrixTuner())
    _placements_agree(monkeypatch, configs.logreg(300, 3), cfg, np.arange(2) + 9, tol=1e-9, primal=True, tma="2")


@pytest.mark.parametrize("k", ["1", "2"])
def test_optimizer_placements_bit_identical(monkeypatch, k):
    model = configs.logreg(700, 4)  # streamed rows, no scatter-add: every evaluation is deterministic
    prir, pcols = model.compile(False)
    rir, cols = model.compile(True)
    n = api.CudaModel(prir, pcols, device=-1).nVars
    x0 = np.random.default_rng(3).normal(size=(2, n)) * 0.1
    x0[0] = 0.0
    got = []
    for place in (0, 1):
        cm, src = _emit(monkeypatch, prir, pcols, None, place, k=k)
        assert ("#define RN_WPC_PLACE %d\n" % place) in src
        got.append(he.optimize(src, cm, x0, eps=1e-5, max_evals=200))
    for g in got[1:]:
        for key in ("x", "f", "info", "evals"):
            assert np.array_equal(g[key], got[0][key]), key
    ref = lbfgs(OracleModel(rir, cols).density_batch, n, eps=1e-5, max_evals=200)
    assert got[0]["info"][0] == ref["info"] == 0 and got[0]["evals"][0] == ref["evals"]
    np.testing.assert_allclose(got[0]["x"][0], ref["x"], rtol=1e-8, atol=1e-10)


# ---- which placement the sizes choose -------------------------------------------------------------------------------

def _three_configs():
    diag = api.DiagonalMassMatrixTuner(50, 1.5, 50, 50)
    return {
        "hmc_identity": api.make_config(10, 10, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                                        massMatrixTuner=api.IdentityMassMatrixTuner()),
        "hmc_diagonal": api.make_config(10, 10, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8), massMatrixTuner=diag),
        "ehmc_diagonal": api.make_config(10, 10, sampler=api.EHMCSampler(64), stepSizeTuner=api.DualAvgTuner(0.8), massMatrixTuner=diag),
    }


@pytest.fixture(scope="module")
def glmm_6000():
    # n = 6003: no placement-0 slice of any sampler configuration or of the optimizer fits 227 KB
    return configs.poisson_glm(6000, 12000).compile(False)


def test_above_the_shared_memory_limit_placement_1(glmm_6000, monkeypatch):
    prir, pcols = glmm_6000
    cm = api.CudaModel(prir, pcols, device=-1)
    for name, cfg in _three_configs().items():
        src = cm.emit_source(cfg)
        assert "#define RN_BACKEND 1\n" in src and "#define RN_WPC_PLACE 1\n" in src, name
    assert "#define RN_WPC_PLACE 1\n" in cm.emit_optimizer_source()
    monkeypatch.setenv("RN_WPC_PLACE", "0")  # forcing a lower placement than the sizes allow is refused
    with pytest.raises(Exception, match="RN_WPC_PLACE=0"):
        api.CudaModel(prir, pcols, device=-1).emit_source(_three_configs()["hmc_identity"])


def test_below_the_shared_memory_limit_placement_0():
    models = os.path.join(ROOT, "rainier_b200", "models")
    fixtures = [(open(os.path.join(models, f), "rb").read(), []) for f in
                ("eight_schools.rir", "eight_schools.primal.rir", "funnel10.rir", "funnel10.primal.rir")]
    for rir, cols in fixtures + [configs.poisson_glm(100, 1000).compile(False), configs.poisson_glm(1000, 4000).compile(False)]:
        cm = api.CudaModel(rir, cols, device=-1)
        for name, cfg in _three_configs().items():
            cfg.backend = abi.RN_BACKEND_WARP
            assert "#define RN_WPC_PLACE 0\n" in cm.emit_source(cfg), name
        assert "#define RN_WPC_PLACE 0\n" in cm.emit_optimizer_source(backend=abi.RN_BACKEND_WARP)


# ---- the sources compile for sm_90a, without new spills ------------------------------------------------------------

def _nvcc():
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    return cand if os.path.exists(cand) else shutil.which("nvcc")


def _ptxas_spills(src, tmp_path, name):
    cu = tmp_path / (name + ".cu")
    cu.write_text(src)
    r = subprocess.run([_nvcc(), "-cubin", "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "--fmad=false", "-Xptxas", "-v",
                        "-o", str(tmp_path / (name + ".cubin")), str(cu)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    spills, fn = {}, None
    for line in r.stderr.splitlines():
        if "Compiling entry function" in line:
            fn = line.split("'")[1]
        elif "spill stores" in line and fn:
            spills[fn] = int(line.split("bytes stack frame,")[1].split("bytes spill stores")[0])
    return spills


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not installed")
def test_placement_sources_compile_for_sm90a_without_new_spills(monkeypatch, tmp_path):
    prir, pcols = configs.poisson_glm(1000, 4000).compile(False)
    cfg = _three_configs()["ehmc_diagonal"]
    cfg.backend = abi.RN_BACKEND_WARP
    spills = {}
    for place in (0, 1):
        monkeypatch.setenv("RN_WPC_PLACE", str(place))
        cm = api.CudaModel(prir, pcols, device=-1)
        spills[place] = _ptxas_spills(cm.emit_source(cfg), tmp_path, "s%d" % place)
        spills[(place, "opt")] = _ptxas_spills(cm.emit_optimizer_source(backend=abi.RN_BACKEND_WARP), tmp_path, "o%d" % place)
    for fn, b in spills[1].items():
        assert b <= spills[0].get(fn, 0), (fn, b)
    for fn, b in spills[(1, "opt")].items():
        assert b <= spills[(0, "opt")].get(fn, 0), (fn, b)

"""
Pooled step-size adaptation on the device (rn_config.step_adaptation = RN_ADAPT_POOLED, rn_step_pool.cuh): against the
oracle's lockstep restatement (tests/pooled_step_oracle.cpp), across chain orders, kernel families (thread per chain, warp
per chain, the DMMA lockstep path), together with pooled mass windows, and through the one-call rn_sample path.
"""
import numpy as np
import pytest

from oracle.rainier_py import configs
from rainier_b200 import abi, api

import parity
import pooled_step as ps

pytestmark = pytest.mark.gpu


def _gpu(rir, cols, config, seeds):
    import torch

    cfg, keep = api.lower_config(config)
    gm = api.CudaModel(rir, cols, device=0)
    s = api.CudaSampler(gm, config, seeds=seeds, trace=True)
    d = torch.empty((max(cfg.iterations, 1), gm.nVars, s.chains), dtype=torch.float64, device="cuda:0")
    s.warmup(-1)
    s.run(cfg.iterations, d.data_ptr())
    s.sync()
    samples = d[: cfg.iterations].permute(2, 0, 1).contiguous().cpu().numpy()
    stats, mass = s.stats()
    trace = s.read_trace()
    s.close()
    gm.close()
    return {"samples": samples, "trace": trace, "stats": stats, "mass": mass}


def _pooled(config, backend=abi.RN_BACKEND_THREAD, **kw):
    config.stepAdaptation = abi.RN_ADAPT_POOLED
    config.backend = backend
    for k, v in kw.items():
        setattr(config, k, v)
    return config


def _shared_step(g, warmup):
    tr = g["trace"]
    assert np.all(tr[:, :, 2] == tr[:1, :, 2]), "chains ran different step sizes"
    assert all(x.stepSize == g["stats"][0].stepSize for x in g["stats"]), "stats.step_size differs between chains"


def _vs_oracle(model, config, seeds, dense=False):
    rir, cols = model.compile(True)
    cfg, keep = api.lower_config(config)
    g = _gpu(rir, cols, config, seeds)
    ref = ps.oracle_sample(rir, cols, cfg, seeds, dense_mass=dense)
    r = {"gpu": g["samples"], "ref": ref["samples"], "gpu_trace": g["trace"], "ref_trace": ref["trace"], "gpu_stats": g["stats"],
         "ref_stats": ref["stats"], "gpu_mass": g["mass"], "ref_mass": ref["mass"]}
    parity.assert_parity(r, tol=1e-9)
    _shared_step(g, cfg.warmup_iterations)
    return g


def test_eight_schools_default_config_matches_the_oracle():
    """EHMC + DualAvg + diagonal windows (the pooled step is reset at each window end), 256 chains"""
    _vs_oracle(configs.eight_schools(), _pooled(api.SamplerConfig(iterations=60, warmupIterations=320)), np.arange(256) + 11)


def test_funnel_hmc_many_ctas_matches_the_oracle():
    """HMC(5) + DualAvg + identity mass, 1024 chains: the sums span many CTAs and warps"""
    cfg = api.make_config(iterations=30, warmupIterations=150, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                          massMatrixTuner=api.IdentityMassMatrixTuner())
    _vs_oracle(configs.funnel(), _pooled(cfg), np.arange(1024) + 5)


def test_reversed_seeds_give_reversed_outputs_on_the_device():
    rir, cols = configs.eight_schools().compile(True)
    seeds = (np.arange(384, dtype=np.int64) * 7919) % 100003 + 1
    mk = lambda: _pooled(api.SamplerConfig(iterations=40, warmupIterations=200))  # noqa: E731
    a, b = _gpu(rir, cols, mk(), seeds), _gpu(rir, cols, mk(), seeds[::-1].copy())
    assert np.array_equal(a["samples"], b["samples"][::-1])
    assert np.array_equal(a["trace"], b["trace"][::-1])


def test_warp_backend_is_bit_identical_to_the_thread_backend():
    rir, cols = configs.eight_schools().compile(True)
    seeds = np.arange(200) + 21
    t = _gpu(rir, cols, _pooled(api.SamplerConfig(iterations=40, warmupIterations=220)), seeds)
    w = _gpu(rir, cols, _pooled(api.SamplerConfig(iterations=40, warmupIterations=220), abi.RN_BACKEND_WARP), seeds)
    assert np.array_equal(t["trace"], w["trace"])
    assert np.array_equal(t["samples"], w["samples"])
    _shared_step(w, 220)


def _eps0_is_a_pooled_power_of_two(eps0, chains):
    """eps0 = exp(ln2 * K / C) for an integer K (step 1); the kernels' exp is the oracle's"""
    k = int(round(np.log2(eps0) * chains))
    return any(float(ps._vec(0, ps.LN2 * (kk / chains))[0]) == eps0 for kk in (k - 1, k, k + 1))


def test_dmma_lockstep_path_replays_on_the_host():
    """streamed logistic regression on the chain-batched DMMA path (HMC: full CTAs in lockstep): the step sequence replayed
    on the host from the traced log acceptance probabilities (steps 2-4, the oracle's exp / pow) equals the traced one"""
    model = configs.logreg(1500, 6)
    prir, pcols = model.compile(False)
    cfg = api.make_config(iterations=20, warmupIterations=120, sampler=api.HMCSampler(4), stepSizeTuner=api.DualAvgTuner(0.8),
                          massMatrixTuner=api.IdentityMassMatrixTuner())
    _pooled(cfg, abi.RN_BACKEND_WARP)
    assert "rn_dmma(z" in api.CudaModel(prir, pcols, device=-1).emit_source(cfg), "the model should take the DMMA path"
    chains = 67  # 4 full CTAs of 16 and a ragged tail on the per-warp path: both launches add into the same slot
    g = _gpu(prir, pcols, cfg, np.arange(chains) + 3)
    tr = g["trace"]
    _shared_step(g, 120)
    eps0 = float(tr[0, 0, 2])
    assert _eps0_is_a_pooled_power_of_two(eps0, chains)
    used, final = ps.replay_steps(tr[:, :120, 0], 120, 0.8, set(), eps0)
    assert np.array_equal(used, tr[0, :120, 2]), "replayed step sequence differs"
    assert final == tr[0, -1, 2]  # sampling runs at exp(logStepSizeBar)


def test_with_pooled_mass_windows_replays_on_the_host():
    """adaptation = RN_ADAPT_POOLED as well: every chain ends warmup with the same mass matrix and step size; the host replay,
    including the resets at the (pooled) window ends, matches the trace"""
    rir, cols = configs.eight_schools().compile(True)
    config = _pooled(api.SamplerConfig(iterations=40, warmupIterations=300), adaptation=abi.RN_ADAPT_POOLED)
    cfg, keep = api.lower_config(config)
    chains = 256
    g = _gpu(rir, cols, config, np.arange(chains) + 1)
    tr = g["trace"]
    _shared_step(g, 300)
    assert np.all(g["mass"] == g["mass"][:1]), "chains ended warmup with different mass matrices"
    closes = ps.window_closes(cfg)
    assert len(closes) >= 2
    eps0 = float(tr[0, 0, 2])
    assert _eps0_is_a_pooled_power_of_two(eps0, chains)
    used, final = ps.replay_steps(tr[:, :300, 0], 300, 0.8, closes, eps0)
    assert np.array_equal(used, tr[0, :300, 2]), "replayed step sequence differs"
    assert final == tr[0, -1, 2]  # sampling runs at exp(logStepSizeBar)


def test_one_call_sample_equals_the_staged_sampler():
    rir, cols = configs.eight_schools().compile(True)
    seeds = np.arange(128, dtype=np.int64) + 9
    config = _pooled(api.SamplerConfig(iterations=50, warmupIterations=200))
    staged = _gpu(rir, cols, config, seeds)
    m = api.CudaModel(rir, cols, device=0)
    tr = m.sample(config, seeds=seeds)
    m.close()
    assert np.array_equal(np.asarray(tr.chains), staged["samples"])
    assert all(a.stepSize == b.stepSize for a, b in zip(tr.stats, staged["stats"]))

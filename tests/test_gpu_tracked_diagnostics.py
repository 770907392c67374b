"""Tracked diagnostics on the device (rn_sampler_track_diagnostics / rn_sampler_tracked_diagnostics): Trace.thin(thin).diagnostics
accumulated while sampling, with no sample block kept.
  * Any split of a run into rn_sampler_run calls gives the same bits, with or without a sample block.
  * The result agrees with rn_sampler_diagnostics over the same draws (the variance is Welford here, two-pass there) and
    with the restatement of Trace.diagnostics; the ESS loop's terminating autocorrelation is checked to be away from 0, so
    that an agreement within the tolerance cannot hide a different number of lags.
  * Tracking changes neither the samples nor rn_sampler_launches, and each error path returns RN_E_INVALID.
"""
import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.diagnostics import r_hat_and_v, sum_seq, variogram
from oracle.rainier_py.diagnostics import trace_diagnostics
from rainier_b200 import abi, api

import parity

pytestmark = pytest.mark.gpu

SPLITS = ([1000], [1, 1, 98, 400, 500], [37] * 27 + [1])


def _models():
    out = {}
    rir, cols = configs.eight_schools().compile(True)
    out["schools"] = (rir, cols, api.SamplerConfig(iterations=1000, warmupIterations=300), 32)
    rir, cols = configs.funnel(10).compile(True)
    out["funnel"] = (rir, cols, api.HMC(300, 1000, 5), 32)
    model = configs.logreg(1500, 6)
    rir, cols = model.compile(False)
    out["logreg"] = (rir, cols, api.make_config(iterations=1000, warmupIterations=100, sampler=api.HMCSampler(4),
                                                stepSizeTuner=api.StaticStepSize(0.01), backend=abi.RN_BACKEND_WARP), 24)
    return out


MODELS = _models()


@pytest.fixture(scope="module")
def runs():
    """per model: the samples of one untracked run [iterations][n][chains] and its launch count"""
    import torch
    out = {}
    for key, (rir, cols, config, chains) in MODELS.items():
        m = api.CudaModel(rir, cols)
        s = api.CudaSampler(m, config, seeds=np.arange(chains) + 5)
        d = torch.empty((1000, m.nVars, chains), dtype=torch.float64, device="cuda")
        s.warmup(-1)
        s.run(1000, d.data_ptr())
        s.sync()
        launches = s.launches
        block = s.diagnostics(d.data_ptr(), 1000, layout=0)
        out[key] = {"d": d, "launches": launches, "block": block, "model": m}
        s.close()
    return out


def _tracked(key, split, keep, thin=1):
    import torch
    rir, cols, config, chains = MODELS[key]
    m = api.CudaModel(rir, cols)
    s = api.CudaSampler(m, config, seeds=np.arange(chains) + 5)
    s.warmup(-1)
    s.track_diagnostics(thin)
    parts = []
    for k in split:
        d = torch.empty((k, m.nVars, chains), dtype=torch.float64, device="cuda") if keep else None
        s.run(k, d.data_ptr() if keep else None)
        if keep:
            parts.append(d)
    launches = s.launches
    got = s.tracked_diagnostics()
    s.close()
    samples = torch.cat(parts, 0) if keep else None
    return got, launches, samples


def _terminating_pt(chains):
    """the autocorrelation at which Trace.autocorrelation stops, per parameter (restated, Trace.scala:97-109)"""
    out = []
    for i in range(chains.shape[2]):
        traces = [[float(a[i]) for a in c] for c in chains]
        n, m = float(len(traces[0])), float(len(traces))
        _, v = r_hat_and_v(traces, n, m)
        lag = 1
        while True:
            pt = 1.0 - (sum_seq([variogram(t, lag) for t in traces]) / m / (2.0 * v))
            if not (pt > 0.0 and lag < 100):
                out.append((lag, pt))
                break
            lag += 1
    return out


@pytest.mark.parametrize("key", list(MODELS))
def test_chunk_invariance_and_parity(runs, key):
    ref_run = runs[key]
    outs = []
    for split in SPLITS:
        for keep in (True, False):
            got, launches, samples = _tracked(key, split, keep)
            outs.append(got)
            if keep and split == SPLITS[0]:
                assert launches == ref_run["launches"], "tracking must not change rn_sampler_launches"
                assert samples.cpu().numpy().tobytes() == ref_run["d"].cpu().numpy().tobytes(), "tracking changed the samples"
    for o in outs[1:]:
        assert o.tobytes() == outs[0].tobytes(), "the split into rn_sampler_run calls changed the result"
    got = outs[0]
    assert parity.rel_err(got, ref_run["block"], 1e-12) < 1e-12, (got, ref_run["block"])
    chains = ref_run["d"].permute(2, 0, 1).contiguous().cpu().numpy()
    ref = np.array(trace_diagnostics(chains))
    assert parity.rel_err(got, ref, 1e-9) < 1e-9, (got, ref)
    for lag, pt in _terminating_pt(chains):
        assert lag == 100 or not abs(pt) < 1e-9, (lag, pt)


@pytest.mark.parametrize("thin", [2, 3, 7])
def test_thinned_matches_restatement(runs, thin):
    got, _, _ = _tracked("schools", [1, 250, 749], False, thin=thin)
    chains = runs["schools"]["d"].permute(2, 0, 1).contiguous().cpu().numpy()[:, ::thin]
    ref = np.array(trace_diagnostics(chains))
    assert parity.rel_err(got, ref, 1e-9) < 1e-9, (got, ref)
    got_split, _, _ = _tracked("schools", [500, 500], True, thin=thin)
    assert got_split.tobytes() == got.tobytes()


def test_restart_and_untracked_run_unchanged(runs):
    """a second track call restarts the accumulation; runs before it are not tracked"""
    import torch
    rir, cols, config, chains = MODELS["schools"]
    m = api.CudaModel(rir, cols)
    s = api.CudaSampler(m, config, seeds=np.arange(chains) + 5)
    s.warmup(-1)
    s.track_diagnostics(5)
    s.run(400)
    s.track_diagnostics(1)
    d = torch.empty((600, m.nVars, chains), dtype=torch.float64, device="cuda")
    s.run(600, d.data_ptr())
    got = s.tracked_diagnostics()
    s.close()
    assert np.array_equal(d.cpu().numpy(), runs["schools"]["d"][400:].cpu().numpy())
    ref = np.array(trace_diagnostics(d.permute(2, 0, 1).contiguous().cpu().numpy()))
    assert parity.rel_err(got, ref, 1e-9) < 1e-9


def test_errors():
    rir, cols, _, _ = MODELS["schools"]
    m = api.CudaModel(rir, cols)
    cfg = api.SamplerConfig(iterations=10, warmupIterations=10)
    s = api.CudaSampler(m, cfg, seeds=np.arange(4) + 1)
    with pytest.raises(api.RainierCudaError, match="before rn_sampler_track_diagnostics") as e:
        s.tracked_diagnostics()
    assert e.value.code == abi.RN_E_INVALID
    for thin in (0, -3):
        with pytest.raises(api.RainierCudaError, match="thin") as e:
            s.track_diagnostics(thin)
        assert e.value.code == abi.RN_E_INVALID
    s.warmup(-1)
    s.track_diagnostics(3)
    s.run(4)  # kept: draws 0 and 3 -> 2
    assert s.tracked_diagnostics().shape == (m.nVars, 2)
    s.track_diagnostics(3)
    s.run(3)  # kept: draw 0 only
    with pytest.raises(api.RainierCudaError, match="at least 2 kept draws") as e:
        s.tracked_diagnostics()
    assert e.value.code == abi.RN_E_INVALID
    s.close()
    one = api.CudaSampler(m, cfg, seeds=np.arange(1) + 1)
    one.warmup(-1)
    one.track_diagnostics(1)
    one.run(10)
    with pytest.raises(api.RainierCudaError, match="Trace.scala:12") as e:
        one.tracked_diagnostics()
    assert e.value.code == abi.RN_E_INVALID
    one.close()

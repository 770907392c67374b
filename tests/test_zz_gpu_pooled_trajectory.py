"""
Pooled EHMC trajectory lengths on the device (rn_config.trajectory_adaptation = RN_ADAPT_POOLED, rn_sampler_common.cuh).
Warmup is the per-chain warmup, bit for bit; the pooled histogram is the histogram of the chains' rings read back from a
checkpoint; every chain's sampling iteration t takes L_t steps as tests/pooled_traj.py restates it; and the mode runs through
both kernel shapes, the DMMA path, rn_sample's chain blocks, the other pooled modes and checkpoints.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from oracle.rainier_py import configs
from oracle.rainier_py.compute import Real
from oracle.rainier_py.core import Model, Normal
from rainier_b200 import abi, api

import parity
import pooled_traj as pt

pytestmark = pytest.mark.gpu


def _cfg(iterations, warmup, pooled=True, **kw):
    kw.setdefault("backend", abi.RN_BACKEND_THREAD)
    c = api.SamplerConfig(iterations=iterations, warmupIterations=warmup, **kw)
    if pooled:
        c.trajectoryAdaptation = abi.RN_ADAPT_POOLED
    return c


def _gpu(rir, cols, config, seeds, split=None, keep_blob=False, track=False):
    """warmup, then the sampling iterations in the calls `split` (default one); samples [chains][iterations][n], trace, stats,
    mass, launches after warmup and after sampling, the pooled histogram (pooled mode), a checkpoint taken at the end
    (keep_blob) and the tracked diagnostics of the sampling phase (track)"""
    import torch

    cfg, keep = api.lower_config(config)
    gm = api.CudaModel(rir, cols, device=0)
    s = api.CudaSampler(gm, config, seeds=seeds, trace=True)
    d = torch.empty((max(cfg.iterations, 1), gm.nVars, s.chains), dtype=torch.float64, device="cuda:0")
    s.warmup(-1)
    s.sync()
    launches = [s.launches]
    if track:
        s.track_diagnostics(1)
    done = 0
    for k in (split or [cfg.iterations]):
        s.run(k, d[done:].data_ptr())
        done += k
    s.sync()
    launches.append(s.launches)
    stats, mass = s.stats()
    out = {"samples": d[: cfg.iterations].permute(2, 0, 1).contiguous().cpu().numpy(), "trace": s.read_trace(), "stats": stats,
           "mass": mass, "launches": launches}
    if track:
        out["diagnostics"] = np.asarray(s.tracked_diagnostics())
    if config.trajectoryAdaptation == abi.RN_ADAPT_POOLED and cfg.iterations > 0:
        out["hist"] = s.trajectory_lengths()
    if keep_blob:
        out["blob"] = bytes(s.save())
    s.close()
    gm.close()
    return out


def _vs_oracle(rir, cols, config, seeds, g, tol):
    """the device run g against the oracle's restatement: equal histograms, accept decisions and trajectory lengths, the rest
    within tol (parity.assert_parity)"""
    cfg, keep = api.lower_config(config)
    ref = pt.oracle_sample(rir, cols, cfg, seeds)
    assert np.array_equal(g["hist"], ref["hist"]), "pooled histogram differs from the oracle's"
    parity.assert_parity({"gpu": g["samples"], "ref": ref["samples"], "gpu_trace": g["trace"], "ref_trace": ref["trace"],
                          "gpu_stats": g["stats"], "ref_stats": ref["stats"], "gpu_mass": g["mass"], "ref_mass": ref["mass"]}, tol=tol)
    return ref


def _check_lengths(g, warmup):
    """every chain's sampling iteration t took L_t steps of the pooled histogram"""
    L = pt.lengths(g["hist"], 0, g["trace"].shape[1] - warmup)
    assert np.array_equal(api.trajectory_lengths_sequence(g["hist"], 0, len(L)), L)
    assert np.all(g["trace"][:, warmup:, 3] == L[None, :]), "a chain's sampling trajectory length differs from L_t"


def test_thread_shape_pools_the_per_chain_warmup():
    """eight schools, DefaultConfig, 1000 chains (a ragged last CTA): bit for bit against the oracle's restatement (samples,
    traces, RNG states, stats, histogram), warmup bit-identical to per-chain EHMC, the histogram is the histogram of the rings in
    a checkpoint, sampling runs L_t"""
    rir, cols = configs.eight_schools().compile(True)
    seeds = np.arange(1000, dtype=np.int64) + 17
    p = _gpu(rir, cols, _cfg(40, 150), seeds, keep_blob=True)
    ref = _vs_oracle(rir, cols, _cfg(40, 150), seeds, p, tol=1e-12)
    assert np.array_equal(p["samples"], ref["samples"]) and np.array_equal(p["trace"], ref["trace"]), "not bit-identical to the oracle"
    q = _gpu(rir, cols, _cfg(40, 150, pooled=False), seeds)
    assert np.array_equal(p["trace"][:, :150], q["trace"][:, :150]), "warmup differs from the per-chain warmup"
    assert np.array_equal(p["hist"], pt.checkpoint_ring_histogram(p["blob"]))
    assert np.array_equal(p["hist"], pt.checkpoint_histogram(p["blob"]))
    assert p["hist"].sum() >= 1000 and len(p["hist"]) == 1025
    _check_lengths(p, 150)
    assert np.all(np.isfinite(p["samples"]))
    for st in p["stats"]:
        assert st.leapfrogSteps == int(p["trace"][0, 150:, 3].sum())


def test_split_calls_and_reversed_seeds():
    rir, cols = configs.eight_schools().compile(True)
    seeds = (np.arange(300, dtype=np.int64) * 7919) % 100003 + 1
    a = _gpu(rir, cols, _cfg(30, 120), seeds)
    b = _gpu(rir, cols, _cfg(30, 120), seeds, split=[7, 1, 22])
    r = _gpu(rir, cols, _cfg(30, 120), seeds[::-1].copy())
    assert np.array_equal(a["samples"], b["samples"]) and np.array_equal(a["trace"], b["trace"])
    assert np.array_equal(a["hist"], r["hist"])
    assert np.array_equal(a["samples"], r["samples"][::-1]) and np.array_equal(a["trace"], r["trace"][::-1])


def test_no_warmup_samples_zero_steps():
    """warmup_iterations = 0: every ring offers its slot 0 (value 0), so L_t = 0 throughout, as per-chain EHMC"""
    rir, cols = configs.eight_schools().compile(True)
    seeds = np.arange(64, dtype=np.int64) + 3
    g = _gpu(rir, cols, _cfg(20, 0), seeds)
    assert g["hist"][0] == 64 and g["hist"][1:].sum() == 0
    assert np.all(g["trace"][:, :, 3] == 0)


def test_warp_shape_is_bit_identical_to_the_thread_shape():
    rir, cols = configs.eight_schools().compile(True)
    seeds = np.arange(200, dtype=np.int64) + 21
    t = _gpu(rir, cols, _cfg(40, 150), seeds)
    w = _gpu(rir, cols, _cfg(40, 150, backend=abi.RN_BACKEND_WARP), seeds)
    assert np.array_equal(t["hist"], w["hist"])
    assert np.array_equal(t["trace"], w["trace"])
    assert np.array_equal(t["samples"], w["samples"])


def test_dmma_path_samples_in_lockstep():
    """streamed logistic regression at 16-chain groups and a ragged tail: the pooled module takes the DMMA path (per-chain EHMC
    does not) and every chain's sampling iteration runs L_t"""
    model = configs.logreg(1500, 6)
    prir, pcols = model.compile(False)
    mk = lambda pooled: _cfg(20, 100, pooled=pooled, backend=abi.RN_BACKEND_WARP,  # noqa: E731
                             _massMatrixTuner=api.IdentityMassMatrixTuner())
    chains = 67
    p = _gpu(prir, pcols, mk(True), np.arange(chains) + 3, keep_blob=True)
    assert api.checkpoint_info(p["blob"])["mma"] == 1, "the pooled module should take the DMMA path"
    # which path each phase took, from the launches: rn_k_init and ONE warmup launch of all 67 chains (tma = 0: the per-warp
    # body), then rn_k_traj_hist and the sampling launch split into the 4 full 16-chain groups on the DMMA / TMA lockstep path
    # and the ragged tail of 3 chains on the per-warp path
    assert p["launches"] == [2, 5], p["launches"]
    _check_lengths(p, 100)
    # against the oracle's restatement: the histogram, accept decisions, U-turn counts and trajectory lengths equal; values
    # within 1e-3.  The density's row sums are tree-ordered on this shape, and each chain's DualAvg warmup turns those
    # last-bit differences in the acceptance probabilities into step sizes that differ by about 4e-5 (relative) after 100
    # iterations, which carries into the samples (and, through cancellation, further into the energy statistics, left out)
    cfg, keep = api.lower_config(mk(True))
    ref = pt.oracle_sample(prir, pcols, cfg, np.arange(chains) + 3)
    assert np.array_equal(p["hist"], ref["hist"]), "pooled histogram differs from the oracle's"
    assert np.array_equal(p["trace"][:, :, 1], ref["trace"][:, :, 1]), "accept decisions differ from the oracle's"
    assert np.array_equal(p["trace"][:, :, 3], ref["trace"][:, :, 3]), "U-turn counts / trajectory lengths differ from the oracle's"
    for g, o in zip(p["stats"], ref["stats"]):
        assert (g.gradientEvaluations, g.leapfrogSteps, g.accepted, g.rng[0]) == (o.gradient_evaluations, o.leapfrog_steps, o.accepted,
                                                                                  o.rng.seed48)
    assert parity.rel_err(p["trace"][:, :, 2], ref["trace"][:, :, 2]) < 1e-3
    assert parity.rel_err(p["samples"], ref["samples"]) < 1e-3
    q = _gpu(prir, pcols, mk(False), np.arange(chains) + 3, keep_blob=True)
    assert api.checkpoint_info(q["blob"])["mma"] == 0, "per-chain EHMC keeps the per-warp path"
    assert q["launches"] == [2, 3], q["launches"]  # one launch of all chains per phase


def test_one_call_sample_equals_the_staged_sampler(monkeypatch):
    rir, cols = configs.eight_schools().compile(True)
    seeds = np.arange(3000, dtype=np.int64) + 9
    config = _cfg(30, 100)
    staged = _gpu(rir, cols, config, seeds)
    for blocks in (None, "3"):
        if blocks:
            monkeypatch.setenv("RN_SAMPLE_BLOCKS", blocks)
        m = api.CudaModel(rir, cols, device=0)
        tr = m.sample(config, seeds=seeds)
        m.close()
        assert np.array_equal(np.asarray(tr.chains), staged["samples"]), "rn_sample with RN_SAMPLE_BLOCKS=%s" % blocks


def test_with_pooled_steps_and_pooled_mass_windows():
    rir, cols = configs.eight_schools().compile(True)
    seeds = np.arange(256, dtype=np.int64) + 1
    kw = dict(stepAdaptation=abi.RN_ADAPT_POOLED, adaptation=abi.RN_ADAPT_POOLED)
    p = _gpu(rir, cols, _cfg(30, 200, **kw), seeds)
    q = _gpu(rir, cols, _cfg(30, 200, pooled=False, **kw), seeds)
    assert np.array_equal(p["trace"][:, :200], q["trace"][:, :200])
    _check_lengths(p, 200)
    assert np.all(p["trace"][:, 200:, 2] == p["trace"][:1, 200:, 2])


def _continue(rir, cols, config, blobs, iterations):
    import torch

    gm = api.CudaModel(rir, cols, device=0)
    s = api.CudaSampler.restore(gm, config, blobs)
    d = torch.empty((iterations, gm.nVars, s.chains), dtype=torch.float64, device="cuda:0")
    s.run(iterations, d.data_ptr())
    s.sync()
    out = d.permute(2, 0, 1).contiguous().cpu().numpy(), s.trajectory_lengths()
    s.close()
    gm.close()
    return out


_RESTORE_SCRIPT = r"""
import sys
import numpy as np
import torch
from oracle.rainier_py import configs
from rainier_b200 import abi, api
blob, out, it = open(sys.argv[1], "rb").read(), sys.argv[2], int(sys.argv[3])
config = api.SamplerConfig(iterations=40, warmupIterations=120, backend=abi.RN_BACKEND_THREAD, trajectoryAdaptation=abi.RN_ADAPT_POOLED)
rir, cols = configs.eight_schools().compile(True)
gm = api.CudaModel(rir, cols, device=0)
s = api.CudaSampler.restore(gm, config, [blob], trace=True)
d = torch.empty((it, gm.nVars, s.chains), dtype=torch.float64, device="cuda:0")
s.run(it, d.data_ptr())
s.sync()
tr = s.read_trace()
np.savez(out, samples=d.permute(2, 0, 1).contiguous().cpu().numpy(), steps=tr[:, :it, 3])
s.close()
gm.close()
"""


def _continue_in_another_process(blob, iterations):
    """restores `blob` in a fresh Python process and runs `iterations` sampling iterations: (samples, traced lengths)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory() as d:
        src, out = os.path.join(d, "blob"), os.path.join(d, "out.npz")
        with open(src, "wb") as f:
            f.write(blob)
        env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
        subprocess.run([sys.executable, "-c", _RESTORE_SCRIPT, src, out, str(iterations)], check=True, cwd=root, env=env)
        z = np.load(out)
        return z["samples"], z["steps"]


def test_checkpoints_continue_bit_for_bit():
    """saved after warmup (before the histogram exists) and mid-sampling, restored in a fresh model, continued; a slice carries
    the histogram and continues as those chains of the full run; blobs with different histograms are not concatenated"""
    import torch

    rir, cols = configs.eight_schools().compile(True)
    seeds = np.arange(96, dtype=np.int64) + 5
    config = _cfg(40, 120)
    full = _gpu(rir, cols, config, seeds)
    gm = api.CudaModel(rir, cols, device=0)
    s = api.CudaSampler(gm, config, seeds=seeds)
    s.warmup(-1)
    after_warmup = bytes(s.save())
    h0 = pt.checkpoint_records(after_warmup)[0]
    assert h0.reserved0 == abi.RN_ADAPT_POOLED and h0.reserved1 == 0
    with pytest.raises(api.RainierCudaError):
        api.checkpoint_slice(after_warmup, 0, 32)  # the slice's own histogram would differ
    d = torch.empty((15, gm.nVars, 96), dtype=torch.float64, device="cuda:0")
    s.run(15, d.data_ptr())
    mid = bytes(s.save())
    s.close()
    gm.close()
    h1 = pt.checkpoint_records(mid)[0]
    assert h1.reserved0 == abi.RN_ADAPT_POOLED and h1.reserved1 == 8 * 1025
    assert np.array_equal(pt.checkpoint_histogram(mid), full["hist"])

    got, hist = _continue(rir, cols, config, [after_warmup], 40)
    assert np.array_equal(got, full["samples"]) and np.array_equal(hist, full["hist"])
    got, _ = _continue(rir, cols, config, [mid], 25)
    assert np.array_equal(got, full["samples"][:, 15:])
    got, steps = _continue_in_another_process(mid, 25)
    assert np.array_equal(got, full["samples"][:, 15:])
    assert np.all(steps == pt.lengths(full["hist"], 15, 25)[None, :]), "the restored run's lengths are not L_t from t = 15"
    part = bytes(api.checkpoint_slice(mid, 32, 64))
    got, hist = _continue(rir, cols, config, [part], 25)
    assert np.array_equal(hist, full["hist"])
    assert np.array_equal(got, full["samples"][32:64, 15:])

    other = _gpu(rir, cols, config, seeds + 1000, keep_blob=True)["blob"]
    assert not np.array_equal(pt.checkpoint_histogram(other), full["hist"])
    gm = api.CudaModel(rir, cols, device=0)
    with pytest.raises(api.RainierCudaError) as e:
        api.CudaSampler.restore(gm, config, [mid, other])
    assert e.value.code == abi.RN_E_INVALID
    gm.close()


def _correlated_gaussian(rho):
    """(x0, x1) ~ N(0, [[1, rho], [rho, 1]]) written as x0 ~ N(0, 1), x1 | x0 ~ N(rho x0, sqrt(1 - rho^2))"""
    s = float(np.sqrt(1.0 - rho * rho))
    th = Real.parameters(2, lambda t: Normal(0, 1).logDensity(t[0]) + Normal(t[0] * rho, s).logDensity(t[1]))
    return Model.track_(list(th))


def test_correct_distribution_on_a_correlated_gaussian():
    """4096 chains of pooled EHMC on a correlated Gaussian with known moments: every mean, variance and the covariance lie
    within 5 standard errors set by the tracked effective sample size (Var of a mean sigma^2 / ESS, of a variance about
    2 sigma^4 / ESS, of the covariance about (1 + rho^2) / ESS)"""
    rho = 0.8
    rir, cols = _correlated_gaussian(rho).compile(True)
    g = _gpu(rir, cols, _cfg(300, 300), np.arange(4096, dtype=np.int64) + 101, track=True)
    x = g["samples"].reshape(-1, 2)
    ess = g["diagnostics"][:, 1]
    assert np.all(g["diagnostics"][:, 0] < 1.01), g["diagnostics"]
    assert np.all(np.abs(x.mean(axis=0)) < 5 * np.sqrt(1.0 / ess)), (x.mean(axis=0), ess)
    assert np.all(np.abs(x.var(axis=0) - 1.0) < 5 * np.sqrt(2.0 / ess)), (x.var(axis=0), ess)
    cov = float(np.mean(x[:, 0] * x[:, 1]))
    assert abs(cov - rho) < 5 * np.sqrt((1 + rho * rho) / ess.min()), (cov, ess)
    _check_lengths(g, 300)

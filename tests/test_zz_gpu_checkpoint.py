"""Checkpoints on the device (rn_sampler_save / rn_sampler_restore).  Every case compares an uninterrupted staged run with
create -> warmup / run -> save -> destroy -> restore -> continue: samples, rn_sampler_stats (every counter and ring, the RNG
state, the mass matrix), the concatenated per-iteration trace and tracked diagnostics must be bit-identical.  The device-time
fields are the exception, and the Poisson GLMM, whose scatter-add atomics are unordered even without a cut: there the
decisions must be equal and the values equal to rounding."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.rainier_py import configs
from rainier_b200 import abi, api

import parity

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DMMA = "rn_dmma(z"
TIME_FIELDS = ("gradient_time_ns_mean", "iteration_time_ns_mean")


class _Env:
    def __init__(self, env):
        self.env = env or {}

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.env}
        os.environ.update(self.env)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _stats(s):
    n = s.model.nVars
    cfg = s.cfg
    dense = cfg.mass_tuner == abi.RN_MASS_DENSE
    st = (abi.ChainStats * s.chains)()
    mass = np.empty((s.chains, n * n if dense else n), dtype=np.float64)
    rings = np.zeros((s.chains, 3, cfg.stats_window), dtype=np.float64)
    api._check(api.lib().rn_sampler_stats(s.h, C.cast(st, C.c_void_p), mass.ctypes.data, rings.ctypes.data))
    fields = {}
    for f, t in abi.ChainStats._fields_:
        if f in TIME_FIELDS:
            continue
        if f == "rng":
            fields["rng"] = np.array([(x.rng.seed48, x.rng.next_gaussian, x.rng.have_next) for x in st], dtype=object)
        elif f in ("ring_pos", "ring_full"):
            fields[f] = np.array([list(getattr(x, f)) for x in st])
        else:
            fields[f] = np.array([getattr(x, f) for x in st])
    return fields, mass, rings


def _run(model, config, seeds, plan, cut=None, restore_env=None, restore_model=None, restore_config=None):
    """plan: steps ("w", k) warmup, ("r", k) run, ("t", thin) track diagnostics.  cut: save -> destroy -> restore before
    plan[cut].  Returns samples [chains][draws][n], trace [chains][iterations][4], stats, mass, rings, tracked diagnostics."""
    import torch
    s = api.CudaSampler(model, config, seeds=seeds, trace=True)
    draws, traces, pos, tracked = [], [], 0, False
    for k, (op, x) in enumerate(plan):
        if k == cut:
            traces.append(s.read_trace()[:, :pos])
            blob = s.save()
            s.close()
            with _Env(restore_env):
                s = api.CudaSampler.restore(restore_model or model, restore_config or config, blob, trace=True)
            pos = 0
        if op == "w":
            s.warmup(x)
            pos += x
        elif op == "r":
            d = torch.empty((x, model.nVars, s.chains), dtype=torch.float64, device="cuda")
            s.run(x, d.data_ptr())
            draws.append(d)
            pos += x
        else:
            s.track_diagnostics(x)
            tracked = True
    s.sync()
    traces.append(s.read_trace()[:, :pos])
    out = {"samples": torch.cat(draws, 0).permute(2, 0, 1).cpu().numpy() if draws else None,
           "trace": np.concatenate(traces, axis=1)}
    out["stats"], out["mass"], out["rings"] = _stats(s)
    out["diag"] = s.tracked_diagnostics() if tracked else None
    s.close()
    return out


def _same(a, b, exact=True):
    if exact:
        for k in ("samples", "trace", "mass", "rings", "diag"):
            if a[k] is not None or b[k] is not None:
                assert np.array_equal(a[k], b[k], equal_nan=True), "%s differ" % k
        for f in a["stats"]:
            assert np.array_equal(a["stats"][f], b["stats"][f]), "rn_chain_stats.%s differs" % f
        return
    for col in (1, 3):  # decisions, leapfrog steps
        assert np.array_equal(a["trace"][:, :, col], b["trace"][:, :, col])
    assert parity.rel_err(a["samples"], b["samples"], 1e-9) < 1e-9
    for f in ("gradient_evaluations", "leapfrog_steps", "accepted", "iterations", "rng"):
        assert np.array_equal(a["stats"][f], b["stats"][f]), f


def _check(model, config, seeds, plan, cuts, exact=True, **kw):
    ref = _run(model, config, seeds, plan)
    for cut in cuts:
        _same(_run(model, config, seeds, plan, cut=cut, **kw), ref, exact)
    return ref


def _model(name):
    if name == "funnel":
        return api.CudaModel(*configs.funnel(10).compile(True))
    return api.CudaModel(*configs.eight_schools().compile(True))


SEEDS = np.arange(40) + 11


def test_funnel_hmc_dualavg_thread_shape():
    m = _model("funnel")
    config = api.make_config(40, 60, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.IdentityMassMatrixTuner(), backend=abi.RN_BACKEND_THREAD)
    plan = [("w", 25), ("w", 35), ("r", 15), ("r", 25)]
    _check(m, config, SEEDS, plan, cuts=[0, 1, 2, 3])  # before the first warmup call, mid-warmup, end of warmup, mid-sampling


@pytest.mark.parametrize("backend", [abi.RN_BACKEND_THREAD, abi.RN_BACKEND_WARP], ids=["tpc", "wpc"])
def test_eight_schools_default_config(backend):
    """DefaultConfig's EHMC + DualAvg + diagonal windows (skip 50, windows 50, 75, ..): cuts in skip_first, mid-window, exactly
    at the first window's end, in skip_last, at the end of warmup and mid-sampling; EHMC's ring of 100 lengths fills during
    the first 100 warmup iterations, so the cuts fall before and after it fills"""
    m = _model("schools")
    config = api.SamplerConfig(iterations=60, warmupIterations=300, backend=backend)
    plan = [("w", 20), ("w", 60), ("w", 19), ("w", 171), ("w", 30), ("r", 25), ("r", 35)]
    _check(m, config, SEEDS[:24], plan, cuts=[1, 2, 3, 4, 5, 6])


def test_dense_mass_thread_shape():
    m = _model("schools")
    config = api.make_config(30, 100, sampler=api.HMCSampler(6), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.DenseMassMatrixTuner(20, 1.5, 10, 10), backend=abi.RN_BACKEND_THREAD)
    _check(m, config, SEEDS, [("w", 45), ("w", 55), ("r", 30)], cuts=[1, 2])


@pytest.mark.parametrize("mass", ["diagonal", "dense"])
def test_pooled_step_and_mass_windows_one_rank(mass):
    m = _model("schools")
    tuner = (api.DiagonalMassMatrixTuner if mass == "diagonal" else api.DenseMassMatrixTuner)(20, 1.5, 10, 10)
    config = api.make_config(30, 100, sampler=api.HMCSampler(6), stepSizeTuner=api.DualAvgTuner(0.8), massMatrixTuner=tuner,
                             backend=abi.RN_BACKEND_THREAD, adaptation=abi.RN_ADAPT_POOLED, stepAdaptation=abi.RN_ADAPT_POOLED)
    _check(m, config, SEEDS, [("w", 45), ("w", 40), ("w", 15), ("r", 30)], cuts=[0, 1, 2, 3])  # mid-windows, at the end, sampling


def test_tracked_diagnostics_thin3_cut_between_kept_draws():
    m = _model("funnel")
    config = api.make_config(60, 40, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.IdentityMassMatrixTuner(), backend=abi.RN_BACKEND_THREAD)
    plan = [("w", 40), ("t", 3), ("r", 10), ("r", 11), ("r", 39)]
    ref = _check(m, config, SEEDS, plan, cuts=[2, 3, 4])  # 10 and 21 draws tracked: kept draws are 0, 3, .., 9 | 12, .., 21
    assert ref["diag"] is not None and np.isfinite(ref["diag"]).all()


STREAMED = {  # name -> (model, environment, chains, text the emitted source must contain, text it must not contain)
    "logreg_dmma_ragged": (lambda: configs.logreg(1500, 6), {"RN_INLINE": "0"}, 13, [_DMMA], []),
    "logreg_rows": (lambda: configs.logreg(300, 3), {"RN_INLINE": "0", "RN_MMA": "0"}, 24, ["#define RN_WPC_PLACE 0\n"], [_DMMA]),
}


@pytest.mark.parametrize("name", list(STREAMED))
def test_streamed_logistic_regression(name):
    build, env, chains, must, must_not = STREAMED[name]
    rir, cols = build().compile(False)
    config = api.make_config(30, 40, sampler=api.HMCSampler(4), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.IdentityMassMatrixTuner(), backend=abi.RN_BACKEND_WARP)
    with _Env(env):
        m = api.CudaModel(rir, cols)
        src = m.emit_source(config)
        assert all(t in src for t in must) and not any(t in src for t in must_not), "%s: not the path named" % name
        _check(m, config, SEEDS[:chains], [("w", 15), ("w", 25), ("r", 12), ("r", 18)], cuts=[1, 2, 3])


def test_poisson_glmm_scatter_add():
    rir, cols = configs.poisson_glm(20, 2000).compile(False)
    config = api.make_config(8, 0, sampler=api.HMCSampler(4), stepSizeTuner=api.StaticStepSize(0.01),
                             massMatrixTuner=api.IdentityMassMatrixTuner(), backend=abi.RN_BACKEND_WARP)
    m = api.CudaModel(rir, cols)
    assert "rn_scatter_add(" in m.emit_source(config)
    _check(m, config, SEEDS[:16], [("r", 4), ("r", 4)], cuts=[1], exact=False)


@pytest.mark.parametrize("name", ["schools", "logreg_rows"])
def test_placement_0_restored_in_placement_1(name):
    config = api.make_config(20, 30, sampler=api.HMCSampler(4), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.DiagonalMassMatrixTuner(8, 1.5, 4, 4), backend=abi.RN_BACKEND_WARP)
    env = {"RN_INLINE": "0", "RN_MMA": "0"} if name != "schools" else {}
    with _Env(env):
        make = (lambda: _model("schools")) if name == "schools" else (lambda: api.CudaModel(*STREAMED["logreg_rows"][0]().compile(False)))
        m, m1 = make(), make()  # m1 compiles its kernels under RN_WPC_PLACE=1 (a model caches them by configuration)
        assert "#define RN_WPC_PLACE 0\n" in m.emit_source(config)
        with _Env({"RN_WPC_PLACE": "1"}):
            assert "#define RN_WPC_PLACE 1\n" in m1.emit_source(config)
        plan = [("w", 13), ("w", 17), ("r", 8), ("r", 12)]
        _check(m, config, SEEDS[:24], plan, cuts=[1, 2, 3], restore_env={"RN_WPC_PLACE": "1"}, restore_model=m1)
        s = api.CudaSampler(m, config, seeds=SEEDS[:24])
        s.warmup(13)
        assert api.checkpoint_info(s.save())["wpc_place"] == 0
        with _Env({"RN_WPC_PLACE": "1"}):
            r = api.CudaSampler.restore(m1, config, s.save())
        assert api.checkpoint_info(r.save())["wpc_place"] == 1  # the placement-1 kernels ran the continuation
        r.close()
        s.close()


_CHILD = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1])
from oracle.rainier_py import configs
from rainier_b200 import abi, api
m = api.CudaModel(*configs.eight_schools().compile(True))
s = api.CudaSampler(m, api.SamplerConfig(iterations=40, warmupIterations=150, backend=abi.RN_BACKEND_THREAD), seeds=np.arange(24) + 11)
s.warmup(70)
open(sys.argv[2], "wb").write(s.save())
"""


def test_restore_in_another_process(tmp_path):
    path = str(tmp_path / "schools.ckpt")
    subprocess.run([sys.executable, "-c", _CHILD, ROOT, path], check=True, timeout=600)
    blob = open(path, "rb").read()
    assert api.checkpoint_info(blob)["warm_done"] == 70
    m = _model("schools")
    config = api.SamplerConfig(iterations=40, warmupIterations=150, backend=abi.RN_BACKEND_THREAD)
    plan = [("w", 70), ("w", 80), ("r", 40)]
    ref = _run(m, config, SEEDS[:24], plan)
    import torch
    s = api.CudaSampler.restore(m, config, blob)
    s.warmup(80)
    d = torch.empty((40, m.nVars, 24), dtype=torch.float64, device="cuda")
    s.run(40, d.data_ptr())
    s.sync()
    assert np.array_equal(d.permute(2, 0, 1).cpu().numpy(), ref["samples"])
    st, mass, rings = _stats(s)
    for f in st:
        assert np.array_equal(st[f], ref["stats"][f]), f
    assert np.array_equal(mass, ref["mass"]) and np.array_equal(rings, ref["rings"])
    s.close()


def _continue(s, plan, model):
    import torch
    draws = []
    for op, x in plan:
        if op == "w":
            s.warmup(x)
        else:
            d = torch.empty((x, model.nVars, s.chains), dtype=torch.float64, device="cuda")
            s.run(x, d.data_ptr())
            draws.append(d)
    s.sync()
    return torch.cat(draws, 0).permute(2, 0, 1).cpu().numpy(), _stats(s)


def test_concatenation_and_slices():
    """two samplers over chains [0, k) and [k, C) restored as one equal one sampler over [0, C); slices of a blob restored
    separately equal the whole"""
    m = _model("funnel")
    config = api.make_config(30, 50, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.IdentityMassMatrixTuner(), backend=abi.RN_BACKEND_THREAD)
    k, rest = 13, [("w", 30), ("r", 30)]
    whole = api.CudaSampler(m, config, seeds=SEEDS)
    whole.warmup(20)
    blob = whole.save()
    ref, ref_stats = _continue(whole, rest, m)
    whole.close()
    parts = []
    for seeds in (SEEDS[:k], SEEDS[k:]):
        s = api.CudaSampler(m, config, seeds=seeds)
        s.warmup(20)
        parts.append(s.save())
        s.close()
    joined = api.CudaSampler.restore(m, config, parts)
    assert joined.chains == len(SEEDS)
    got, got_stats = _continue(joined, rest, m)
    joined.close()
    assert np.array_equal(got, ref)
    for f in ref_stats[0]:
        assert np.array_equal(got_stats[0][f], ref_stats[0][f]), f
    for b, e in [(0, k), (k, 29), (29, len(SEEDS))]:
        sl = api.checkpoint_slice(blob, b, e)
        assert api.checkpoint_info(sl)["chain_offset"] == b
        s = api.CudaSampler.restore(m, config, sl)
        got, _ = _continue(s, rest, m)
        s.close()
        assert np.array_equal(got, ref[b:e])


def test_extension_of_a_finished_run():
    m = _model("schools")
    short = api.make_config(40, 60, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                            massMatrixTuner=api.DiagonalMassMatrixTuner(10, 1.5, 5, 5), backend=abi.RN_BACKEND_THREAD)
    longer = api.make_config(100, 60, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.DiagonalMassMatrixTuner(10, 1.5, 5, 5), backend=abi.RN_BACKEND_THREAD)
    ref = _run(m, longer, SEEDS, [("w", 60), ("r", 40), ("r", 60)])
    first = _run(m, short, SEEDS, [("w", 60), ("r", 40)])
    assert np.array_equal(first["samples"], ref["samples"][:, :40])
    s = api.CudaSampler(m, short, seeds=SEEDS)
    s.warmup(60)
    s.run(40)
    blob = s.save()
    s.close()
    s = api.CudaSampler.restore(m, longer, blob)
    got, st = _continue(s, [("r", 60)], m)
    s.close()
    assert np.array_equal(got, ref["samples"][:, 40:])
    for f in st[0]:
        assert np.array_equal(st[0][f], ref["stats"][f]), f


def test_page_locked_buffer_and_chunked_staging():
    """save into rn_host_alloc memory and through 4 KB device staging buffers (many chunks, boundaries inside records' tiles):
    the same bytes as the pageable, single-chunk save"""
    m = _model("schools")
    config = api.SamplerConfig(iterations=20, warmupIterations=100, backend=abi.RN_BACKEND_THREAD)
    s = api.CudaSampler(m, config, seeds=SEEDS)
    s.warmup(50)
    s.track_diagnostics(2)
    plain = bytes(s.save())
    buf = api.PinnedBuffer((len(plain) + 64,), dtype=np.uint8)
    with _Env({"RN_CKPT_STAGE": "4096"}):
        pinned = s.save(out=buf.array)
        chunked = bytes(s.save())
    assert bytes(pinned) == plain and chunked == plain
    with _Env({"RN_CKPT_STAGE": "4096"}):
        r = api.CudaSampler.restore(m, config, pinned)
    assert bytes(r.save()) == plain
    r.close()
    s.close()
    buf.close()


def test_refusals_on_the_device():
    funnel, schools = _model("funnel"), _model("schools")
    assert funnel.nVars == schools.nVars
    config = api.make_config(20, 30, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.IdentityMassMatrixTuner(), backend=abi.RN_BACKEND_THREAD)
    s = api.CudaSampler(funnel, config, seeds=SEEDS)
    s.warmup(10)
    blob = s.save()
    s.close()

    def refused(fn, word):
        with pytest.raises(api.RainierCudaError) as e:
            fn()
        assert e.value.code == abi.RN_E_INVALID and word in str(e.value), str(e.value)

    refused(lambda: api.CudaSampler.restore(schools, config, blob), "fingerprint")
    other = api.make_config(20, 30, sampler=api.HMCSampler(6), stepSizeTuner=api.DualAvgTuner(0.8),
                            massMatrixTuner=api.IdentityMassMatrixTuner(), backend=abi.RN_BACKEND_THREAD)
    refused(lambda: api.CudaSampler.restore(funnel, other, blob), "rn_config.n_steps")
    warp = api.make_config(20, 30, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                           massMatrixTuner=api.IdentityMassMatrixTuner(), backend=abi.RN_BACKEND_WARP)
    refused(lambda: api.CudaSampler.restore(funnel, warp, blob), "kernel shape: backend")
    refused(lambda: api.CudaSampler.restore(funnel, config, blob[:-1]), "truncated")
    bad = bytearray(blob)
    bad[len(bad) // 2] ^= 4
    refused(lambda: api.CudaSampler.restore(funnel, config, bad), "checksum")
    logreg = api.CudaModel(*configs.logreg(300, 3).compile(False))
    refused(lambda: api.CudaSampler.restore(logreg, config, blob), "n differs")
    pooled = api.make_config(20, 30, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.DiagonalMassMatrixTuner(8, 1.5, 4, 4), backend=abi.RN_BACKEND_THREAD,
                             adaptation=abi.RN_ADAPT_POOLED)
    s = api.CudaSampler(funnel, pooled, seeds=SEEDS)
    s.warmup(12)
    pb = s.save()
    s.close()
    refused(lambda: api.checkpoint_slice(pb, 0, 7), "pooled warmup")
    refused(lambda: api.CudaSampler.restore(funnel, pooled, [pb, pb]), "pooled warmup")
    api.CudaSampler.restore(funnel, pooled, pb).close()  # one whole blob is no re-sharding


def test_restore_on_a_second_device():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one device: the cross-device restore needs a second GPU")
    rir, cols = configs.eight_schools().compile(True)
    m0, m1 = api.CudaModel(rir, cols, device=0), api.CudaModel(rir, cols, device=1)
    config = api.SamplerConfig(iterations=30, warmupIterations=100, backend=abi.RN_BACKEND_THREAD)
    ref = _run(m0, config, SEEDS, [("w", 40), ("w", 60), ("r", 30)])
    s = api.CudaSampler(m0, config, seeds=SEEDS)
    s.warmup(40)
    blob = s.save()
    s.close()
    s = api.CudaSampler.restore(m1, config, blob)
    s.warmup(60)
    with torch.cuda.device(1):
        d = torch.empty((30, m1.nVars, len(SEEDS)), dtype=torch.float64, device="cuda:1")
        s.run(30, d.data_ptr())
        s.sync()
        assert np.array_equal(d.permute(2, 0, 1).cpu().numpy(), ref["samples"])
    s.close()

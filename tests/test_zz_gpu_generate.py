"""
GPU side of the posterior-predictive draws (rn_generator_*, rn_sample_generate): the device equals the plan executor and the
host emulation bit for bit -- draws and returned RNG states -- through both entry points and both layouts, at chain counts
around the CTA size and at 65 537, under chunk splits; the SBC data; and sample_generate against single-chain oracle runs.
No test here feeds parameter values that would not terminate: the RNG budget is exercised on the CPU only.
"""
import json
import os

import numpy as np
import pytest

from oracle.rainier_py import configs, sbc_models
from oracle.rainier_py.binding import OracleFunction, OracleModel, ScalaRNG
from oracle.rainier_py.core import Binomial, Gamma, Geometric, NegativeBinomial, Normal, Poisson, to_generator
from rainier_b200 import abi, api
from rainier_b200 import generate as G

import generate_reference as R
from test_generate_host import CASES, GOLD, PARAMS, _params, _synthesize_parts, q0, q1

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mixed():
    return (Normal(q0, q1 + 1), Poisson(q0 * 40), Gamma(q1 * 0.8 + 0.1, 2), to_generator(Geometric(q0 * 0.5 + 0.2)).repeat(2),
            Binomial(q1, 10), NegativeBinomial(q0 * 0.3 + 0.1, 5), q1)


def _states(chains, seed):
    return [ScalaRNG(int(s)).rand.state() for s in np.random.default_rng(seed).integers(1, 1 << 40, size=chains)]


def _key(states):
    return [(s.seed48, s.next_gaussian, s.have_next) for s in states]


@pytest.mark.parametrize("chains", [1, 127, 129, 65537])
def test_device_equals_emulation_and_executor(chains):
    import torch
    rir = G.lower_generator(_mixed(), PARAMS)
    g = api.CudaGenerator(rir)
    iters = 6
    x = np.random.default_rng(chains).random(size=(chains, iters, 2))
    states = _states(chains, chains + 1)
    ref, ref_st, err, _ = R.emulate(api.CudaGenerator(rir, device=-1).emit_source(), x, states, g.nOutputs)
    assert not err.any()
    for c in sorted({0, chains // 2, chains - 1}):  # the executor on a few chains
        out_c, st_c, bad = R.run_plan(rir, OracleFunction(rir)(x[c]), states[c])
        assert bad is None and np.array_equal(ref[c], out_c) and _key([ref_st[c]]) == _key([st_c])
    # host entry point
    out, st = g(x, states)
    assert np.array_equal(out, ref) and _key(st) == _key(ref_st)
    # split into two calls, and chunks of one iteration
    g.set_chunk(1)
    o1, s1 = g(x[:, :2], states)
    o2, s2 = g(x[:, 2:], s1)
    assert np.array_equal(np.concatenate([o1, o2], axis=1), ref) and _key(s2) == _key(ref_st)
    g.set_chunk(0)
    # device entry point, both layouts
    dev = torch.device("cuda:0")
    for layout, xin in ((abi.RN_LAYOUT_ROWS, x), (abi.RN_LAYOUT_SAMPLER, np.ascontiguousarray(x.transpose(1, 2, 0)))):
        d_x = torch.from_numpy(np.ascontiguousarray(xin)).to(dev)
        d_out = torch.full((chains, iters, g.nOutputs), float("nan"), dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        st = g.eval_device(d_x.data_ptr(), iters, chains, states, d_out.data_ptr(), layout=layout)
        assert np.array_equal(d_out.cpu().numpy(), ref) and _key(st) == _key(ref_st)


@pytest.mark.parametrize("name", sorted(CASES))
def test_every_case_on_device(name):
    rir = G.lower_generator(CASES[name](), PARAMS)
    chains, iters = 33, 5
    x = np.random.default_rng(3).random(size=(chains, iters, 2))
    states = _states(chains, 9)
    out, st = api.CudaGenerator(rir)(x, states)
    for c in (0, 17, 32):
        ref, ref_st, _ = R.run_plan(rir, OracleFunction(rir)(x[c]), states[c])
        assert np.array_equal(out[c], ref) and _key([st[c]]) == _key([ref_st])


@pytest.mark.parametrize("name", sbc_models.ENABLED)
def test_golden_sbc_data_on_device(name):
    d, state, values = _synthesize_parts(name)
    rir = G.lower_generator(d.generator.repeat(GOLD["synthetic_samples"]), PARAMS)
    out, _ = api.CudaGenerator(rir)(np.zeros((1, 1, 2)), [state])
    assert np.array_equal(out[0, 0], np.array(values, dtype=np.float64))


def _oracle_chain_then_predict(rir_model, cols, cfg, seed, grir):
    res = OracleModel(rir_model, cols).sample(cfg, seeds=[seed])
    slots = OracleFunction(grir)(res["samples"][0])
    out, st, bad = R.run_plan(grir, slots, res["stats"][0].rng)
    assert bad is None
    return out, st


def _compare_with_sample(m, cfg, seeds, g, draws, tr):
    ref = m.sample(cfg, seeds=seeds)
    assert np.array_equal(tr.mass, ref.mass)
    for a, b in zip(tr.stats, ref.stats):
        for f in ("gradientEvaluations", "leapfrogSteps", "iterations", "accepted", "stepSize", "energyVarianceMean",
                  "energyVarianceRaw", "energyTransitions2"):
            assert getattr(a, f) == getattr(b, f), f
    # the generator continues the sampling states of rn_sample
    out, st = g(ref.chains, [api.RngState(*s.rng, 0) for s in ref.stats])
    assert np.array_equal(draws, out) and _key(st) == [s.rng for s in tr.stats]


def test_sample_generate_eight_schools_against_single_chain_oracle():
    model, mu, tau, thetas, sigmas = configs.eight_schools_parts()
    rir, cols = model.compile(True)
    t = [Normal(thetas.at(i), sigmas[i]) for i in range(8)]
    grir = G.lower_generator(t, model.parameters)
    m, g = api.CudaModel(rir, cols), api.CudaGenerator(grir)
    config = api.SamplerConfig(iterations=200, warmupIterations=200)  # DefaultConfig's sampler and tuners
    seeds = [11, 12, 13]
    draws, tr = m.sample_generate(g, config, seeds=seeds)
    cfg, _ = api.lower_config(config)
    for c, s in enumerate(seeds):
        out, st = _oracle_chain_then_predict(rir, cols, cfg, s, grir)
        assert np.array_equal(draws[c], out) and tr.stats[c].rng == _key([st])[0]
    _compare_with_sample(m, config, seeds, g, draws, tr)


@pytest.mark.parametrize("name", ["SBCLargePoisson", "SBCBinomial"])
def test_sample_generate_sbc_against_single_chain_oracle(name):
    model, real, rng, _ = sbc_models.build(name, GOLD["seed"], GOLD["synthetic_samples"])
    rir, cols = model.compile(True)
    d = {"SBCLargePoisson": lambda r: Poisson(r * 1000), "SBCBinomial": lambda r: Binomial(r, 10)}[name](real)
    grir = G.lower_generator(to_generator(d).repeat(3), model.parameters)
    m, g = api.CudaModel(rir, cols), api.CudaGenerator(grir)
    config = api.make_config(iterations=50, warmupIterations=100, sampler=api.HMCSampler(1), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.IdentityMassMatrixTuner())
    seeds = [5, 6]
    draws, tr = m.sample_generate(g, config, seeds=seeds)
    cfg, _ = api.lower_config(config)
    for c, s in enumerate(seeds):
        out, st = _oracle_chain_then_predict(rir, cols, cfg, s, grir)
        assert np.array_equal(draws[c], out) and tr.stats[c].rng == _key([st])[0]
    _compare_with_sample(m, config, seeds, g, draws, tr)


def test_sample_generate_streamed_warp_shape():
    z = np.load(os.path.join(ROOT, "rainier_b200", "models", "logreg_700x4.primal.npz"))
    cols = [z["c%d" % i] for i in range(int(z["ncols"]))]
    m = api.CudaModel(z["rir"].tobytes(), cols)
    q, params = _params(m.nVars)
    grir = G.lower_generator([Normal(q[0] + q[1], q[2].exp()), Poisson(q[3].exp())], params)
    g = api.CudaGenerator(grir)
    config = api.make_config(iterations=20, warmupIterations=20, sampler=api.HMCSampler(3), stepSizeTuner=api.StaticStepSize(0.01),
                             massMatrixTuner=api.IdentityMassMatrixTuner())
    seeds = list(range(100, 140))
    draws, tr = m.sample_generate(g, config, seeds=seeds)
    assert np.all(np.isfinite(draws))
    _compare_with_sample(m, config, seeds, g, draws, tr)


def test_chain_blocks_when_one_iteration_of_slots_exceeds_the_scratch():
    """100 slots x 400 000 chains = 320 MB per iteration, more than the 256 MB slot scratch: the call runs in blocks of
    chains, invisibly -- every chain equals the same chain drawn alone"""
    xs = np.linspace(-1.0, 1.0, 100)
    rir = G.lower_generator([Poisson((q0 + q1 * float(v)).exp()) for v in xs], PARAMS)
    g = api.CudaGenerator(rir)
    chains, iters = 400000, 2
    x = np.random.default_rng(8).random(size=(chains, iters, 2))
    states = [api.RngState(int(s), 0.0, 0, 0) for s in np.random.default_rng(9).integers(1, 1 << 48, size=chains)]
    out, st = g(x, states)
    block = (256 << 20) // (100 * 8)
    for c in (0, block - 1, block, chains - 1):
        ref, ref_st, bad = R.run_plan(rir, OracleFunction(rir)(x[c]), states[c])
        assert bad is None and np.array_equal(out[c], ref) and _key([st[c]]) == _key([ref_st])

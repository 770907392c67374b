"""
Posterior-predictive draws on the device (rn_generator_*, rn_generate.cuh), CPU side:

  * the plan executor (generate_reference.run_plan) equals the closures of core.py's Generator.predict bit for bit, for every
    supported piece and regime, over random draws and RNG states (Java's Math.log / exp / pow pinned to fdlibm on both sides);
  * the emitted generator source, compiled for the host, equals the executor bit for bit, returned RNG states included, over
    several chains, both input layouts, chunkings and random splits of the iterations into calls;
  * for the 11 SBC models, the lowered `d.generator.repeat(1000)` reproduces SBC.synthesize's data from the RNG state after
    the prior draw;
  * the per-draw RNG budget (host emulation only; a chain stops at its first over-budget draw) and its error report, malformed
    plans, unsupported pieces, no CPU fallback.
"""
import json
import os
import struct
import zlib

import numpy as np
import pytest

from oracle.rainier_py import sbc_models
from oracle.rainier_py.binding import OracleFunction, ScalaRNG
from oracle.rainier_py.compute import Evaluator, Real, compile_function_rir, to_real
from oracle.rainier_py.core import (Bernoulli, Beta, Binomial, Cauchy, Exponential, Gamma, Generator, Geometric, Laplace,
                                    LogNormal, Model, Multinomial, NegativeBinomial, Normal, Poisson, Uniform, to_generator)
from rainier_b200 import abi, api
from rainier_b200 import generate as G

import generate_reference as R

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "sbc_goldsets.json")))


def _params(n):
    holder = {}

    def keep(t):
        holder["t"] = list(t)
        return Real.sum(list(t))

    Real.parameters(n, keep)
    model = Model.track_(list(holder["t"]))
    return holder["t"], model.parameters


Q, PARAMS = _params(2)
q0, q1 = Q

# name -> ToGenerator value over q0, q1 (draws put both in [0, 1)): every supported piece and every regime
CASES = {
    "normal": lambda: Normal(q0, q1.exp()),
    "cauchy": lambda: Cauchy(q0, q1.exp()),
    "laplace": lambda: Laplace(q0, q1.exp()),
    "uniform": lambda: Uniform(q0, q0 + q1.exp()),
    "lognormal": lambda: LogNormal(q0, q1.exp()),
    "gamma_below_1": lambda: Gamma(q0 * 0.5 + 0.2, q1 + 1),
    "gamma_above_1": lambda: Gamma(q0 * 5 + 1, q1 + 1),
    "exponential": lambda: Exponential(q0 + 1),
    "beta": lambda: Beta(q0 + 0.5, q1 * 3 + 0.3),
    "beta_scaled": lambda: Beta(q0 + 0.5, q1 + 2).scale(q1 + 3).translate(q0),
    "bernoulli": lambda: Bernoulli(q0),
    "geometric": lambda: Geometric(q0 * 0.8 + 0.1),
    "poisson_small": lambda: Poisson(q0 * 30),
    "poisson_large": lambda: Poisson(q0 * 1000 + 30),
    "binomial_poisson": lambda: Binomial(q0 * 0.05, 200),
    "binomial_normal": lambda: Binomial(q0 * 0.4 + 0.3, 200),
    "binomial_multinomial": lambda: Binomial(q0, 10),
    "negbinomial_normal": lambda: NegativeBinomial(q0 * 0.2 + 0.5, 1000),
    "negbinomial_geometric": lambda: NegativeBinomial(q0 * 0.3 + 0.1, 10),
    "real": lambda: q0 * 2 + q1,
    "tuple": lambda: (Normal(q0, 1), Poisson(q1 * 5), q0, Gamma(q1 + 0.1, 2)),
    "traverse": lambda: [Normal(q0 + i, q1 + 1) for i in range(4)] + [Bernoulli(q1)],
    "repeat": lambda: to_generator(Poisson(q0 * 10)).repeat(5),
    "repeat_nested": lambda: to_generator((Laplace(q0, 1), [Geometric(q1 * 0.5 + 0.2), q1])).repeat(3).repeat(2),
    "zip3_real_generator": lambda: to_generator(Normal(q0, 2)).zip(Generator.real(q1)).zip(to_generator(Cauchy(q1, 1))),
}


def _flat(v):
    if isinstance(v, (list, tuple)):
        return [x for u in v for x in _flat(u)]
    return [float(v)]


def _draws(seed, count):
    return np.random.default_rng(seed).random(size=(count, 2))


@pytest.mark.parametrize("name", sorted(CASES))
def test_plan_executor_equals_closures(name):
    t = CASES[name]()
    rir = G.lower_generator(t, PARAMS)
    draws = _draws(zlib.crc32(name.encode()) % 1000, 30)
    seed = 1000 + len(name)
    rng = ScalaRNG(seed)
    with R.fdlibm():
        ref = to_generator(t).predict(PARAMS, draws, rng, OracleFunction)
    ref = np.array([_flat(v) for v in ref])
    slots = OracleFunction(rir)(draws)
    out, st, bad = R.run_plan(rir, slots, ScalaRNG(seed).rand.state())
    assert bad is None
    assert out.shape == ref.shape and np.array_equal(out, ref)
    s2 = rng.rand.state()
    assert (st.seed48, st.next_gaussian, st.have_next) == (s2.seed48, s2.next_gaussian, s2.have_next)
    # the slots the compiled function computes are the values the reference's Evaluator gives those Reals (the reference
    # reads inner Reals -- Binomial's p*k, NegativeBinomial's, requirements past the first 500 -- through the Evaluator)
    reals = G.slots_of(t)
    with R.fdlibm():
        for a, row in zip(draws, slots):
            ev = Evaluator({p: float(v) for p, v in zip(PARAMS, a)})
            assert [ev.toDouble(r) for r in reals] == [float(v) for v in row]


@pytest.mark.parametrize("name", ["tuple", "repeat_nested", "binomial_normal", "negbinomial_geometric", "gamma_below_1", "beta_scaled"])
def test_emitted_source_equals_executor_over_chains_and_splits(name):
    t = CASES[name]()
    rir = G.lower_generator(t, PARAMS)
    g = api.CudaGenerator(rir, device=-1)
    assert (g.nInputs, g.nSlots) == (2, len(G.slots_of(t)))
    src = g.emit_source()
    chains, iters = 5, 13
    x = np.random.default_rng(4).random(size=(chains, iters, 2))  # [chain][iteration][n]
    rs = np.random.default_rng(5)
    states = [ScalaRNG(int(s)).rand.state() for s in rs.integers(1, 1 << 40, size=chains)]
    refs = [R.run_plan(rir, OracleFunction(rir)(x[c]), states[c]) for c in range(chains)]
    ref = np.stack([r[0] for r in refs])
    ref_states = [(r[1].seed48, r[1].next_gaussian, r[1].have_next) for r in refs]
    for layout in ("rows", "sampler"):
        xin = x if layout == "rows" else np.ascontiguousarray(x.transpose(1, 2, 0))
        for chunk in (None, 1, 4):
            out, st, err, _ = R.emulate(src, xin, states, g.nOutputs, layout=layout, chunk=chunk)
            assert not err.any() and np.array_equal(out, ref)
            assert [(s.seed48, s.next_gaussian, s.have_next) for s in st] == ref_states
    # any split of the iterations into calls gives the same bits
    for trial in range(3):
        cuts = sorted(rs.choice(np.arange(1, iters), size=2, replace=False))
        st, parts = states, []
        for a, b in zip([0] + cuts, cuts + [iters]):
            out, st, err, _ = R.emulate(src, x[:, a:b], st, g.nOutputs)
            assert not err.any()
            parts.append(out)
        assert np.array_equal(np.concatenate(parts, axis=1), ref)
        assert [(s.seed48, s.next_gaussian, s.have_next) for s in st] == ref_states


def _synthesize_parts(name):
    """SBC.synthesize (K/SBC.scala:53-61) split at the prior draw: (likelihood d, RNG state after the prior draw, data)"""
    seed, samples = GOLD["seed"], GOLD["synthetic_samples"]
    with R.fdlibm():
        values, _ = sbc_models.MODELS[name]().synthesize(samples, ScalaRNG(seed))
        sbc = sbc_models.MODELS[name]()
        rng = ScalaRNG(seed)
        prior = sbc.priorGenerator.get(rng, Evaluator())
    d, _ = sbc.fn([to_real(p) for p in prior])
    return d, rng.rand.state(), values


@pytest.mark.parametrize("name", sbc_models.ENABLED)
def test_golden_sbc_data_from_the_lowered_likelihood(name):
    d, state, values = _synthesize_parts(name)
    n = GOLD["synthetic_samples"]
    rir = G.lower_generator(d.generator.repeat(n), PARAMS)  # the likelihood at the prior draw: constant slots
    x = np.zeros((1, 1, 2))
    slots = OracleFunction(rir)(x[0])
    out, _, bad = R.run_plan(rir, slots, state)
    assert bad is None and np.array_equal(out[0], np.array(values, dtype=np.float64))
    g = api.CudaGenerator(rir, device=-1)
    emu, _, err, _ = R.emulate(g.emit_source(), x, [state], g.nOutputs)
    assert not err.any() and np.array_equal(emu[0, 0], out[0])


def _lcg_advance(seed, steps):
    """java.util.Random's state after `steps` more next() calls (the affine map x -> a x + c mod 2^48, squared up)"""
    a, c, M = 0x5DEECE66D, 0xB, (1 << 48) - 1
    ra, rc = 1, 0
    while steps:
        if steps & 1:
            ra, rc = (a * ra) & M, (a * rc + c) & M
        a, c = (a * a) & M, (a * c + c) & M
        steps >>= 1
    return (ra * seed + rc) & M


def test_budget_stops_a_chain_at_its_first_over_budget_draw():
    """Poisson.large with lambda = NaN and a Binomial repeat of 2^30 would not finish in the reference.  The chain stops at
    the draw that would make RNG call 2^24 + 1: that iteration and the later ones are NaN, its state is where the draw
    stopped, its error bit and iteration are set (and become RN_E_INVALID naming them); the other chains are intact.  Gamma
    with a NaN or negative shape is not such a case: Marsaglia-Tsang's first acceptance test does not read
    c = (1/3) / sqrt(d), so the draw ends with NaN after a few calls, as in the reference."""
    for t, bad_row, budget in ((Poisson(q0), [np.nan, 0.0], True), (Binomial(q1, q0), [2.0 ** 30, 1.0], True),
                               (Gamma(q0, 1), [-2.0, 0.0], False), (Gamma(q0, 1), [np.nan, 0.0], False)):
        rir = G.lower_generator((t, Normal(q1, 1)), PARAMS)
        g = api.CudaGenerator(rir, device=-1)
        chains, iters = 3, 5
        x = np.random.default_rng(2).random(size=(chains, iters, 2)) + 0.5
        x[1, 2] = bad_row
        states = [ScalaRNG(50 + c).rand.state() for c in range(chains)]
        out, st, err, err_iter = R.emulate(g.emit_source(), x, states, g.nOutputs)
        for c in ((0, 2) if budget else (0, 1, 2)):
            ref, ref_st, bad = R.run_plan(rir, OracleFunction(rir)(x[c]), states[c])
            assert bad is None and np.array_equal(out[c], ref, equal_nan=True) and st[c].seed48 == ref_st.seed48
        if not budget:
            assert not err.any() and np.isnan(out[1, 2, 0])
            continue
        assert list(err) == [0, 1, 0] and err_iter[1] == 2
        ref, ref_st, _ = R.run_plan(rir, OracleFunction(rir)(x[1, :2]), states[1])
        assert np.array_equal(out[1, :2], ref) and np.all(np.isnan(out[1, 2:]))
        # one budget of uniforms (two next() calls each) after the first two iterations, then nothing
        assert st[1].seed48 == _lcg_advance(ref_st.seed48, 2 * R.BUDGET)
        assert (st[1].next_gaussian, st[1].have_next) == (ref_st.next_gaussian, ref_st.have_next)
        with pytest.raises(api.RainierCudaError, match="chain 1, iteration 2") as e:
            api.generator_report(err, err_iter)
        assert e.value.code == abi.RN_E_INVALID
    api.generator_report(np.zeros(3, np.int32), np.full(3, -1, np.int64))  # no error bit: RN_OK


def test_a_chain_whose_every_draw_is_bad_costs_one_budget():
    rir = G.lower_generator(to_generator(Poisson(q0)).repeat(50), PARAMS)
    g = api.CudaGenerator(rir, device=-1)
    chains, iters = 2, 40
    x = np.full((chains, iters, 2), np.nan)
    x[0] = 0.5
    states = [ScalaRNG(7 + c).rand.state() for c in range(chains)]
    out, st, err, err_iter = R.emulate(g.emit_source(), x, states, g.nOutputs, chunk=7)
    assert list(err) == [0, 1] and err_iter[1] == 0 and np.all(np.isnan(out[1]))
    assert st[1].seed48 == _lcg_advance(states[1].seed48, 2 * R.BUDGET)
    ref, ref_st, bad = R.run_plan(rir, OracleFunction(rir)(x[0]), states[0])
    assert bad is None and np.array_equal(out[0], ref) and st[0].seed48 == ref_st.seed48


def test_unsupported_pieces_raise_at_lowering():
    for t, what in ((to_generator(Normal(q0, 1)).map(lambda v: v * 2), "map closure"),
                    (to_generator(Normal(q0, 1)).flatMap(lambda v: Normal(v, 1)), "flatMap"),
                    (Generator.from_(lambda r, n: r.standardUniform()), "from / require closure"),
                    (Generator.categorical([(1, q0), (2, 1 - q0)]), "categorical"),
                    (Multinomial([("a", q0), ("b", 1 - q0)], 3), "Multinomial"),
                    (Generator.constant(5), "constant"),
                    (to_generator(Normal(q0, 1)).repeat(q1), "non-constant count")):
        with pytest.raises(G.Unsupported, match=what):
            G.lower_generator(t, PARAMS)


def test_malformed_plans_are_refused_and_no_cpu_fallback():
    rir = G.lower_generator((Normal(q0, 1), Binomial(q1, 10)), PARAMS)
    g = api.CudaGenerator(rir, device=-1)
    with pytest.raises(api.RainierCudaError) as e:  # emit/compile only: evaluation fails loudly
        g(np.zeros((1, 1, 2)), [ScalaRNG(1).rand.state()])
    assert e.value.code == abi.RN_E_CUDA
    ops, m, nslots = R.parse(rir)
    base = len(rir) - len(ops) * G.GEN_OP.size - G.GEN_HEADER.size
    fn = rir[:base]

    def build(ops_, m_=1):
        return G.pack(fn, ops_, m_)

    bad = [
        compile_function_rir(PARAMS, [q0]),                                     # no RIR_FLAG_GENERATOR
        rir[:-8],                                                               # truncated op
        build([(99, [-1] * 6, 0), (G.EMIT, [-1] * 6, 0)]),                      # unknown kind
        build([(G.VALUE, [nslots] + [-1] * 5, 0), (G.EMIT, [-1] * 6, 0)]),      # slot out of range
        build([(G.VALUE, [0, 0] + [-1] * 4, 0), (G.EMIT, [-1] * 6, 0)]),        # unused slot field set
        build([(G.REPEAT, [-1] * 6, 2), (G.EMIT, [-1] * 6, 0)]),                # REPEAT without END
        build([(G.EMIT, [-1] * 6, 0), (G.END, [-1] * 6, 0)]),                   # END without REPEAT
        build([(G.REPEAT, [-1] * 6, -1), (G.EMIT, [-1] * 6, 0), (G.END, [-1] * 6, 0)], m_=1),  # negative count
        build([(G.EMIT, [-1] * 6, 3)]),                                         # count on a non-REPEAT op
        build([(G.NORMAL, [-1] * 6, 0)], m_=0),                                 # emits nothing
        build(ops, m_=m + 1),
        build(ops, m_=m)[:-1],                                                   # m_out does not match
        build([(G.REPEAT, [-1] * 6, 1)] * 9 + [(G.EMIT, [-1] * 6, 0)] + [(G.END, [-1] * 6, 0)] * 9),  # nested too deeply
        build([(G.REPEAT, [-1] * 6, 2 ** 31 - 1), (G.REPEAT, [-1] * 6, 2 ** 31 - 1), (G.NORMAL, [-1] * 6, 0), (G.END, [-1] * 6, 0),
               (G.END, [-1] * 6, 0), (G.EMIT, [-1] * 6, 0)]),                  # 2^62 draws for one value
        build([(G.REPEAT, [-1] * 6, 2 ** 25), (G.NORMAL, [-1] * 6, 0), (G.EMIT, [-1] * 6, 0), (G.END, [-1] * 6, 0)], m_=2 ** 25),
    ]
    for b in bad:
        with pytest.raises(api.RainierCudaError) as e:
            api.CudaGenerator(b, device=-1)
        assert e.value.code == abi.RN_E_INVALID
    hdr = bytearray(rir)
    struct.pack_into("<I", hdr, base, 0)  # n_ops = 0
    with pytest.raises(api.RainierCudaError):
        api.CudaGenerator(bytes(hdr), device=-1)
    # the largest plan allowed: 2^26 ops per draw
    ok = build([(G.REPEAT, [-1] * 6, 2 ** 24 - 1), (G.NORMAL, [-1] * 6, 0), (G.EMIT, [-1] * 6, 0), (G.END, [-1] * 6, 0)], m_=2 ** 24 - 1)
    assert api.CudaGenerator(ok, device=-1).nOutputs == 2 ** 24 - 1
    # creating a generator on a device needs one: no CPU fallback
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except ImportError:
        have_gpu = False
    if not have_gpu:
        with pytest.raises(api.RainierCudaError) as e:
            api.CudaGenerator(rir, device=0)
        assert e.value.code == abi.RN_E_CUDA
    # a generator container is still a function container: the slots alone
    assert api.CudaFunction(rir, device=-1).nOutputs == nslots

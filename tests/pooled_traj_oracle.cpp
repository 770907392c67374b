/* tests/pooled_traj_oracle.cpp -- TEST INFRASTRUCTURE ONLY: the oracle's restatement of pooled EHMC trajectory lengths
 * (rn_config.trajectory_adaptation == RN_ADAPT_POOLED, rainier_b200/csrc/rn_sampler_common.cuh).
 *   1. Every chain runs the reference's warmup on its own (Driver.scala:48-90), exactly as the per-chain oracle does.
 *   2. h[l] counts, over every chain, the entries of its ring of U-turn counts that steps.sample() would choose from:
 *      indices [0, full ? bufSize : i + 1) (Stats.scala:40-45), so an unfilled ring offers slot 0, whose value is 0.
 *   3. Sampling iteration t of every chain is lf.startIteration, lf.takeSteps(L_t), lf.finishIteration -- EHMC.scala:52-61
 *      without the ring draw -- where, as rainier_cuda.h defines it: T = sum h, c[l] the inclusive prefix sums, F the word hash
 *      of the counts, z = splitmix64(F + (t + 1) * 0x9E3779B97F4A7C15), r = mulhi64(z, T), L_t = min { l : c[l] > r }.
 * The per-chain oracle (oracle/rainier_oracle.cpp) is compiled into this library unchanged and only extended. */
#include "../oracle/rainier_oracle.cpp"

namespace rno {

/* the word hash of the checkpoints (four interleaved FNV-1a-style lanes over 64-bit words, then the lanes and the length) */
static uint64_t traj_fingerprint(const std::vector<int64_t>& h) {
  const uint64_t basis = 1469598103934665603ull, prime = 1099511628211ull;
  uint64_t lane[4] = {basis, basis ^ 1, basis ^ 2, basis ^ 3};
  for (size_t i = 0; i < h.size(); i++) lane[i & 3] = (lane[i & 3] ^ (uint64_t)h[i]) * prime;
  uint64_t r = basis * prime;  /* whole words: no tail bytes */
  for (int l = 0; l < 4; l++) r = (r ^ lane[l]) * prime;
  return (r ^ (uint64_t)(h.size() * 8)) * prime;
}

static int traj_length(const std::vector<int64_t>& h, const std::vector<int64_t>& cum, uint64_t F, int64_t t) {
  uint64_t z = F + (uint64_t)(t + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  const uint64_t r = (uint64_t)(((unsigned __int128)z * (uint64_t)cum.back()) >> 64);
  for (size_t l = 0; l < h.size(); l++)  /* a linear scan: the restatement, not the runtime's search */
    if ((uint64_t)cum[l] > r) return (int)l;
  return (int)h.size() - 1;
}

struct TrajChain {
  std::unique_ptr<RirDensity> interpreted;
  std::unique_ptr<CompiledDensity> compiled;
  std::unique_ptr<AdjointDensity> adjoint;
  std::unique_ptr<LeapFrog> lf;
  std::unique_ptr<Sampler> sampler;
  std::unique_ptr<StepSizeTuner> stepTuner;
  std::unique_ptr<MassMatrixTuner> massTuner;
  std::vector<double> params;
  MassMatrix mass;
  RNG rng;
  int error_flags = 0;
};

} /* namespace rno */

extern "C" {
/* seeds[c]: ScalaRNG(seeds[c]).  samples [chains][iterations][n]; mass [chains][n] (diagonal / identity); stats [chains];
 * trace [chains][warmup + iterations][4] as driver_sample writes it; hist [max_steps + 1] (all optional but samples). */
int rno_sample_pooled_traj(rno_model* mm, const rn_config* cfg, const int64_t* seeds, int chains, double* samples, double* mass,
                           rn_chain_stats* stats, double* trace, int64_t* hist) {
  using namespace rno;
  if (cfg->sampler != RN_SAMPLER_EHMC || cfg->trajectory_adaptation != RN_ADAPT_POOLED || cfg->step_adaptation != RN_ADAPT_PER_CHAIN ||
      cfg->adaptation != RN_ADAPT_PER_CHAIN || cfg->mass_tuner == RN_MASS_DENSE)
    return fail(RN_E_UNSUPPORTED, "the pooled-trajectory oracle covers EHMC with per-chain step and diagonal / identity mass adaptation");
  const Model& model = mm->m;
  const int n = model.n();
  const size_t T = (size_t)cfg->warmup_iterations + (size_t)cfg->iterations;
  std::vector<TrajChain> ch(chains);
  std::vector<double> sample(n);
  for (int c = 0; c < chains; c++) { /* 1. the per-chain warmup, driver_sample's loop */
    TrajChain& x = ch[c];
    x.rng.rand = JRandom(seeds[c]);
    x.interpreted.reset(new RirDensity(model));
    x.compiled.reset(new CompiledDensity(model));
    if (!(model.h.flags & RIR_FLAG_GRADIENT)) x.adjoint.reset(new AdjointDensity(model));
    DensityFunction& d = x.adjoint ? (DensityFunction&)*x.adjoint
                                   : (model.compiled ? (DensityFunction&)*x.compiled : (DensityFunction&)*x.interpreted);
    x.sampler = make_sampler(*cfg);
    x.stepTuner = make_step_tuner(*cfg);
    x.massTuner = make_mass_tuner(*cfg, n);
    x.lf.reset(new LeapFrog(d, cfg->stats_window));
    MassMatrix identity;
    x.params = x.lf->initialize(identity, x.rng);
    x.sampler->initialize(x.params, *x.lf, x.rng);
    double stepSize = x.stepTuner->initialize(x.params, *x.lf);
    x.mass = x.massTuner->initialize(*x.lf, cfg->warmup_iterations);
    for (int i = 0; i < cfg->warmup_iterations; i++) {
      const int64_t steps0 = x.lf->stats.leapfrogSteps;
      const int acc0 = x.lf->stats.accepted;
      const double used = stepSize;
      const double a = x.sampler->warmup(x.params, *x.lf, stepSize, x.mass, x.rng);
      stepSize = x.stepTuner->update(a);
      x.lf->variables(x.params, sample.data());
      MassMatrix m;
      if (x.massTuner->update(sample.data(), m)) {
        x.mass = m;
        if (m.invalid) x.error_flags |= 2;
        stepSize = x.stepTuner->reset();
      }
      if (trace) {
        double* tr = trace + ((size_t)c * T + (size_t)i) * 4;
        tr[0] = a;
        tr[1] = (double)(x.lf->stats.accepted - acc0);
        tr[2] = used;
        tr[3] = (double)(x.lf->stats.leapfrogSteps - steps0);
      }
    }
    x.lf->resetStats(); /* Driver.scala:31 */
  }
  std::vector<int64_t> h((size_t)cfg->max_steps + 1, 0), cum(h.size());
  for (TrajChain& x : ch) { /* 2. the pooled histogram */
    const RingBuffer& r = static_cast<EHMCSampler&>(*x.sampler).steps;
    const int k = r.full ? r.size : r.i + 1;
    for (int j = 0; j < k; j++) h[(size_t)jd2i(r.buf[j])] += 1;
  }
  int64_t run = 0;
  for (size_t l = 0; l < h.size(); l++) cum[l] = run += h[l];
  const uint64_t F = traj_fingerprint(h);
  if (hist) std::memcpy(hist, h.data(), h.size() * 8);
  for (int c = 0; c < chains; c++) { /* 3. sampling at the shared lengths */
    TrajChain& x = ch[c];
    LeapFrog& lf = *x.lf;
    const double finalStep = x.stepTuner->stepSize(); /* Driver.scala:37 */
    for (int i = 0; i < cfg->iterations; i++) {
      const int64_t steps0 = lf.stats.leapfrogSteps;
      const int acc0 = lf.stats.accepted;
      lf.startIteration(x.params, x.mass, x.rng);
      lf.takeSteps(traj_length(h, cum, F, i), finalStep, x.mass);
      lf.finishIteration(x.params, x.mass, x.rng);
      lf.variables(x.params, samples + ((size_t)c * cfg->iterations + i) * n);
      if (trace) {
        double* tr = trace + ((size_t)c * T + (size_t)cfg->warmup_iterations + i) * 4;
        tr[0] = lf.lastLogAcceptanceProb;
        tr[1] = (double)(lf.stats.accepted - acc0);
        tr[2] = finalStep;
        tr[3] = (double)(lf.stats.leapfrogSteps - steps0);
      }
    }
    if (x.interpreted->lookup_error | x.compiled->lookup_error | (x.adjoint ? x.adjoint->fwd.lookup_error : 0)) x.error_flags |= 1;
    if (mass) {
      double* mo = mass + (size_t)c * n;
      for (int e = 0; e < n; e++) mo[e] = x.mass.kind == RN_MATRIX_IDENTITY ? 1.0 : x.mass.elements[e];
    }
    if (stats) {
      const Stats& s = lf.stats;
      rn_chain_stats* st = stats + c;
      std::memset(st, 0, sizeof(*st));
      st->gradient_evaluations = s.gradientEvaluations;
      st->leapfrog_steps = s.leapfrogSteps;
      st->iterations = s.iterations;
      st->accepted = s.accepted;
      st->error_flags = x.error_flags;
      st->step_size = finalStep;
      st->energy_mean = s.energyVariance.mean[0];
      st->energy_raw = s.energyVariance.raw[0];
      st->energy_transitions2 = s.energyTransitions2;
      st->energy_samples = s.energyVariance.samples;
      st->ring_pos[0] = s.stepSizes.i;
      st->ring_pos[1] = s.acceptanceRates.i;
      st->ring_pos[2] = s.gradsPerIteration.i;
      st->ring_full[0] = s.stepSizes.full ? 1 : 0;
      st->ring_full[1] = s.acceptanceRates.full ? 1 : 0;
      st->ring_full[2] = s.gradsPerIteration.full ? 1 : 0;
      st->step_sizes_mean = s.stepSizes.mean();
      st->acceptance_rates_mean = s.acceptanceRates.mean();
      st->grads_per_iteration_mean = s.gradsPerIteration.mean();
      st->rng.seed48 = x.rng.rand.seed;
      st->rng.next_gaussian = x.rng.rand.next_next_gaussian;
      st->rng.have_next = x.rng.rand.have_next_next_gaussian ? 1 : 0;
    }
  }
  int err = 0;
  for (TrajChain& x : ch) err |= x.error_flags;
  if (err & 1) return fail(RN_E_LOOKUP, "lookup index out of range");
  if (err & 2) return fail(RN_E_INVALID, "requirement failed: adapted mass matrix contains 0.0 (MassMatrix.scala:8,16)");
  return RN_OK;
}
} /* extern "C" */

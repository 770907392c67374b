/* tests/pooled_step_oracle.cpp -- TEST INFRASTRUCTURE ONLY: the oracle's restatement of the two pooled adaptation modes,
 * pooled step sizes (rn_config.step_adaptation == RN_ADAPT_POOLED, rainier_b200/csrc/rn_sampler_common.cuh) and pooled mass
 * windows (rn_config.adaptation == RN_ADAPT_POOLED, rn_k_pool_reduce / rn_k_pool_apply).  The reference adapts per chain;
 * these extensions share state over all chains, so the chains can no longer run one after another: a lockstep driver runs
 * iterations outer, chains inner.
 * Pooled steps, with the same exact integer sums as the kernels:
 *   1. k_c = log2 of chain c's findReasonableStepSize (clamped to [-1075, 1024]); eps0 = jexp(ln2 * (K / C))
 *   2. q_c = rint(jexp(a_c) * 2^32), P_t = Q_t / (2^32 C), DualAvg.update with newAcceptanceProb = P_t
 * Pooled mass windows (diagonal tuner), in rn_k_pool_reduce's summation order:
 *   per chain, Welford statistics of the window: mean += od / win_i, raw += od * (q - mean) (win_i: position in the window)
 *   at the window end, pass 0: 256 partials (thread t adds chains t, t + 256, ... from 0.0), halving tree, / C = pooled mean;
 *   pass 1: the same over raw_c + L (mean_c - pooled mean)^2; variance = sum / (C L); error flag 2 where !(variance > 0)
 * Both: Driver.scala:67-80 order (step update, mass update, stepSizeTuner.reset() when a window closed), sampling at the
 * final step size; Stats stay per chain.
 * The per-chain oracle (oracle/rainier_oracle.cpp) is compiled into this library unchanged and only extended. */
#include "../oracle/rainier_oracle.cpp"

namespace rno {

struct LockstepChain {
  std::unique_ptr<RirDensity> interpreted;
  std::unique_ptr<CompiledDensity> compiled;
  std::unique_ptr<AdjointDensity> adjoint;
  std::unique_ptr<LeapFrog> lf;
  std::unique_ptr<Sampler> sampler;
  std::unique_ptr<MassMatrixTuner> massTuner;
  std::unique_ptr<StepSizeTuner> stepTuner;  /* per-chain steps only */
  double stepSize = 0.0;
  std::vector<double> params;
  std::vector<double> wmean, wraw;           /* pooled mass windows: the chain's Welford statistics of the window */
  MassMatrix mass;
  RNG rng;
  ChainResult res;
};

static const double kLn2 = 0.6931471805599453;
static const double kQScale = 4294967296.0;

/* rn_k_pool_reduce restated (one rank): the pooled population variance of the window that just closed, L draws per chain */
static void pool_reduce(const std::vector<LockstepChain>& ch, int n, int L, std::vector<double>& var) {
  const int C = (int)ch.size();
  std::vector<double> pool(2 * (size_t)n + 1, 0.0);
  double red[256];
  for (int pass = 0; pass < 2; pass++)
    for (int i = 0; i < n; i++) {
      const double gmean = pass ? pool[1 + i] / pool[0] : 0.0;
      for (int t = 0; t < 256; t++) {
        double acc = 0.0;
        for (int c = t; c < C; c += 256) {
          if (pass) {
            const double d = ch[c].wmean[i] - gmean;
            acc += ch[c].wraw[i] + (double)L * d * d;
          } else {
            acc += ch[c].wmean[i];
          }
        }
        red[t] = acc;
      }
      for (int o = 128; o > 0; o >>= 1)
        for (int t = 0; t < o; t++) red[t] += red[t + o];
      pool[1 + (pass ? n : 0) + i] = red[0];
      if (!pass && i == 0) pool[0] = (double)C;
    }
  for (int i = 0; i < n; i++) var[i] = pool[1 + n + i] / (pool[0] * (double)L);
}

/* trace: optional [chains][warmup+iterations][4], as driver_sample writes it; warm: optional [chains][warmup][n], the
 * position after every warmup iteration (what the mass-matrix tuner sees); win_mass: optional [windows][n], the pooled
 * variance of every window that closed */
static void lockstep_sample(const Model& model, const rn_config& cfg, std::vector<RNG>& rngs, double* samples, double* mass_out,
                            size_t mass_stride, rn_chain_stats* stats, double* trace, double* warm, double* win_mass,
                            int& error_flags) {
  const int C = (int)rngs.size();
  const int n = model.n();
  const size_t T = (size_t)cfg.warmup_iterations + (size_t)cfg.iterations;
  const bool pooled_step = cfg.step_adaptation == RN_ADAPT_POOLED;
  const bool pooled_mass = cfg.adaptation == RN_ADAPT_POOLED && cfg.mass_tuner == RN_MASS_DIAGONAL;
  std::vector<LockstepChain> ch(C);
  DualAvgTuner finder(cfg.delta);
  int64_t K = 0;
  for (int c = 0; c < C; c++) {
    LockstepChain& x = ch[c];
    x.rng = rngs[c];
    x.interpreted.reset(new RirDensity(model));
    x.compiled.reset(new CompiledDensity(model));
    if (!(model.h.flags & RIR_FLAG_GRADIENT)) x.adjoint.reset(new AdjointDensity(model));
    DensityFunction& d = x.adjoint ? (DensityFunction&)*x.adjoint
                                   : (model.compiled ? (DensityFunction&)*x.compiled : (DensityFunction&)*x.interpreted);
    x.sampler = make_sampler(cfg);
    x.massTuner = make_mass_tuner(cfg, n);
    x.lf.reset(new LeapFrog(d, cfg.stats_window));
    MassMatrix identity;
    x.params = x.lf->initialize(identity, x.rng);     /* Driver.scala:22 */
    x.sampler->initialize(x.params, *x.lf, x.rng);    /* :59 */
    x.wmean.assign(n, 0.0);
    x.wraw.assign(n, 0.0);
    if (!pooled_step) { /* :60, per chain */
      x.stepTuner = make_step_tuner(cfg);
      x.stepSize = x.stepTuner->initialize(x.params, *x.lf);
      x.mass = x.massTuner->initialize(*x.lf, cfg.warmup_iterations); /* :61 */
      continue;
    }
    const double s0 = finder.findReasonableStepSize(x.params, *x.lf, identity);
    int k;                                            /* s0 == 2^k exactly (0 = 2^-1075, inf = 2^1024) */
    if (s0 == 0.0)
      k = -1075;
    else if (std::isinf(s0))
      k = 1024;
    else {
      std::frexp(s0, &k);
      k -= 1;
    }
    K += std::max(-1075, std::min(1024, k));
    x.mass = x.massTuner->initialize(*x.lf, cfg.warmup_iterations); /* :61 */
  }
  double stepSize = pooled_step ? jexp(kLn2 * ((double)K / (double)C)) : 0.0; /* eps0: what DualAvgTuner.initialize returns (DualAvg.scala:6-10) */
  DualAvg da = DualAvg::apply(cfg.delta, stepSize);
  std::vector<double> sample(n), var(n);
  int win_size = cfg.initial_window_size, win_i = 0, win_j = 0, windows = 0; /* pooled mass windows: the same for every chain */
  for (int t = 0; t < cfg.warmup_iterations; t++) { /* Driver.scala:67-88, chains in lockstep */
    int64_t Q = 0;
    bool closed = false;
    for (int c = 0; c < C; c++) {
      LockstepChain& x = ch[c];
      const int64_t steps0 = x.lf->stats.leapfrogSteps;
      const int acc0 = x.lf->stats.accepted;
      const double used = pooled_step ? stepSize : x.stepSize;
      const double a = x.sampler->warmup(x.params, *x.lf, used, x.mass, x.rng);
      if (pooled_step)
        Q += (int64_t)std::rint(jexp(a) * kQScale);
      else
        x.stepSize = x.stepTuner->update(a); /* :69 */
      if (trace) {
        double* tr = trace + ((size_t)c * T + (size_t)t) * 4;
        tr[0] = a;
        tr[1] = (double)(x.lf->stats.accepted - acc0);
        tr[2] = used;
        tr[3] = (double)(x.lf->stats.leapfrogSteps - steps0);
      }
    }
    if (pooled_step) { /* stepSizeTuner.update(P_t), DualAvg.scala:58-77 */
      const double newAcceptanceProb = (double)Q / (kQScale * (double)C);
      da.iteration = da.iteration + 1;
      double avgErrorMultiplier = 1.0 / ((double)da.iteration + da.acceptanceProbUpdateDenom);
      double stepSizeMultiplier = jpow((double)da.iteration, -da.decayRate);
      da.avgError = ((1.0 - avgErrorMultiplier) * da.avgError + (avgErrorMultiplier * (da.delta - newAcceptanceProb)));
      da.logStepSize = (da.shrinkageTarget - (da.avgError * std::sqrt((double)da.iteration) / da.stepSizeUpdateDenom));
      da.logStepSizeBar = (stepSizeMultiplier * da.logStepSize + (1.0 - stepSizeMultiplier) * da.logStepSizeBar);
      stepSize = da.stepSize();
    }
    if (pooled_mass) { /* massMatrixTuner.update, :74-80, with the window statistics pooled over all chains */
      win_j += 1;
      const bool in_window = !(win_j < cfg.skip_first || (cfg.warmup_iterations - win_j) < cfg.skip_last);
      if (in_window) win_i += 1;
      for (int c = 0; c < C; c++) {
        LockstepChain& x = ch[c];
        x.lf->variables(x.params, sample.data());
        if (warm) std::memcpy(warm + ((size_t)c * cfg.warmup_iterations + t) * n, sample.data(), sizeof(double) * n);
        if (!in_window) continue;
        for (int i = 0; i < n; i++) {
          double mean = x.wmean[i];
          const double od = sample[i] - mean;
          mean += od / (double)win_i;
          x.wmean[i] = mean;
          x.wraw[i] += od * (sample[i] - mean);
        }
      }
      if (in_window && win_i == win_size) {
        pool_reduce(ch, n, win_size, var);
        if (win_mass) std::memcpy(win_mass + (size_t)windows * n, var.data(), sizeof(double) * n);
        windows += 1;
        win_i = 0;
        win_size = jd2i(win_size * cfg.window_expansion);
        closed = true;
        for (int c = 0; c < C; c++) {
          LockstepChain& x = ch[c];
          x.mass = DiagonalMassMatrix(var);
          for (int i = 0; i < n; i++) {
            if (!(var[i] > 0.0)) x.res.error_flags |= 2;
            x.wmean[i] = 0.0;
            x.wraw[i] = 0.0;
          }
        }
      }
    } else {
      for (int c = 0; c < C; c++) { /* massMatrixTuner.update, :74-80 (the windows close on the same iteration for every chain) */
        LockstepChain& x = ch[c];
        x.lf->variables(x.params, sample.data());
        if (warm) std::memcpy(warm + ((size_t)c * cfg.warmup_iterations + t) * n, sample.data(), sizeof(double) * n);
        MassMatrix m;
        if (x.massTuner->update(sample.data(), m)) {
          x.mass = m;
          if (m.invalid) x.res.error_flags |= 2;
          closed = true;
        }
      }
    }
    if (closed) { /* stepSizeTuner.reset(), DualAvg.scala:17-21 */
      if (pooled_step) {
        const double ss = da.finalStepSize();
        da = DualAvg::apply(cfg.delta, ss);
        stepSize = ss;
      } else {
        for (LockstepChain& x : ch) x.stepSize = x.stepTuner->reset();
      }
    }
  }
  for (int c = 0; c < C; c++) {
    LockstepChain& x = ch[c];
    LeapFrog& lf = *x.lf;
    const double finalStep = pooled_step ? da.finalStepSize() : x.stepTuner->stepSize(); /* Driver.scala:37 */
    lf.resetStats(); /* :31 */
    for (int i = 0; i < cfg.iterations; i++) {
      const int64_t steps0 = lf.stats.leapfrogSteps;
      const int acc0 = lf.stats.accepted;
      x.sampler->run(x.params, lf, finalStep, x.mass, x.rng);
      lf.variables(x.params, samples + ((size_t)c * cfg.iterations + i) * n);
      if (trace) {
        double* tr = trace + ((size_t)c * T + (size_t)cfg.warmup_iterations + i) * 4;
        tr[0] = lf.lastLogAcceptanceProb;
        tr[1] = (double)(lf.stats.accepted - acc0);
        tr[2] = finalStep;
        tr[3] = (double)(lf.stats.leapfrogSteps - steps0);
      }
    }
    if (x.interpreted->lookup_error | x.compiled->lookup_error | (x.adjoint ? x.adjoint->fwd.lookup_error : 0)) x.res.error_flags |= 1;
    error_flags |= x.res.error_flags;
    if (mass_out) {
      double* mo = mass_out + (size_t)c * mass_stride;
      if (x.mass.kind == RN_MATRIX_IDENTITY) {
        for (size_t e = 0; e < mass_stride; e++) mo[e] = (mass_stride == (size_t)n || e % (size_t)(n + 1) == 0) ? 1.0 : 0.0;
      } else {
        std::memcpy(mo, x.mass.elements.data(), sizeof(double) * x.mass.elements.size());
      }
    }
    if (stats) {
      const Stats& s = lf.stats;
      rn_chain_stats* st = stats + c;
      std::memset(st, 0, sizeof(*st));
      st->gradient_evaluations = s.gradientEvaluations;
      st->leapfrog_steps = s.leapfrogSteps;
      st->iterations = s.iterations;
      st->divergences = s.divergences;
      st->accepted = s.accepted;
      st->error_flags = x.res.error_flags;
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
}

} /* namespace rno */

extern "C" {
/* rno_sample_traced for pooled step sizes (cfg->step_adaptation == RN_ADAPT_POOLED, DualAvg) and / or pooled diagonal mass
 * windows (cfg->adaptation == RN_ADAPT_POOLED); warm: optional [chains][warmup][n] warmup positions; win_mass: optional
 * [windows][n] pooled variance of every closed window */
int rno_sample_pooled_step(rno_model* mm, const rn_config* cfg, const int64_t* seeds, int chains, double* samples, double* mass,
                           rn_chain_stats* stats, double* trace, double* warm, double* win_mass) {
  const bool pooled_step = cfg->step_adaptation == RN_ADAPT_POOLED, pooled_mass = cfg->adaptation == RN_ADAPT_POOLED;
  if ((pooled_step && cfg->step_size_tuner != RN_STEP_DUAL_AVG) || (pooled_mass && cfg->mass_tuner != RN_MASS_DIAGONAL) ||
      !(pooled_step || pooled_mass))
    return fail(RN_E_UNSUPPORTED, "the lockstep oracle covers pooled DualAvg steps and pooled diagonal mass windows");
  const Model& m = mm->m;
  const int n = m.n();
  const size_t mass_stride = (cfg->mass_tuner == RN_MASS_DENSE || (cfg->mass_tuner == RN_MASS_STATIC && cfg->static_matrix == RN_MATRIX_DENSE))
                                 ? (size_t)n * n
                                 : (size_t)n;
  std::vector<RNG> rngs(chains);
  for (int c = 0; c < chains; c++) rngs[c].rand = JRandom(seeds[c]); /* ScalaRNG(seed), S/RNG.scala:20-26 */
  int err = 0;
  lockstep_sample(m, *cfg, rngs, samples, mass, mass_stride, stats, trace, warm, win_mass, err);
  if (err & 1) return fail(RN_E_LOOKUP, "lookup index out of range");
  if (err & 2) return fail(RN_E_INVALID, "requirement failed: adapted mass matrix contains 0.0 (MassMatrix.scala:8,16)");
  return RN_OK;
}
} /* extern "C" */

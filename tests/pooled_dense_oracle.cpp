/* tests/pooled_dense_oracle.cpp -- TEST INFRASTRUCTURE ONLY: the lockstep oracle of pooled dense mass windows
 * (DenseMassMatrixTuner with rn_config.adaptation == RN_ADAPT_POOLED; rn_k_pool_reduce pass 0, rn_k_pool_reduce_dense,
 * rn_k_pool_factor, rn_k_pool_apply_dense in rainier_b200/csrc/rn_sampler_common.cuh), with per-chain or pooled DualAvg
 * steps.  Built on tests/pooled_step_oracle.cpp (pooled steps, chains in lockstep) and the per-chain oracle, both unchanged.
 *   per chain, the window's Welford mean and co-moment: mean += od / win_i, cov[j][k] += nd[j] * od[k] (nd = q - new mean,
 *   win_i the position in the window)
 *   at the window end, pass 0: 256 partials (thread t adds chains t, t + 256, ... from 0.0), halving tree, / C = pooled
 *   mean; pass 1 over all n^2 entries of cov_c[j][k] + (L d_c[j]) d_c[k], d_c = mean_c - pooled mean; M = sum / (C L),
 *   factored by the per-chain oracle's choleskyUpperTriangular; error flag 2 where M has an element 0.0 or a pivot is not > 0
 * Driver.scala:67-80 order (step update, mass update, stepSizeTuner.reset() when a window closed), sampling at the final
 * step size; Stats stay per chain. */
#include "pooled_step_oracle.cpp"

namespace rno {

/* rn_k_pool_reduce (pass 0) and rn_k_pool_reduce_dense (pass 1) restated (one rank): the pooled covariance M [n][n] of the
 * window that just closed, L draws per chain */
static void pool_reduce_dense(const std::vector<std::vector<double>>& wmean, const std::vector<std::vector<double>>& wcov, int n,
                              int L, std::vector<double>& M) {
  const int C = (int)wmean.size();
  const size_t nn = (size_t)n * n;
  std::vector<double> pool(1 + n + nn, 0.0);
  double red[256];
  auto tree = [&]() {
    for (int o = 128; o > 0; o >>= 1)
      for (int t = 0; t < o; t++) red[t] += red[t + o];
    return red[0];
  };
  for (int i = 0; i < n; i++) {
    for (int t = 0; t < 256; t++) {
      double acc = 0.0;
      for (int c = t; c < C; c += 256) acc += wmean[c][i];
      red[t] = acc;
    }
    pool[1 + i] = tree();
  }
  pool[0] = (double)C;
  for (size_t e = 0; e < nn; e++) {
    const int j = (int)(e / n), k = (int)(e % n);
    const double gj = pool[1 + j] / pool[0], gk = pool[1 + k] / pool[0];
    for (int t = 0; t < 256; t++) {
      double acc = 0.0;
      for (int c = t; c < C; c += 256) {
        const double dj = wmean[c][j] - gj, dk = wmean[c][k] - gk;
        acc += wcov[c][e] + (double)L * dj * dk;
      }
      red[t] = acc;
    }
    pool[1 + n + e] = tree();
  }
  for (size_t e = 0; e < nn; e++) M[e] = pool[1 + n + e] / (pool[0] * (double)L);
}

/* the shared matrix of a pooled dense window: DenseMassMatrix(M), flagged when M has an element 0.0 or a pivot is not > 0
 * (then sqrt(pivot), the diagonal of the factor, is not > 0 either) */
static MassMatrix pooled_dense_mass(const std::vector<double>& M, int n, bool& bad) {
  MassMatrix m = DenseMassMatrix(M);
  bad = m.invalid;
  for (int i = 0, row = 0; i < n; row += n - i, i++)
    if (!(m.choleskyUpperTriangular[row] > 0.0)) bad = true;
  return m;
}

/* lockstep_sample (pooled_step_oracle.cpp) with pooled dense mass windows.  warm: optional [chains][warmup][n], the position
 * after every warmup iteration; win_mass: optional [windows][n * n], the pooled covariance of every window that closed */
static void lockstep_sample_dense(const Model& model, const rn_config& cfg, std::vector<RNG>& rngs, double* samples, double* mass_out,
                                  rn_chain_stats* stats, double* trace, double* warm, double* win_mass, int& error_flags) {
  const int C = (int)rngs.size();
  const int n = model.n();
  const size_t nn = (size_t)n * n;
  const size_t T = (size_t)cfg.warmup_iterations + (size_t)cfg.iterations;
  const bool pooled_step = cfg.step_adaptation == RN_ADAPT_POOLED;
  std::vector<LockstepChain> ch(C);
  std::vector<std::vector<double>> wmean(C, std::vector<double>(n, 0.0)), wcov(C, std::vector<double>(nn, 0.0));
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
    x.lf.reset(new LeapFrog(d, cfg.stats_window));
    MassMatrix identity;
    x.params = x.lf->initialize(identity, x.rng);  /* Driver.scala:22 */
    x.sampler->initialize(x.params, *x.lf, x.rng); /* :59 */
    if (!pooled_step) {                            /* :60, per chain */
      x.stepTuner = make_step_tuner(cfg);
      x.stepSize = x.stepTuner->initialize(x.params, *x.lf);
      continue; /* the mass matrix stays the identity until the first window closes (:61) */
    }
    const double s0 = finder.findReasonableStepSize(x.params, *x.lf, identity);
    int k; /* s0 == 2^k exactly (0 = 2^-1075, inf = 2^1024) */
    if (s0 == 0.0)
      k = -1075;
    else if (std::isinf(s0))
      k = 1024;
    else {
      std::frexp(s0, &k);
      k -= 1;
    }
    K += std::max(-1075, std::min(1024, k));
  }
  double stepSize = pooled_step ? jexp(kLn2 * ((double)K / (double)C)) : 0.0; /* DualAvgTuner.initialize, DualAvg.scala:6-10 */
  DualAvg da = DualAvg::apply(cfg.delta, stepSize);
  std::vector<double> sample(n), M(nn), od(n), nd(n);
  int win_size = cfg.initial_window_size, win_i = 0, win_j = 0, windows = 0; /* the same for every chain */
  for (int t = 0; t < cfg.warmup_iterations; t++) {                        /* Driver.scala:67-88, chains in lockstep */
    int64_t Q = 0;
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
    /* massMatrixTuner.update, :74-80, with the window statistics pooled over all chains */
    win_j += 1;
    const bool in_window = !(win_j < cfg.skip_first || (cfg.warmup_iterations - win_j) < cfg.skip_last);
    if (in_window) win_i += 1;
    for (int c = 0; c < C; c++) {
      LockstepChain& x = ch[c];
      x.lf->variables(x.params, sample.data());
      if (warm) std::memcpy(warm + ((size_t)c * cfg.warmup_iterations + t) * n, sample.data(), sizeof(double) * n);
      if (!in_window) continue;
      for (int i = 0; i < n; i++) {
        double mean = wmean[c][i];
        od[i] = sample[i] - mean;
        mean += od[i] / (double)win_i;
        wmean[c][i] = mean;
        nd[i] = sample[i] - mean;
      }
      for (int j = 0; j < n; j++)
        for (int k = 0; k < n; k++) wcov[c][(size_t)j * n + k] += nd[j] * od[k];
    }
    if (in_window && win_i == win_size) {
      pool_reduce_dense(wmean, wcov, n, win_size, M);
      if (win_mass) std::memcpy(win_mass + (size_t)windows * nn, M.data(), sizeof(double) * nn);
      windows += 1;
      win_i = 0;
      win_size = jd2i(win_size * cfg.window_expansion);
      bool bad = false;
      const MassMatrix shared = pooled_dense_mass(M, n, bad); /* one factorisation for all chains */
      for (int c = 0; c < C; c++) {
        ch[c].mass = shared;
        if (bad) ch[c].res.error_flags |= 2;
        std::fill(wmean[c].begin(), wmean[c].end(), 0.0);
        std::fill(wcov[c].begin(), wcov[c].end(), 0.0);
      }
      if (pooled_step) { /* stepSizeTuner.reset(), DualAvg.scala:17-21 */
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
    lf.resetStats();                                                                       /* :31 */
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
      double* mo = mass_out + (size_t)c * nn;
      if (x.mass.kind == RN_MATRIX_IDENTITY) {
        for (size_t e = 0; e < nn; e++) mo[e] = e % (size_t)(n + 1) == 0 ? 1.0 : 0.0;
      } else {
        std::memcpy(mo, x.mass.elements.data(), sizeof(double) * nn);
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
/* rno_sample_traced for pooled dense mass windows (cfg->adaptation == RN_ADAPT_POOLED, cfg->mass_tuner == RN_MASS_DENSE) with
 * per-chain or pooled DualAvg steps or a static step; mass [chains][n * n]; warm: optional [chains][warmup][n] warmup
 * positions; win_mass: optional [windows][n * n] pooled covariance of every closed window */
int rno_sample_pooled_dense(rno_model* mm, const rn_config* cfg, const int64_t* seeds, int chains, double* samples, double* mass,
                            rn_chain_stats* stats, double* trace, double* warm, double* win_mass) {
  if (cfg->adaptation != RN_ADAPT_POOLED || cfg->mass_tuner != RN_MASS_DENSE ||
      (cfg->step_adaptation == RN_ADAPT_POOLED && cfg->step_size_tuner != RN_STEP_DUAL_AVG))
    return fail(RN_E_UNSUPPORTED, "the dense lockstep oracle covers pooled dense mass windows (with per-chain or pooled DualAvg steps)");
  std::vector<rno::RNG> rngs(chains);
  for (int c = 0; c < chains; c++) rngs[c].rand = rno::JRandom(seeds[c]); /* ScalaRNG(seed), S/RNG.scala:20-26 */
  int err = 0;
  rno::lockstep_sample_dense(mm->m, *cfg, rngs, samples, mass, stats, trace, warm, win_mass, err);
  if (err & 1) return fail(RN_E_LOOKUP, "lookup index out of range");
  if (err & 2) return fail(RN_E_INVALID, "requirement failed: adapted mass matrix contains 0.0 (MassMatrix.scala:8,16)");
  return RN_OK;
}

/* the factor the dense lockstep oracle gives every chain at a window end: upper [n(n+1)/2] of M [n*n]; returns the flag */
int rno_pooled_dense_factor(const double* M, int n, double* upper) {
  bool bad = false;
  const rno::MassMatrix m = rno::pooled_dense_mass(std::vector<double>(M, M + (size_t)n * n), n, bad);
  std::memcpy(upper, m.choleskyUpperTriangular.data(), sizeof(double) * m.choleskyUpperTriangular.size());
  return bad ? 1 : 0;
}
} /* extern "C" */

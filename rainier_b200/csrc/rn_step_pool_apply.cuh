// rn_step_pool_apply.cuh -- rn_k_step_pool: the per-iteration update of pooled step-size adaptation (see rn_step_pool.cuh for
// the semantics).  Emitted after the sampler kernels, in RN_STEP_POOL modules only.
#ifndef RN_STEP_POOL_APPLY_CUH
#define RN_STEP_POOL_APPLY_CUH

// acc: [0] K, [1] C, [2 + t] Q_t (all-reduced over ranks).  t < 0: DualAvg.apply(delta, eps0) after rn_k_init.  t >= 0: the
// update of warmup iteration t and, if `reset`, stepSizeTuner.reset() of the mass window that closed there.  One thread per
// chain; da / da_iter are [field][chains] in both kernel families.
RN_GLOBAL void rn_k_step_pool(const RnArgs A, const rn_i64* acc, int t, int reset) {
  const int c = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (c >= A.chains) return;
  const size_t ld = (size_t)A.chains;
  double* da = A.da + c;
  const double chains = (double)acc[1];
  if (t < 0) {  // DualAvg.apply, DualAvg.scala:80-90
    const double eps0 = rn_exp(RN_LN2 * ((double)acc[0] / chains));
    da[0] = eps0;
    da[1 * ld] = rn_log(eps0);
    da[2 * ld] = 0.0;
    da[3 * ld] = 0.0;
    da[4 * ld] = rn_log(10 * eps0);
    A.da_iter[c] = 0;
    return;
  }
  // DualAvg.update, DualAvg.scala:58-77, with the pooled acceptance probability
  const double newAcceptanceProb = (double)acc[2 + t] / (RN_POOL_Q_SCALE * chains);
  const int daIter = A.da_iter[c] + 1;
  const double avgErrorMultiplier = 1.0 / ((double)daIter + 10);
  const double stepSizeMultiplier = rn_pow((double)daIter, -0.75);
  const double avgError = ((1.0 - avgErrorMultiplier) * da[3 * ld] + (avgErrorMultiplier * (A.delta - newAcceptanceProb)));
  const double logStepSize = (da[4 * ld] - (avgError * sqrt((double)daIter) / 0.05));
  const double logStepSizeBar = (stepSizeMultiplier * logStepSize + (1.0 - stepSizeMultiplier) * da[2 * ld]);
  if (reset) {  // stepSizeTuner.reset(), Driver.scala:78 / DualAvg.scala:17-21
    const double ss = rn_exp(logStepSizeBar);
    da[0] = ss;
    da[1 * ld] = rn_log(ss);
    da[2 * ld] = 0.0;
    da[3 * ld] = 0.0;
    da[4 * ld] = rn_log(10 * ss);
    A.da_iter[c] = 0;
    return;
  }
  da[0] = rn_exp(logStepSize);
  da[1 * ld] = logStepSize;
  da[2 * ld] = logStepSizeBar;
  da[3 * ld] = avgError;
  A.da_iter[c] = daIter;
}

#endif  // RN_STEP_POOL_APPLY_CUH

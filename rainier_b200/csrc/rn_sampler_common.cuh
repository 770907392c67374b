// rn_sampler_common.cuh -- what the thread-per-chain (rn_sampler.cuh) and warp-per-chain (rn_sampler_wpc.cuh) kernels
// share: the adaptation arithmetic of the reference (DualAvg, the variance estimator, the mass-matrix window schedule, the
// Cholesky factorisation of a dense window end), pooled step-size adaptation and the kernels that do not depend on the
// shape (rn_k_transpose, the pooled mass-window kernels).  The emitter writes it, after rn_args.h, between the prelude and
// the density into every sampler module.  The two shapes keep the DualAvg state in different places (the thread shape
// in global memory, the warp shape in registers), so the helpers take the fields by reference and each caller passes its own
// storage.  Every floating-point operation keeps its operands and association, so parity runs keep every bit.
#ifndef RN_SAMPLER_COMMON_CUH
#define RN_SAMPLER_COMMON_CUH

#define RN_LN2 0.6931471805599453
#ifndef RN_STEP_POOL
#define RN_STEP_POOL 0 /* 1: pooled step-size adaptation (rn_k_step_pool below) */
#endif
#ifndef RN_MASS_POOL
#define RN_MASS_POOL 0 /* 1: pooled dense mass windows (rn_k_pool_reduce_dense / rn_k_pool_factor / rn_k_pool_apply_dense below) */
#endif
// field `field` of chain c in a [field][chains] (SoA) array
#define RN_AT(ptr, field, c) (ptr)[(size_t)(field) * (size_t)A.chains + (size_t)(c)]

// ---- DualAvg (rainier-sampler/src/main/scala/com/stripe/rainier/sampler/DualAvg.scala) ------------------------------
// The state is stepSize, logStepSize, logStepSizeBar, avgError, shrinkageTarget and the iteration (RnArgs::da, da_iter).
// DualAvg.apply(delta, stepSize), DualAvg.scala:80-90 (the end of findReasonableStepSize): stepSize itself stays with the caller.
RN_DEVICE void rn_da_apply(double stepSize, double& logStepSize, double& logStepSizeBar, double& avgError, double& shrinkageTarget,
                           int& iteration) {
  logStepSize = rn_log(stepSize);
  logStepSizeBar = 0.0;
  avgError = 0.0;
  iteration = 0;
  shrinkageTarget = rn_log(10 * stepSize);
}
// DualAvg.update(newAcceptanceProb), DualAvg.scala:58-77.  Returns the new logStepSize (the tuner's stepSize is its exp).
RN_DEVICE double rn_da_update(const RnArgs& A, double newAcceptanceProb, double& logStepSize, double& logStepSizeBar, double& avgError,
                              const double& shrinkageTarget, int& iteration) {
  const int daIter = iteration + 1;
  iteration = daIter;
  const double avgErrorMultiplier = 1.0 / ((double)daIter + 10);
  const double stepSizeMultiplier = rn_pow((double)daIter, -0.75);
  const double newAvgError = ((1.0 - avgErrorMultiplier) * avgError + (avgErrorMultiplier * (A.delta - newAcceptanceProb)));
  avgError = newAvgError;
  const double newLogStepSize = (shrinkageTarget - (newAvgError * sqrt((double)daIter) / 0.05));
  logStepSize = newLogStepSize;
  logStepSizeBar = (stepSizeMultiplier * newLogStepSize + (1.0 - stepSizeMultiplier) * logStepSizeBar);
  return newLogStepSize;
}
// stepSizeTuner.reset(), DualAvg.scala:17-21 (Driver.scala:75-80 at a mass-window end): DualAvg.apply at the averaged step size
// Returns the new stepSize.
RN_DEVICE double rn_da_reset(double& logStepSize, double& logStepSizeBar, double& avgError, double& shrinkageTarget, int& iteration) {
  const double ss = rn_exp(logStepSizeBar);
  rn_da_apply(ss, logStepSize, logStepSizeBar, avgError, shrinkageTarget, iteration);
  return ss;
}

// ---- mass-matrix adaptation (MassMatrix.scala, MassMatrixEstimator.scala) ------------------------------------------------
// WindowedMassMatrixTuner.update, MassMatrix.scala:147-164: warmup iteration win_j feeds the estimator.  A macro, not a
// function: as a function the test compiles to different (speculated) loads in the warp-per-chain kernel.
#define RN_IN_WINDOW(A, win_j) (!((win_j) < (A).skip_first || ((A).total_warmup - (win_j)) < (A).skip_last))
// VarianceEstimator.update, MassMatrixEstimator.scala:69-83: element i (value x) of chain c's n-th sample into est_mean /
// est_raw.  Returns newDiff and sets oldDiff, the two differences CovarianceEstimator.update (:28-41) multiplies.
RN_DEVICE double rn_variance_update(const RnArgs& A, int c, int i, double x, int n, double& oldDiff) {
  double mean = RN_AT(A.est_mean, i, c);
  const double od = x - mean;
  mean += (od / (double)n);
  const double nd = x - mean;
  RN_AT(A.est_mean, i, c) = mean;
  RN_AT(A.est_raw, i, c) += od * nd;
  oldDiff = od;
  return nd;
}
#if RN_MASS_MAX >= 2
// choleskyUpperTriangular, MassMatrix.scala:76-117: the packed upper factor (chol, [N(N+1)/2][chains]) of the dense matrix
// (mass, [N*N][chains]) of chain c, through the packed lower factor at lower[e * lower_ld].  Ld is the call site's index
// type: int for the thread shape's local array, size_t for the warp shape's [e][chains] block.
template <typename Ld>
RN_DEVICE void rn_cholesky_upper(const RnArgs& A, int c, double* lower, Ld lower_ld) {
  int l = 0;
  for (int i = 0; i < RN_N; i++)
    for (int k = 0; k <= i; k++) {
      double sum = 0.0;
      for (int j = 0; j < k; j++)
        sum += lower[((i * (i + 1)) / 2 + j) * lower_ld] * lower[((k * (k + 1)) / 2 + j) * lower_ld];
      const double x = RN_AT(A.mass, i * RN_N + k, c) - sum;
      if (i == k)
        lower[l * lower_ld] = sqrt(x);
      else {
        const double diag = lower[(((k + 1) * (k + 2)) / 2 - 1) * lower_ld];
        lower[l * lower_ld] = (1.0 / diag * x);
      }
      l += 1;
    }
  l = 0;
  for (int i = 0; i < RN_N; i++)
    for (int k = 0; k < (RN_N - i); k++) {
      RN_AT(A.chol, l, c) = lower[(((k + i) * (k + i + 1)) / 2 + i) * lower_ld];
      l += 1;
    }
}
#endif

#if RN_STEP_POOL
// ---- pooled step-size adaptation (rn_config.step_adaptation == RN_ADAPT_POOLED; an extension, not reference semantics) --
// Let C be the number of chains over all ranks.  Every quantity that crosses chains is an exact integer sum, so the
// result depends neither on chain order, CTA shape, the order of the atomics nor on how chains are split over ranks:
//   init    chain c's findReasonableStepSize ends at 2^k_c (k_c counted, clamped to [-1075, 1024]);
//           K = sum k_c, eps0 = exp(ln2 * K / C); every chain's DualAvg becomes DualAvg.apply(delta, eps0)
//   warmup  iteration t: q_c = rint(exp(a_c) * 2^32), Q_t = sum q_c, P_t = Q_t / (2^32 C); every chain applies
//           DualAvg.update with newAcceptanceProb = P_t (DualAvg.scala:58-77), then -- if a mass window closed --
//           stepSizeTuner.reset() (Driver.scala:67-80), so every chain's copy of the DualAvg state is bit-identical.
// In this mode a warmup launch covers one iteration: the sampler kernels add their terms into the iteration's int64 slot
// (rn_pool_add), the host all-reduces the slot across ranks, and rn_k_step_pool applies the update.  Compiled in only
// when the emitter defines RN_STEP_POOL, so per-chain modules are unchanged.
#define RN_POOL_Q_SCALE 4294967296.0 /* 2^32: quantum of the pooled acceptance probability */

// rint(p * 2^32) of this chain's acceptance probability p = exp(a) in [0, 1]
RN_DEVICE rn_i64 rn_pool_quantise(double p) { return (rn_i64)rint(p * RN_POOL_Q_SCALE); }

// *slot += v, exactly.  The converged lanes of the warp sum their terms first (three 22-bit limbs: a sum of 32 limbs fits 32
// bits; two's complement makes the limb sum of signed terms exact modulo 2^64) and one of them issues the atomic.  Any split
// of the chains into atomics gives the same integer.
RN_DEVICE void rn_pool_add(rn_i64* slot, rn_i64 v) {
#ifdef RN_HOST_EMULATION
  __atomic_fetch_add(slot, v, __ATOMIC_RELAXED);  // emulated warps of one CTA run as concurrent host threads
#else
  const unsigned long long u = (unsigned long long)v;
  const unsigned mask = __activemask();
  const unsigned l0 = __reduce_add_sync(mask, (unsigned)(u & 0x3FFFFFull));
  const unsigned l1 = __reduce_add_sync(mask, (unsigned)((u >> 22) & 0x3FFFFFull));
  const unsigned l2 = __reduce_add_sync(mask, (unsigned)(u >> 44));
  if ((int)(threadIdx.x & 31) == __ffs(mask) - 1)
    atomicAdd((unsigned long long*)slot, (unsigned long long)l0 + ((unsigned long long)l1 << 22) + ((unsigned long long)l2 << 44));
#endif
}

// rn_k_init's share of K and C: the chain's findReasonableStepSize ended at 2^log2Step (doubling / halving 1.0 is exact down
// to 0 = 2^-1075 and up to inf = 2^1024)
RN_DEVICE void rn_pool_add_initial_step(rn_i64* acc, int log2Step) {
  rn_pool_add(acc + 0, log2Step < -1075 ? -1075 : (log2Step > 1024 ? 1024 : log2Step));
  rn_pool_add(acc + 1, 1);
}

// acc: [0] K, [1] C, [2 + t] Q_t (all-reduced over ranks).  t < 0: DualAvg.apply(delta, eps0) after rn_k_init.  t >= 0: the
// update of warmup iteration t and, if `reset`, stepSizeTuner.reset() of the mass window that closed there.  One thread per
// chain; da / da_iter are [field][chains] in both kernel families.
RN_GLOBAL void rn_k_step_pool(const RnArgs A, const rn_i64* acc, int t, int reset) {
  const int c = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (c >= A.chains) return;
  const size_t ld = (size_t)A.chains;
  double* da = A.da + c;
  const double chains = (double)acc[1];
  if (t < 0) {
    const double eps0 = rn_exp(RN_LN2 * ((double)acc[0] / chains));
    da[0] = eps0;
    rn_da_apply(eps0, da[1 * ld], da[2 * ld], da[3 * ld], da[4 * ld], A.da_iter[c]);
    return;
  }
  const double newAcceptanceProb = (double)acc[2 + t] / (RN_POOL_Q_SCALE * chains);
  const double logStepSize = rn_da_update(A, newAcceptanceProb, da[1 * ld], da[2 * ld], da[3 * ld], da[4 * ld], A.da_iter[c]);
  if (reset)
    da[0] = rn_da_reset(da[1 * ld], da[2 * ld], da[3 * ld], da[4 * ld], A.da_iter[c]);
  else
    da[0] = rn_exp(logStepSize);
}
#endif  // RN_STEP_POOL

#ifndef RN_TRAJ_POOL
#define RN_TRAJ_POOL 0 /* 1: pooled EHMC trajectory lengths in the sampling phase (rn_traj_length below) */
#endif
#if RN_TRAJ_POOL
// ---- pooled trajectory lengths (rn_config.trajectory_adaptation == RN_ADAPT_POOLED; an extension) ------------------------
// Warmup fills every chain's ring of U-turn counts as the reference does.  Before the first sampling launch rn_k_traj_hist
// counts, over every chain, the ring entries steps.sample() would choose from (indices [0, ring_full ? buf_size : ring_i + 1),
// Stats.scala:40-45) into h[l]; the host all-reduces h over ranks (int64) and uploads the prefix sums c.  Sampling iteration t
// of every chain then takes L_t steps (the definition is in rainier_cuda.h, rn_config.trajectory_adaptation): a function of
// the histogram and t alone, so no chain's RNG is consumed and every chain of a warp or CTA runs the same trajectory length.
RN_GLOBAL void rn_k_traj_hist(const RnArgs A) {
  const int c = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (c >= A.chains) return;
  const int k = A.ring_full[c] ? A.buf_size : A.ring_i[c] + 1;
  for (int i = 0; i < k; i++) {
    const int l = rn_d2i(RN_AT(A.ring, i, c));  // 0 <= l <= max_steps (countSteps stops at maxSteps, EHMC.scala:32-50)
#ifdef RN_HOST_EMULATION
    __atomic_fetch_add(&A.traj_hist[l], (rn_i64)1, __ATOMIC_RELAXED);
#else
    atomicAdd((unsigned long long*)&A.traj_hist[l], 1ull);
#endif
  }
}

// L_t: z = splitmix64(F + (t + 1) * 0x9E3779B97F4A7C15), r = mulhi64(z, T), L_t = min { l : c[l] > r }.  Every thread of a warp
// evaluates it with the same arguments, so the binary search over the prefix table is warp-uniform.
RN_DEVICE int rn_traj_length(const RnArgs& A, rn_i64 t) {
  unsigned long long z = (unsigned long long)A.traj_fp + (unsigned long long)(t + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z = z ^ (z >> 31);
#ifdef RN_HOST_EMULATION
  const unsigned long long r = (unsigned long long)(((unsigned __int128)z * (unsigned long long)A.traj_total) >> 64);
#else
  const unsigned long long r = __umul64hi(z, (unsigned long long)A.traj_total);
#endif
  int lo = 0, hi = A.traj_bins - 1;  // c[traj_bins - 1] = T > r
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((unsigned long long)A.traj_cum[mid] > r)
      hi = mid;
    else
      lo = mid + 1;
  }
  return lo;
}
#endif  // RN_TRAJ_POOL

#ifndef RN_HOST_EMULATION
// =============================================================================================================
// rn_k_transpose: [rows][cols] -> [cols][rows] (sample chunks [iter][n][chain] -> [chain][iter][n] before the
// device->host copy of rn_sample).  32x32 tiles through shared memory, both sides coalesced.
// =============================================================================================================
RN_GLOBAL void rn_k_transpose(const double* RN_RESTRICT src, double* RN_RESTRICT dst, int rows, int cols,
                              long long src_ld, long long dst_ld, long long dst_off) {
  // dst[c * dst_ld + dst_off + r] = src[r * src_ld + c]   (a block of `cols` chains out of src_ld)
  __shared__ double tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    if (r < rows && c < cols) tile[j][threadIdx.x] = src[(size_t)r * (size_t)src_ld + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r < rows && c < cols) dst[(size_t)c * (size_t)dst_ld + (size_t)dst_off + r] = tile[threadIdx.x][j];
  }
}

// =============================================================================================================
// Pooled mass-matrix adaptation (RN_ADAPT_POOLED; an extension, not reference semantics): at a window end the
// chains' Welford statistics of the window (mean_c, M2_c over L draws) are reduced over all chains of this GPU in two
// passes -- pool[0] = number of chains and pool[1..n] = sum of the means, all-reduced over ranks by the host (NCCL),
// then pool[n+1..2n] = sum of M2_c + L (mean_c - pooled mean)^2, all-reduced again -- and applied to every chain: one
// shared diagonal mass matrix, statistics cleared, DualAvg restarted from each chain's averaged step size
// (Driver.scala:75-80).
// =============================================================================================================
RN_GLOBAL void rn_k_pool_reduce(const RnArgs A, double* pool, int window_len, int pass) {
  // One block per parameter; thread t adds chains t, t + 256, ... in order, then a fixed tree: the result does not depend
  // on scheduling (no atomics).  pass 0: pool[1 + i] = sum over chains of the chain's window mean, pool[0] = chains.
  // pass 1 (after the all-reduce of pass 0): pool[1 + n + i] = sum over chains of [M2_c + L (mean_c - mean)^2] -- Chan's
  // combination of the chains' Welford statistics around the POOLED mean (no s2/n - mean^2 cancellation).
  __shared__ double red[256];
  const int i = (int)blockIdx.x;
  const double gmean = pass ? pool[1 + i] / pool[0] : 0.0;
  const double* mean = A.est_mean + (size_t)i * A.chains;
  const double* m2 = A.est_raw + (size_t)i * A.chains;
  double acc = 0.0;
  for (int c = (int)threadIdx.x; c < A.chains; c += (int)blockDim.x) {
    if (pass) {
      const double d = mean[c] - gmean;
      acc += m2[c] + (double)window_len * d * d;
    } else {
      acc += mean[c];
    }
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = (int)blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    pool[1 + (pass ? RN_N : 0) + i] = red[0];
    if (!pass && i == 0) pool[0] = (double)A.chains;
  }
}
RN_GLOBAL void rn_k_pool_apply(const RnArgs A, const double* pool, int window_len) {
  const int c = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (c >= A.chains) return;
  const double cnt = pool[0] * (double)window_len;  // draws of the window over all chains of all ranks
  for (int i = 0; i < RN_N; i++) {
    const double var = pool[1 + RN_N + i] / cnt;
    if (!(var > 0.0)) A.st_err[c] |= 2;
    RN_AT(A.mass, i, c) = var;
    RN_AT(A.est_mean, i, c) = 0.0;
    RN_AT(A.est_raw, i, c) = 0.0;
  }
  if (A.step_tuner == 0)
    RN_AT(A.da, 0, c) = rn_da_reset(RN_AT(A.da, 1, c), RN_AT(A.da, 2, c), RN_AT(A.da, 3, c), RN_AT(A.da, 4, c), A.da_iter[c]);
}

#if RN_MASS_POOL
// ---- pooled dense mass windows (DenseMassMatrixTuner with RN_ADAPT_POOLED; an extension, not reference semantics) ---------
// The chains keep their window mean and co-moment C2[j][k] += newDiff[j] * oldDiff[k] (CovarianceEstimator.update,
// MassMatrixEstimator.scala:22-36) with the position in the window as the count.  At a window end pass 0 is rn_k_pool_reduce's
// (pool[0] = chains, pool[1..n] = sum of the means), then pool[1 + n + j n + k] = sum over chains of
// C2_c[j][k] + (L d_c[j]) d_c[k], d_c = mean_c - pooled mean, over all n^2 entries (C2 is not exactly symmetric and the
// velocity reads the full matrix).  M = S / (C L), with the diagonal kernels' association throughout, so M's diagonal is
// the pooled diagonal tuner's variance bit for bit.  rn_k_pool_factor factors M once, in one CTA, into the scratch behind
// the pool; rn_k_pool_apply_dense broadcasts M and the factor to every chain.
// pool layout: [0] C | [1, 1+n) sum of means | [1+n, 1+n+n^2) S | lower factor [n(n+1)/2] | upper factor [n(n+1)/2] | flag
#define RN_POOL_TRI ((RN_N * (RN_N + 1)) / 2)
#define RN_POOL_FACTOR_OFF (1 + RN_N + RN_N * RN_N)
RN_GLOBAL void rn_k_pool_reduce_dense(const RnArgs A, double* pool, int window_len) {
  // one block per entry e = j n + k, rn_k_pool_reduce's order: thread t adds chains t, t + 256, ..., then a halving tree
  __shared__ double red[256];
  const int e = (int)blockIdx.x, j = e / RN_N, k = e % RN_N;
  const double gj = pool[1 + j] / pool[0], gk = pool[1 + k] / pool[0];
  const double* mj = A.est_mean + (size_t)j * A.chains;
  const double* mk = A.est_mean + (size_t)k * A.chains;
  const double* cov = A.est_cov + (size_t)e * A.chains;
  double acc = 0.0;
  for (int c = (int)threadIdx.x; c < A.chains; c += (int)blockDim.x) {
    const double dj = mj[c] - gj, dk = mk[c] - gk;
    acc += cov[c] + (double)window_len * dj * dk;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = (int)blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) pool[1 + RN_N + e] = red[0];
}
// choleskyUpperTriangular (MassMatrix.scala:76-117) of M = S / (C L), column by column: for column k every row i >= k
// forms x_i = M[i][k] - sum_{j<k} L[i][j] L[k][j] with its own sequential sum from j = 0, then L[k][k] = sqrt(x_k) and
// L[i][k] = 1 / L[k][k] * x_i.  Each entry is the operation sequence of rn_cholesky_upper, so parity builds give its bits.
// Flag = 1 when M has an element equal to 0.0 (MassMatrix.scala:16) or a pivot is not > 0.  One CTA, thread t owns rows
// t, t + blockDim.x, ...; the factor stays in global memory (a packed factor at n = 512 does not fit in shared memory).
RN_GLOBAL void rn_k_pool_factor(double* pool, int window_len) {
  __shared__ double xs[RN_N];
  const double cnt = pool[0] * (double)window_len;
  const double* S = pool + 1 + RN_N;
  double* lower = pool + RN_POOL_FACTOR_OFF;
  double* upper = lower + RN_POOL_TRI;
  int bad = 0;
  for (int e = (int)threadIdx.x; e < RN_N * RN_N; e += (int)blockDim.x)
    if (S[e] / cnt == 0.0) bad = 1;
  for (int k = 0; k < RN_N; k++) {
    for (int i = k + (int)threadIdx.x; i < RN_N; i += (int)blockDim.x) {
      double sum = 0.0;
      for (int j = 0; j < k; j++) sum += lower[(i * (i + 1)) / 2 + j] * lower[(k * (k + 1)) / 2 + j];
      xs[i] = S[i * RN_N + k] / cnt - sum;
    }
    __syncthreads();
    const double diag = sqrt(xs[k]);
    if (threadIdx.x == 0 && !(diag > 0.0)) bad = 1;
    for (int i = k + (int)threadIdx.x; i < RN_N; i += (int)blockDim.x) {
      const double v = i == k ? diag : (1.0 / diag * xs[i]);
      lower[(i * (i + 1)) / 2 + k] = v;
      upper[k * RN_N - (k * (k - 1)) / 2 + (i - k)] = v;  // row k of the packed upper factor, column i
    }
    __syncthreads();
  }
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) upper[RN_POOL_TRI] = bad ? 1.0 : 0.0;
}
// every chain: M (mass, [n^2][chains]) and the packed upper factor (chol, [n(n+1)/2][chains]), estimator cleared, error flag
// 2 where rn_k_pool_factor flagged, DualAvg restarted as in rn_k_pool_apply.  x: chains; y: entries strided by gridDim.y.
RN_GLOBAL void rn_k_pool_apply_dense(const RnArgs A, const double* pool, int window_len) {
  const int c = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (c >= A.chains) return;
  const double cnt = pool[0] * (double)window_len;
  const double* S = pool + 1 + RN_N;
  const double* upper = pool + RN_POOL_FACTOR_OFF + RN_POOL_TRI;
  for (int e = (int)blockIdx.y; e < RN_N * RN_N; e += (int)gridDim.y) {
    RN_AT(A.mass, e, c) = S[e] / cnt;
    RN_AT(A.est_cov, e, c) = 0.0;
  }
  for (int e = (int)blockIdx.y; e < RN_POOL_TRI; e += (int)gridDim.y) RN_AT(A.chol, e, c) = upper[e];
  for (int i = (int)blockIdx.y; i < RN_N; i += (int)gridDim.y) {
    RN_AT(A.est_mean, i, c) = 0.0;
    RN_AT(A.est_raw, i, c) = 0.0;
  }
  if (blockIdx.y != 0) return;
  if (upper[RN_POOL_TRI] != 0.0) A.st_err[c] |= 2;
  if (A.step_tuner == 0)
    RN_AT(A.da, 0, c) = rn_da_reset(RN_AT(A.da, 1, c), RN_AT(A.da, 2, c), RN_AT(A.da, 3, c), RN_AT(A.da, 4, c), A.da_iter[c]);
}
#endif  // RN_MASS_POOL
#endif  // !RN_HOST_EMULATION

#endif  // RN_SAMPLER_COMMON_CUH

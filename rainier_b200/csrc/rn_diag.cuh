// rn_diag.cuh -- on-device convergence diagnostics over a device-resident sample block: the reductions behind
// Trace.diagnostics (rainier-core/src/main/scala/com/stripe/rainier/core/Trace.scala:11-21,49-121: rHat / v of the
// Stan manual 30.3, variogram-based autocorrelation / effective sample size of 30.4).  With thousands of chains the
// reference's host-side loops (O(chains * iterations * lags) over List[List[Array[Double]]]) and the device->host copy
// of every sample dominate the call; here only [n][2] numbers leave the device.
//
//   rn_k_diag_chain   one thread per (parameter, chain): mean, variance and the variograms of lags 1..max_lag of that
//                     chain's series (summed over iterations in the reference's sequential order), reduced over the 128
//                     chains of the block in a fixed order.
//   rn_k_diag_reduce  fixed-shape tree sums over blocks / chains (deterministic), optionally of squared deviations.
//   rn_k_diag_accum   tracked diagnostics: the same sums carried from one sampling launch to the next (no sample block).
//   rn_k_diag_terms   tracked diagnostics: the per-chain terms of the tracked state, for rn_k_diag_reduce.
// The scalar epilogue (b, w, v, rHat, the lag loop with its termination rule, ess) runs on the host in rn_runtime.cpp.
#ifndef RN_DIAG_CUH
#define RN_DIAG_CUH
#ifndef RN_HOST_EMULATION

// sample(t, i, c) = s[t*st + i*si + c*sc].  grid = (ceil(C/128), n), 128 threads: thread = chain, blockIdx.y = parameter.
// The chain's series is staged once in shared memory (x[t][thread], conflict-free) when iterations*128 doubles fit
// (`use_smem`), so the O(iterations * lags) variogram loops never touch global memory again.  Per block the 128 chains'
// contributions are added in a fixed order (warp shuffles, then 4 warp totals) and written as one partial per
// (quantity, parameter, block): partial[(q * n + i) * nblk + blockIdx.x], q = 0 mean, 1 variance, 2.. variogram(lag).
extern __shared__ double rn_diag_smem[];
RN_DEVICE double rn_diag_block_sum(double v, double* red4) {
  RN_UNROLL
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red4[threadIdx.x >> 5] = v;
  __syncthreads();
  return ((red4[0] + red4[1]) + red4[2]) + red4[3];
}
RN_GLOBAL void rn_k_diag_chain(const double* RN_RESTRICT s, long long st, long long si, long long sc, int I, int n, int C,
                               int max_lag, int use_smem, double* RN_RESTRICT mean, double* RN_RESTRICT partial) {
  __shared__ double red4[4];
  const int i = blockIdx.y, c = blockIdx.x * 128 + threadIdx.x, nblk = gridDim.x;
  const bool live = c < C;
  const double* xg = s + (long long)i * si + (long long)(live ? c : 0) * sc;
  double* xs = rn_diag_smem + threadIdx.x;  // x[t] at xs[t * 128]
  if (use_smem)
    for (int t = 0; t < I; t++) xs[(size_t)t * 128] = live ? xg[(long long)t * st] : 0.0;
#define RN_DIAG_X(t) (use_smem ? xs[(size_t)(t) * 128] : (live ? xg[(long long)(t) * st] : 0.0))
  double sum = 0.0;  // t.sum / n, Trace.scala:69-71 (sequential over iterations, like the reference)
  for (int t = 0; t < I; t++) sum += RN_DIAG_X(t);
  const double m = sum / (double)I;
  double ss = 0.0;  // t.map(a => pow(a - m, 2)).sum / (n - 1), Trace.scala:79-86
  for (int t = 0; t < I; t++) {
    const double d = RN_DIAG_X(t) - m;
    ss += d * d;
  }
  if (live) mean[(size_t)i * C + c] = m;
  double tot = rn_diag_block_sum(live ? m : 0.0, red4);
  if (threadIdx.x == 0) partial[((size_t)0 * n + i) * nblk + blockIdx.x] = tot;
  tot = rn_diag_block_sum(live ? ss / (double)(I - 1) : 0.0, red4);
  if (threadIdx.x == 0) partial[((size_t)1 * n + i) * nblk + blockIdx.x] = tot;
  for (int lag = 1; lag <= max_lag; lag++) {  // Trace.variogram, Trace.scala:111-119
    double v = 0.0;
    for (int t = lag; t < I; t++) {
      const double d = RN_DIAG_X(t) - RN_DIAG_X(t - lag);
      v += d * d;
    }
    tot = rn_diag_block_sum(live ? v / (double)(I - lag) : 0.0, red4);
    if (threadIdx.x == 0) partial[((size_t)(1 + lag) * n + i) * nblk + blockIdx.x] = tot;
  }
#undef RN_DIAG_X
}

// out[q] = sum_c f(in[q*C + c]),  f(x) = x or (x - shift[q])^2 ; one 256-thread block per q
RN_GLOBAL void rn_k_diag_reduce(const double* RN_RESTRICT in, int C, const double* RN_RESTRICT shift, double* RN_RESTRICT out) {
  __shared__ double red[256];
  const int q = blockIdx.x;
  const double sh = shift ? shift[q] : 0.0;
  double acc = 0.0;
  for (int c = threadIdx.x; c < C; c += 256) {
    const double x = in[(size_t)q * C + c];
    acc += shift ? (x - sh) * (x - sh) : x;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[q] = red[0];
}

#endif

// Trace.thin(thin).diagnostics accumulated while sampling (rn_sampler_track_diagnostics): no sample block is kept.  Every
// quantity of the reference is a sum in iteration order that can be carried from one draw to the next -- the chain's sum
// (Trace.scala:65-67) and, per lag, the variogram sum of (x_t - x_{t-lag})^2 (:112-120) -- and the ESS loop only adds lags
// 1..99 (`lag < 100`, :106), so a (parameter, chain) pair keeps the last 99 kept draws and 99 variogram accumulators.  The
// chain variance, a two-pass form around the final mean in the reference (:75-81), is carried as Welford mean and M2.
// State, RN_DIAG_FIELDS doubles per pair, field-major with the chain fastest: state[(f * n + i) * C + c];
//   f = 0 sum, 1 Welford mean, 2 Welford M2, 3 + (t % 99) kept draw t of the ring, 3 + 99 + lag - 1 variogram(lag).
#define RN_DIAG_LAGS 99
#define RN_DIAG_FIELDS (3 + 2 * RN_DIAG_LAGS)
#define RN_DIAG_GROUP 9  // lags updated together: 2 shared-memory loads per 9 FMAs (RN_DIAG_LAGS % RN_DIAG_GROUP == 0)
#ifdef RN_HOST_EMULATION
static thread_local double* rn_diag_accum_smem;  // the emulation driver's buffer, (RN_DIAG_LAGS + sub) * blockDim.x doubles
#define RN_DIAG_ACCUM_SMEM rn_diag_accum_smem
#else
#define RN_DIAG_ACCUM_SMEM rn_diag_smem
#endif

// One thread per (chain, parameter): grid = (ceil(C / blockDim.x), n).  s: one sampling launch's draws, [k][n][C]; the
// launch keeps its draws j0, j0 + thin, .. (m of them), which are kept draws T0 .. T0 + m - 1 of the tracked run.  The
// thread's column of dynamic shared memory holds rows x[0..99) = kept draws T - 99 .. T - 1 (the ring) and x[99..99+sub) =
// up to `sub` new draws; per stage every accumulator is loaded once, takes its new terms in increasing t, and is stored
// once.  The order of every sum is the reference's whatever the launches were, so any split of a run into rn_sampler_run
// calls gives the same bits.  No warp primitive or barrier: each thread reads and writes only its own column.
RN_GLOBAL void rn_k_diag_accum(const double* RN_RESTRICT s, int n, int C, int j0, int thin, int m, long long T0, int sub,
                               double* RN_RESTRICT state) {
  const int i = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x, B = blockDim.x;
  if (c >= C) return;
  const size_t P = (size_t)n * C, at = (size_t)i * C + c;
  double* st = state + at;
  double* x = RN_DIAG_ACCUM_SMEM + threadIdx.x;
#define RN_DIAG_ROW(r) x[(size_t)(r) * B]
  long long T = T0;
  for (int r = 0; r < RN_DIAG_LAGS; r++) {  // kept draws of negative index are never read as a term
    const long long t = T - RN_DIAG_LAGS + r;
    RN_DIAG_ROW(r) = t >= 0 ? st[(size_t)(3 + t % RN_DIAG_LAGS) * P] : 0.0;
  }
  double sum = st[0], mean = st[P], m2 = st[2 * P];
  for (int r0 = 0; r0 < m; r0 += sub) {
    const int k = (m - r0) < sub ? (m - r0) : sub;
    for (int r = 0; r < k; r++) {
      const double v = s[(size_t)(j0 + (size_t)(r0 + r) * thin) * P + at];
      RN_DIAG_ROW(RN_DIAG_LAGS + r) = v;
      sum += v;
      const double d = v - mean;  // VarianceEstimator-style Welford update, count = kept index + 1
      mean += d / (double)(T + r + 1);
      m2 += d * (v - mean);
    }
    for (int l0 = 1; l0 <= RN_DIAG_LAGS; l0 += RN_DIAG_GROUP) {
      double acc[RN_DIAG_GROUP], w[RN_DIAG_GROUP];  // w[g] = x_{t - l0 - g}, slid along t
      RN_UNROLL
      for (int g = 0; g < RN_DIAG_GROUP; g++) {
        acc[g] = st[(size_t)(3 + RN_DIAG_LAGS + l0 + g - 1) * P];
        w[g] = RN_DIAG_ROW(RN_DIAG_LAGS - l0 - g);
      }
      for (int r = 0; r < k; r++) {
        const double xt = RN_DIAG_ROW(RN_DIAG_LAGS + r);
        const long long t = T + r;
        RN_UNROLL
        for (int g = 0; g < RN_DIAG_GROUP; g++)
          if (t >= l0 + g) {
            const double d = xt - w[g];
            acc[g] += d * d;
          }
        RN_UNROLL
        for (int g = RN_DIAG_GROUP - 1; g > 0; g--) w[g] = w[g - 1];
        w[0] = RN_DIAG_ROW(RN_DIAG_LAGS + r + 1 - l0);
      }
      RN_UNROLL
      for (int g = 0; g < RN_DIAG_GROUP; g++) st[(size_t)(3 + RN_DIAG_LAGS + l0 + g - 1) * P] = acc[g];
    }
    for (int r = 0; r < RN_DIAG_LAGS; r++) RN_DIAG_ROW(r) = RN_DIAG_ROW(r + k);  // the newest 99 rows become the ring
    T += k;
  }
  for (int r = RN_DIAG_LAGS - (m < RN_DIAG_LAGS ? m : RN_DIAG_LAGS); r < RN_DIAG_LAGS; r++) {
    const long long t = T - RN_DIAG_LAGS + r;
    if (t >= 0) st[(size_t)(3 + t % RN_DIAG_LAGS) * P] = RN_DIAG_ROW(r);
  }
  st[0] = sum;
  st[P] = mean;
  st[2 * P] = m2;
#undef RN_DIAG_ROW
}

// The per-chain terms of Trace.diagnostics from the tracked state of T kept draws, quantity q = 0 mean (sum / T), 1 variance
// (M2 / (T - 1)), 1 + lag variogram(lag) / (T - lag) for lag = 1..L -- rn_k_diag_chain's quantity order -- for the quantities
// q0 .. q0 + nq - 1, so that rn_k_diag_reduce sums them over chains: out[((q - q0) * n + i) * C + c].  One thread per
// (chain, parameter): grid = (ceil(C / 128), n).
RN_GLOBAL void rn_k_diag_terms(const double* RN_RESTRICT state, int n, int C, long long T, int L, int q0, int nq, double* RN_RESTRICT out) {
  const int i = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const size_t P = (size_t)n * C, at = (size_t)i * C + c;
  for (int q = q0; q < q0 + nq && q <= 1 + L; q++) {
    double v;
    if (q == 0)
      v = state[at] / (double)T;
    else if (q == 1)
      v = state[2 * P + at] / (double)(T - 1);
    else
      v = state[(size_t)(3 + RN_DIAG_LAGS + q - 2) * P + at] / (double)(T - (q - 1));
    out[(size_t)(q - q0) * P + at] = v;
  }
}
#endif  // RN_DIAG_CUH

// rn_sampler_wpc.cuh -- "warp per chain" variant of the fused HMC/EHMC iteration kernels (RN_BACKEND == 1).
//
// Used when the frozen DAG streams observation rows (or has too many parameters for registers): the 32 lanes of
// a warp own ONE chain.  Rows of a streamed target are spread over the lanes (coalesced 256-byte column reads,
// per-lane partial sums, butterfly __shfl_xor reduction -- see the emitted rn_density()); the chain's vectors
// (q, p, gradient, mass) live in the warp's slice of shared memory and are updated lane-parallel; every scalar
// decision (energies, RNG draws, accept test, step-size adaptation) is computed redundantly and identically by
// all lanes, so the control flow stays warp-uniform and follows the reference exactly as in rn_sampler.cuh
// (same file:line citations apply).  Sequential reductions of the reference (dot products, LeapFrog.scala:221-231)
// keep their left-to-right order; only the row sum of the density changes order (tree instead of sequential),
// which moves results in the last ~3 digits (SURVEY.md 7.3-2).
//
// Supported here: HMC / EHMC, DualAvg / static step size, identity / diagonal / dense mass (adaptive or static).
// Dense mass (RN_MASS_MAX == 2; opt-in for this shape, AUTO keeps dense configurations on the thread-per-chain kernels):
// the n x n matrix, its packed Cholesky factor and the covariance estimator stay in the chain's global-memory state --
// for the streamed models this shape serves, n^2 loads per leapfrog step are noise beside rows x columns per gradient --
// row i of every mat-vec belongs to lane i % RN_G and is summed left to right like DenseMassMatrix.squareMultiply
// (MassMatrix.scala:35-51); the back-substitution of the momentum draw and the Cholesky factorisation at a window end are
// sequential by nature and run on one lane, in the reference's order.
#ifndef RN_SAMPLER_WPC_CUH
#define RN_SAMPLER_WPC_CUH

// RnArgs (rn_args.h), RN_AT and the adaptation arithmetic: rn_sampler_common.cuh
#define RN_LANE ((int)(threadIdx.x % RN_G))  // thread index inside the chain's group (RN_G, RN_SYNC: rn_prelude.cuh)
#define RN_FOR_LANES(i) for (int i = RN_LANE; i < RN_N; i += RN_G)

struct RnStats {
  rn_i64 grads, steps;
  int iters, accepted, err;
  double e_mean, e_raw, trans2;
  int e_n;
  int ring_i[3], ring_full[3];
};

// ---- shared data tiles (RN_TMA_STAGES > 0) --------------------------------------------------------------------
// The observation columns are laid out tile-major ([tile][column][32 rows], rn_runtime.cpp), so one tile of a streamed
// target is one contiguous chunk.  When every chain of the CTA evaluates the density the same number of times (HMC:
// control flow is uniform over chains), the CTA walks the tiles in lockstep: one thread fetches tile t+S-1 with a single
// cp.async.bulk (TMA, completion on an mbarrier) while all warps consume tile t from shared memory, so a tile crosses
// L2 -> SM once per CTA instead of once per chain.  EHMC (per-chain trajectory lengths) and the init kernel keep the
// independent per-warp path (__ldg from L2/L1).  struct RnTma and the mbarrier / bulk-copy helpers live in rn_prelude.cuh.
// Where a chain's state lives (RN_WPC_PLACE, chosen by rn_runtime.cpp:wpc_place from the sizes): 0 all of it in the chain's
// shared-memory slice; 1 the chain vectors (q, p, gradient, mass, EHMC snapshot, dense work vectors) and the density scratch in
// the chain's slice of RnArgs::wpc_state in global memory, with only the cross-warp reduction slots left in shared memory.  The
// global slices are chain-major and 128-byte aligned, so the lane-strided loops over a vector stay coalesced.
// A slice carries nothing from one launch to the next (every launch reloads q, p, gradient and mass from RnArgs), so the host
// emulation (tests/host_emulation.py), which runs one CTA at a time and passes no slice array, keeps the slices of one
// emulated CTA's chains in a static array of its own.
#if RN_WPC_PLACE == 0
#define RN_WPC_GSLICE(state, c) ((double*)nullptr)
#elif defined(RN_HOST_EMULATION)
static double rn_emu_wpc_state[(size_t)RN_WPC_GLOBAL_DOUBLES * 32];  // up to 32 chains per emulated CTA
#define RN_WPC_GSLICE(state, c) (rn_emu_wpc_state + (size_t)RN_GROUP * (size_t)RN_WPC_GLOBAL_DOUBLES)
#else
#define RN_WPC_GSLICE(state, c) ((state) + (size_t)(c) * (size_t)RN_WPC_GLOBAL_DOUBLES)
#endif
#ifdef RN_WPC_EXPECT_SMEM  // what rn_runtime.cpp:get_kernel allocates per chain; a mismatch is a slice overrun on the device
static_assert(RN_WPC_SMEM_DOUBLES == RN_WPC_EXPECT_SMEM, "launcher and kernel disagree on the shared-memory slice of a chain");
#endif
#ifdef RN_WPC_EXPECT_GLOBAL
static_assert(RN_WPC_GLOBAL_DOUBLES == RN_WPC_EXPECT_GLOBAL, "launcher and kernel disagree on the global-memory slice of a chain");
#endif
// per-chain state
struct RnW {
  double* q;   // pqBuf.q
  double* p;   // pqBuf.p
  double* g;   // gradient at q
  double* m;   // diagonal mass (variances)
  double* sq;  // EHMC snapshot
  double* sp;
  double* sg;
  double* scr;  // emitted density scratch (lookup tables, scatter accumulators)
  double* red;  // its cross-warp reduction slots (RN_WPC_K doubles and more; shared memory in every placement)
#if RN_MASS_MAX >= 2
  double* v;    // dense mass: velocity M^-1 p / oldDiff of the covariance estimator
  double* v2;   //             newDiff
  const double* M;     // [N*N][chains] (this chain's column of the SoA array)
  const double* chol;  // packed upper Cholesky factor [N(N+1)/2][chains]
  size_t ld;           // chains
#endif
  double U;     // potential of pqBuf (replicated in registers)
  int mass_kind;
  RnTma tma;    // shared data-tile pipeline of the CTA (off unless the kernel enables it)
};

// sbase: the chain's shared-memory slice (RN_WPC_SMEM_DOUBLES); gbase: its global-memory slice (RN_WPC_GLOBAL_DOUBLES)
RN_DEVICE void rn_w_setup(RnW& w, double* sbase, double* gbase) {
  w.tma.on = 0;
  w.tma.seq = 0;
  w.tma.nthreads = 0;
  w.tma.stage = nullptr;
  w.tma.full = nullptr;
#if RN_WPC_PLACE == 0
  (void)gbase;
  double* const base = sbase;
#else
  double* const base = gbase;
#endif
  w.q = base;
  w.p = base + RN_N;
  w.g = base + 2 * RN_N;
  // RN_W_VECS (rn_emit.cpp: wpc_vectors()) = 3 with the identity mass compiled in alone -- no mass vector: on cfg 5 those 8 KB
  // per chain are what lets a second data-tile stage fit beside 4 chains
#if RN_MASS_MAX >= 1
  w.m = base + 3 * RN_N;
  double* const rest = base + 4 * RN_N;
#else
  w.m = base;  // never read: mass_kind stays 0
  double* const rest = base + 3 * RN_N;
#endif
#if RN_ENABLE_EHMC
  w.sq = rest;
  w.sp = rest + RN_N;
  w.sg = rest + 2 * RN_N;
  w.scr = rest + 3 * RN_N;
#else
  w.sq = w.sp = w.sg = base;
  w.scr = rest;
#endif
#if RN_MASS_MAX >= 2
  w.v = w.scr;  // the slice is [vectors | v | v2 | density scratch] when dense mass is compiled in
  w.v2 = w.scr + RN_N;
  w.scr = w.scr + 2 * RN_N;
  w.M = nullptr;
  w.chol = nullptr;
  w.ld = 0;
#endif
#if RN_WPC_PLACE == 1
  w.red = sbase;
#else
  w.red = w.scr + RN_WPC_RED_OFF;
#endif
}

#if RN_MASS_MAX >= 2
// (M^-1 p)_i for the rows of this lane, left to right over j (DenseMassMatrix.squareMultiply, MassMatrix.scala:35-51)
RN_DEVICE double rn_dense_row(const RnW& w, const double* p, int i) {
  double y = 0.0;
  for (int j = 0; j < RN_N; j++) y += p[j] * w.M[(size_t)(i * RN_N + j) * w.ld];
  return y;
}
#endif

// OR over the chain's RN_G threads (red: RN_WPC_K doubles of the group's reduction scratch)
RN_DEVICE unsigned rn_group_or(unsigned x, double* red) {
  unsigned r = __reduce_or_sync(0xffffffffu, x);
#if RN_WPC_K > 1
  if ((threadIdx.x & 31) == 0) red[(threadIdx.x % RN_G) >> 5] = (double)r;
  RN_SYNC();
  r = 0;
  for (int k = 0; k < RN_WPC_K; k++) r |= (unsigned)red[k];
  RN_SYNC();
#else
  (void)red;
#endif
  return r;
}

RN_DEVICE void rn_ring_add(const RnArgs& A, int c, RnStats& S, int which, double value) {  // Stats.scala:24-30
  int i = S.ring_i[which] + 1;
  if (i == A.stats_window) S.ring_full[which] = 1;
  i = i % A.stats_window;
  S.ring_i[which] = i;
  if (RN_LANE == 0) RN_AT(A.st_rings, which * A.stats_window + i, c) = value;
}

// energy = potential + dot(velocity, p)/2, sequential order (LeapFrog.scala:134-139,205-231)
RN_DEVICE double rn_energy(const RnW& w, const double* p, double U) {
  double k = 0.0;
#if RN_MASS_MAX >= 2
  if (w.mass_kind == 2) {  // velocity rows across the lanes, then the dot product in every lane, in index order
    RN_SYNC();             // (w.v may still be read by the previous caller)
    RN_FOR_LANES(i) w.v[i] = rn_dense_row(w, p, i);
    RN_SYNC();
    for (int i = 0; i < RN_N; i++) k += (w.v[i] * p[i]);
    return U + k / 2.0;
  }
#endif
  if (w.mass_kind == 1) {
    for (int i = 0; i < RN_N; i++) k += ((p[i] * w.m[i]) * p[i]);
  } else {
    for (int i = 0; i < RN_N; i++) k += (p[i] * p[i]);
  }
  return U + k / 2.0;
}
RN_DEVICE double rn_log_accept(double deltaH) {  // LeapFrog.scala:141-145
  if (deltaH != deltaH) return -RN_INF;
  return rn_jmin0(-deltaH);
}
// One out-of-line instance of the emitted density per kernel: rn_update is reached from ~10 call sites (leapfrog inside
// HMC / EHMC count / EHMC sample / step-size search); inlining a 1000-parameter density at each of them costs minutes of
// NVRTC time and megabytes of SASS for nothing -- the row loop dominates, not the call.
__device__ __noinline__ void rn_update(const RnArgs& A, RnW& w, RnStats& S) {
  double dens;
  rn_density(w.q, dens, w.g, w.scr RN_DENSITY_RED(w.red), A.data, S.err, w.tma);
  w.U = dens * -1;
  S.grads += 1;
}
RN_DEVICE void rn_full_ps(RnW& w, double stepSize, RnStats& S) {  // LeapFrog.scala:168-176
  S.grads += 1;
  RN_SYNC();  // every thread of the group has finished reading p (energies, isUTurn) before anyone rewrites it
  RN_FOR_LANES(i) w.p[i] += stepSize * w.g[i];
  RN_SYNC();
}
RN_DEVICE void rn_new_qs(RnW& w, double stepSize) {  // LeapFrog.scala:147-154
#if RN_MASS_MAX >= 2
  if (w.mass_kind == 2) {
    RN_FOR_LANES(i) w.q[i] += (stepSize * rn_dense_row(w, w.p, i));
    RN_SYNC();
    return;
  }
#endif
  if (w.mass_kind == 1) {
    RN_FOR_LANES(i) w.q[i] += (stepSize * (w.p[i] * w.m[i]));
  } else {
    RN_FOR_LANES(i) w.q[i] += (stepSize * w.p[i]);
  }
  RN_SYNC();
}
RN_DEVICE void rn_leapfrog(const RnArgs& A, RnW& w, int l, double stepSize, RnStats& S) {  // :24-33,156-191
  rn_full_ps(w, stepSize / 2.0, S);
  rn_new_qs(w, stepSize);
  rn_update(A, w, S);
  for (int i = 1; i < l; i++) {
    rn_full_ps(w, stepSize, S);
    rn_new_qs(w, stepSize);
    rn_update(A, w, S);
  }
  rn_full_ps(w, stepSize / 2.0, S);
}
RN_DEVICE void rn_take_steps(const RnArgs& A, int c, RnW& w, int l, double stepSize, RnStats& S) {
  rn_ring_add(A, c, S, 0, stepSize);
  rn_leapfrog(A, w, l, stepSize, S);
  S.steps += l;
}
// momentum draw into dst (LeapFrog.scala:233-255): every lane draws the whole stream, lane i%32 keeps element i
RN_DEVICE void rn_initialize_ps(const RnW& w, RnRng& rng, double* dst) {
  for (int i = 0; i < RN_N; i++) {
    const double z = rn_normal(rng);
    if ((i % RN_G) == RN_LANE) dst[i] = (w.mass_kind == 1) ? z / sqrt(w.m[i]) : z;
  }
  RN_SYNC();
#if RN_MASS_MAX >= 2
  if (w.mass_kind == 2) {  // DenseMassMatrix.upperTriangularSolve (MassMatrix.scala:55-72), in place: dst holds z on entry
    if (RN_LANE == 0) {
      int i = RN_N - 1;
      int m = ((i + 1) * (i + 2)) / 2 - 1;
      while (i >= 0) {
        int j = RN_N - 1;
        double dot = 0.0;
        while (j > i) {
          dot += dst[j] * w.chol[(size_t)m * w.ld];
          j -= 1;
          m -= 1;
        }
        dst[i] = (dst[i] - dot) / w.chol[(size_t)m * w.ld];
        i -= 1;
        m -= 1;
      }
    }
    RN_SYNC();
  }
#endif
}

RN_DEVICE void rn_load_stats(const RnArgs& A, int c, RnStats& S) {
  S.grads = A.st_grads[c];
  S.steps = A.st_steps[c];
  S.iters = A.st_iters[c];
  S.accepted = A.st_accepted[c];
  S.err = A.st_err[c];
  S.e_mean = RN_AT(A.st_energy, 0, c);
  S.e_raw = RN_AT(A.st_energy, 1, c);
  S.trans2 = RN_AT(A.st_energy, 2, c);
  S.e_n = A.st_energy_n[c];
  for (int r = 0; r < 3; r++) {
    S.ring_i[r] = RN_AT(A.st_ring_i, r, c);
    S.ring_full[r] = RN_AT(A.st_ring_full, r, c);
  }
}
RN_DEVICE void rn_store_stats(const RnArgs& A, int c, const RnStats& S) {
  if (RN_LANE != 0) return;
  A.st_grads[c] = S.grads;
  A.st_steps[c] = S.steps;
  A.st_iters[c] = S.iters;
  A.st_accepted[c] = S.accepted;
  A.st_err[c] = S.err;
  RN_AT(A.st_energy, 0, c) = S.e_mean;
  RN_AT(A.st_energy, 1, c) = S.e_raw;
  RN_AT(A.st_energy, 2, c) = S.trans2;
  A.st_energy_n[c] = S.e_n;
  for (int r = 0; r < 3; r++) {
    RN_AT(A.st_ring_i, r, c) = S.ring_i[r];
    RN_AT(A.st_ring_full, r, c) = S.ring_full[r];
  }
}

#ifdef RN_HOST_EMULATION
static double rn_smem[1 << 16];  // one emulated CTA (= one chain) at a time
#else
extern __shared__ __align__(128) double rn_smem[];
#endif

// =============================================================================================================
RN_GLOBAL void rn_k_init(const RnArgs A) {
  const int c = (int)((blockIdx.x * blockDim.x + threadIdx.x) / RN_G);
  if (c >= A.chains) return;  // whole warp exits
  RnW w;
  rn_w_setup(w, rn_smem + (size_t)RN_GROUP * RN_WPC_SMEM_DOUBLES, RN_WPC_GSLICE(A.wpc_state, c));
  w.mass_kind = 0;
  RnRng rng;
  rng.seed = A.rng_seed[c];
  rng.nng = A.rng_nng[c];
  rng.have = A.rng_have[c];
  RnStats S;
  rn_load_stats(A, c, S);

  // LeapFrog.initialize, LeapFrog.scala:102-116
  for (int i = 0; i < RN_N; i++) {
    const double z = rn_normal(rng);
    if ((i % RN_G) == RN_LANE) {
      w.q[i] = z;
      w.p[i] = 0.0;
    }
  }
  RN_SYNC();
  rn_update(A, w, S);
  const double cU = w.U;
  RN_FOR_LANES(i) {
    RN_AT(A.params, RN_N + i, c) = w.q[i];
    RN_AT(A.grad, i, c) = w.g[i];
  }
  rn_initialize_ps(w, rng, w.p);
  RN_FOR_LANES(i) RN_AT(A.params, i, c) = w.p[i];
  if (RN_LANE == 0) RN_AT(A.params, 2 * RN_N, c) = cU;

  double stepSize;
  if (A.step_tuner == 0) {  // DualAvgTuner.findReasonableStepSize, DualAvg.scala:27-41
    const double H0 = rn_energy(w, w.p, cU);
    stepSize = 1.0;
    rn_leapfrog(A, w, 1, stepSize, S);  // tryStepping, LeapFrog.scala:14-22 (pqBuf == params here)
    double lap = rn_log_accept(rn_energy(w, w.p, w.U) - H0);
    const double exponent = (lap > -RN_LN2) ? 1.0 : -1.0;
    const double doubleOrHalf = (exponent > 0) ? 2.0 : 0.5;
#if RN_STEP_POOL
    int log2Step = 0;  // stepSize == 2^log2Step
#endif
    while (stepSize != 0.0 && (exponent * lap > -exponent * RN_LN2)) {
      stepSize *= doubleOrHalf;
#if RN_STEP_POOL
      log2Step += (exponent > 0) ? 1 : -1;
#endif
      RN_SYNC();
      RN_FOR_LANES(i) {  // copy(params, pqBuf)
        w.p[i] = RN_AT(A.params, i, c);
        w.q[i] = RN_AT(A.params, RN_N + i, c);
        w.g[i] = RN_AT(A.grad, i, c);
      }
      w.U = cU;
      RN_SYNC();
      rn_leapfrog(A, w, 1, stepSize, S);
      lap = rn_log_accept(rn_energy(w, w.p, w.U) - H0);
    }
    if (RN_LANE == 0) {
      rn_da_apply(stepSize, RN_AT(A.da, 1, c), RN_AT(A.da, 2, c), RN_AT(A.da, 3, c), RN_AT(A.da, 4, c), A.da_iter[c]);
#if RN_STEP_POOL
      // pooled: K and C over all chains, one lane per chain; rn_k_step_pool installs the shared DualAvg
      rn_pool_add_initial_step(A.step_acc, log2Step);
#endif
    }
  } else {
    stepSize = A.static_step;
  }
  if (RN_LANE == 0) {
    RN_AT(A.da, 0, c) = stepSize;
    A.rng_seed[c] = rng.seed;
    A.rng_nng[c] = rng.nng;
    A.rng_have[c] = rng.have;
  }
  rn_store_stats(A, c, S);
}

// =============================================================================================================
#define RN_K_WARMUP rn_k_iter  /* one entry point for both phases on this shape (rn_sampler.cuh has two) */
RN_GLOBAL void rn_k_iter(const RnArgs A) {
  const int c = A.chain_begin + (int)((blockIdx.x * blockDim.x + threadIdx.x) / RN_G);
#if RN_TMA_STAGES > 0
  const int slots = (int)(blockDim.x / RN_G);  // chains per CTA
  double* const stage0 = rn_smem + (((size_t)slots * RN_WPC_SMEM_DOUBLES + 15) & ~(size_t)15);
  unsigned long long* const bars = (unsigned long long*)(stage0 + (size_t)RN_TMA_STAGES * RN_TMA_TILE_DOUBLES);
  // HMC, and EHMC sampling with pooled trajectory lengths: every chain calls the density equally often
  const bool lockstep = (A.sampler == 0 || (RN_TRAJ_POOL && A.phase == 1)) && (A.tma != 0);
  if (lockstep) {
    if (threadIdx.x == 0) {
      // RN_TMA_STAGES barriers of the CTA-shared tile pipeline, or one per warp of the chain-batched DMMA path
      for (int s = 0; s < (RN_MMA_BARS > RN_TMA_STAGES ? RN_MMA_BARS : RN_TMA_STAGES); s++) rn_mbar_init(&bars[s], 1);
#ifndef RN_HOST_EMULATION
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
    }
    __syncthreads();
  }
#endif
  if (c >= A.chain_end) return;
  RnW w;
  rn_w_setup(w, rn_smem + (size_t)RN_GROUP * RN_WPC_SMEM_DOUBLES, RN_WPC_GSLICE(A.wpc_state, c));  // c: the absolute chain index
#if RN_TMA_STAGES > 0
  if (lockstep) {
    const int first = A.chain_begin + (int)(blockIdx.x * (blockDim.x / RN_G));
    const int active = (A.chain_end - first) < slots ? (A.chain_end - first) : slots;
    w.tma.on = 1;
    w.tma.stage = stage0;
    w.tma.full = bars;
    w.tma.nthreads = (unsigned)active * (unsigned)RN_G;
  }
#endif
  w.mass_kind = A.mass_kind;
  RnRng rng;
  rng.seed = A.rng_seed[c];
  rng.nng = A.rng_nng[c];
  rng.have = A.rng_have[c];
  RnStats S;
  rn_load_stats(A, c, S);
  if (w.mass_kind == 1) {
    RN_FOR_LANES(i) w.m[i] = RN_AT(A.mass, i, c);
    RN_SYNC();
  }
#if RN_MASS_MAX >= 2
  w.M = A.mass + c;
  w.chol = A.chol + c;
  w.ld = (size_t)A.chains;
#endif
  double stepSize = RN_AT(A.da, 0, c);
  double logStepSize = 0, logStepSizeBar = 0, avgError = 0, shrinkageTarget = 0;
  int daIter = 0;
  if (A.step_tuner == 0) {
    logStepSize = RN_AT(A.da, 1, c);
    logStepSizeBar = RN_AT(A.da, 2, c);
    avgError = RN_AT(A.da, 3, c);
    shrinkageTarget = RN_AT(A.da, 4, c);
    daIter = A.da_iter[c];
    if (A.phase == 1) stepSize = rn_exp(logStepSizeBar);
  }
  int win_size = A.win_size, win_i = A.win_i, win_j = A.win_j, est_samples = A.est_samples;
  int ring_i = 0, ring_full = 0;
  if (A.sampler == 1) {
    ring_i = A.ring_i[c];
    ring_full = A.ring_full[c];
  }

  for (int it = 0; it < A.n_iter; it++) {
    // ---- startIteration, LeapFrog.scala:52-59 ----
    RN_SYNC();
    RN_FOR_LANES(i) w.p[i] = RN_AT(A.params, i, c);
    RN_SYNC();
    const double cU = RN_AT(A.params, 2 * RN_N, c);
    const double prevH = rn_energy(w, w.p, cU);
    RN_SYNC();
    rn_initialize_ps(w, rng, w.p);
    RN_FOR_LANES(i) {
      RN_AT(A.params, i, c) = w.p[i];
      w.q[i] = RN_AT(A.params, RN_N + i, c);
      w.g[i] = RN_AT(A.grad, i, c);
    }
    w.U = cU;
    RN_SYNC();
    const double startH = rn_energy(w, w.p, cU);
    const rn_i64 iterationStartGrads = S.grads;
    const rn_i64 steps0 = S.steps;
    const double usedStep = stepSize;

    if (A.sampler == 0) {
      rn_take_steps(A, c, w, A.n_steps, stepSize, S);
    } else {  // EHMC.scala:15-61
      bool count = false;
      if (A.phase == 0) count = (!ring_full) || (rn_uniform(rng) < A.p_count);
      if (count) {
        double sU = 0.0;
        int l = 0;
        for (;;) {
          double out = 0.0;  // isUTurn(params): sequential order, params.q read back from global memory
          for (int i = 0; i < RN_N; i++) out += (w.q[i] - RN_AT(A.params, RN_N + i, c)) * w.p[i];
          const bool uturn = (out != out) ? true : (out < 0);
          if (uturn || !(l < A.max_steps)) break;
          l += 1;
          rn_take_steps(A, c, w, 1, stepSize, S);
          if (l == A.min_steps) {  // snapshot
            RN_FOR_LANES(i) {
              w.sq[i] = w.q[i];
              w.sp[i] = w.p[i];
              w.sg[i] = w.g[i];
            }
            sU = w.U;
            RN_SYNC();
          }
        }
        if (l < A.min_steps) {
          rn_take_steps(A, c, w, A.min_steps - l, stepSize, S);
        } else {  // restore
          RN_SYNC();  // the isUTurn sums above read q and p of every element
          RN_FOR_LANES(i) {
            w.q[i] = w.sq[i];
            w.p[i] = w.sp[i];
            w.g[i] = w.sg[i];
          }
          w.U = sU;
          RN_SYNC();
        }
        ring_i += 1;
        if (ring_i == A.buf_size) ring_full = 1;
        ring_i = ring_i % A.buf_size;
        if (RN_LANE == 0) RN_AT(A.ring, ring_i, c) = (double)l;
        RN_SYNC();
      }
#if RN_TRAJ_POOL
      else if (A.phase == 1) {  // pooled: the sampling iteration's shared length, no draw (rn_sampler_common.cuh)
        rn_take_steps(A, c, w, rn_traj_length(A, A.traj_t0 + it), stepSize, S);
      }
#endif
      else {
        const int idx = ring_full ? rn_rng_int(rng, A.buf_size) : rn_rng_int(rng, ring_i + 1);
        const int nsteps = rn_d2i(RN_AT(A.ring, idx, c));
        rn_take_steps(A, c, w, nsteps, stepSize, S);
      }
    }

    // ---- finishIteration, LeapFrog.scala:61-82 ----
    const double endH = rn_energy(w, w.p, w.U);
    const double deltaH = endH - startH;
    const double a = rn_log_accept(deltaH);
    const bool accept = a > rn_log(rn_uniform(rng));
    double eH;
    RN_SYNC();
    if (accept) {
      RN_FOR_LANES(i) {
        RN_AT(A.params, i, c) = w.p[i];
        RN_AT(A.params, RN_N + i, c) = w.q[i];
        RN_AT(A.grad, i, c) = w.g[i];
      }
      if (RN_LANE == 0) RN_AT(A.params, 2 * RN_N, c) = w.U;
      eH = endH;
      S.accepted += 1;
    } else {
      RN_FOR_LANES(i) w.q[i] = RN_AT(A.params, RN_N + i, c);
      eH = startH;
    }
    RN_SYNC();
    {
      S.e_n += 1;
      const double oldDiff = eH - S.e_mean;
      S.e_mean += (oldDiff / (double)S.e_n);
      const double newDiff = eH - S.e_mean;
      S.e_raw += oldDiff * newDiff;
      const double d = eH - prevH;
      S.trans2 += d * d;
    }
    S.iters += 1;
    rn_ring_add(A, c, S, 1, rn_exp(a));
    rn_ring_add(A, c, S, 2, (double)(S.grads - iterationStartGrads));
    if (A.trace && RN_LANE == 0) {
      double* tr = A.trace + (size_t)it * 4 * (size_t)A.chains;
      tr[0 * (size_t)A.chains + c] = a;
      tr[1 * (size_t)A.chains + c] = accept ? 1.0 : 0.0;
      tr[2 * (size_t)A.chains + c] = usedStep;
      tr[3 * (size_t)A.chains + c] = (double)(S.steps - steps0);
    }

    if (A.phase == 0) {
#if RN_STEP_POOL
      // pooled: one lane per chain adds the chain's share of the iteration's acceptance sum; rn_k_step_pool applies the update
      if (A.step_tuner == 0 && RN_LANE == 0) rn_pool_add(A.step_acc + it, rn_pool_quantise(rn_exp(a)));
#else
      if (A.step_tuner == 0)
        stepSize = rn_exp(rn_da_update(A, rn_exp(a), logStepSize, logStepSizeBar, avgError, shrinkageTarget, daIter));
#endif
#if RN_MASS_MAX >= 2
      if (A.mass_tuner == 2) {  // DenseMassMatrixTuner: WindowedMassMatrixTuner (MassMatrix.scala:147-164) over CovarianceEstimator
        win_j += 1;
#if RN_MASS_POOL
        // pooled extension: the chain's Welford mean and co-moment of the window (the count is the position in the window);
        // rn_k_pool_reduce / rn_k_pool_reduce_dense / rn_k_pool_factor / rn_k_pool_apply_dense do the window end
        if (RN_IN_WINDOW(A, win_j)) {
          win_i += 1;
          RN_SYNC();
          RN_FOR_LANES(i) {
            double mean = RN_AT(A.est_mean, i, c);
            const double od = w.q[i] - mean;
            mean += od / (double)win_i;
            RN_AT(A.est_mean, i, c) = mean;
            const double nd = w.q[i] - mean;
            RN_AT(A.est_raw, i, c) += od * nd;
            w.v[i] = od;
            w.v2[i] = nd;
          }
          RN_SYNC();
          for (int e = RN_LANE; e < RN_N * RN_N; e += RN_G)  // CovarianceEstimator.update, :28-41
            RN_AT(A.est_cov, e, c) += w.v2[e / RN_N] * w.v[e % RN_N];
          if (win_i == win_size) {
            win_i = 0;
            win_size = rn_d2i(win_size * A.win_expansion);
          }
          RN_SYNC();
        }
#else
        if (RN_IN_WINDOW(A, win_j)) {
          win_i += 1;
          est_samples += 1;
          RN_SYNC();
          RN_FOR_LANES(i) {  // the differences are kept for the outer product
            double oldDiff;
            const double newDiff = rn_variance_update(A, c, i, w.q[i], est_samples, oldDiff);
            w.v[i] = oldDiff;
            w.v2[i] = newDiff;
          }
          RN_SYNC();
          for (int e = RN_LANE; e < RN_N * RN_N; e += RN_G)  // CovarianceEstimator.update, :28-41
            RN_AT(A.est_cov, e, c) += w.v2[e / RN_N] * w.v[e % RN_N];
          if (win_i == win_size) {
            win_i = 0;
            win_size = rn_d2i(win_size * A.win_expansion);
            const double z = (double)(est_samples - 1);
            for (int e = RN_LANE; e < RN_N * RN_N; e += RN_G) {  // DenseMassMatrix(covariance()), :43-50
              const double v = RN_AT(A.est_cov, e, c) / z;
              if (v == 0.0) S.err |= 2;  // require(!elements.contains(0.0)), MassMatrix.scala:16
              RN_AT(A.mass, e, c) = v;
              RN_AT(A.est_cov, e, c) = 0.0;
            }
            RN_FOR_LANES(i) {  // reset(): mean/raw only, NOT samples (:60-67)
              RN_AT(A.est_mean, i, c) = 0.0;
              RN_AT(A.est_raw, i, c) = 0.0;
            }
            S.err |= (int)rn_group_or((unsigned)(S.err & 2), w.red);
            RN_SYNC();
#ifndef RN_HOST_EMULATION
            __threadfence_block();  // the matrix written lane-strided above is read by lane 0 below
#endif
            if (RN_LANE == 0) {  // choleskyUpperTriangular (MassMatrix.scala:76-117); `lower` borrows the estimator's
              double* lower = A.est_cov + c;  // covariance block, which was just reset and is zeroed again below
              const size_t ld = (size_t)A.chains;
              rn_cholesky_upper(A, c, lower, ld);
              for (int e = 0; e < (RN_N * (RN_N + 1)) / 2; e++) lower[(size_t)e * ld] = 0.0;
            }
#ifndef RN_HOST_EMULATION
            __threadfence_block();
#endif
            RN_SYNC();
            w.mass_kind = 2;
            if (A.step_tuner == 0 && !RN_STEP_POOL)  // stepSizeTuner.reset() (pooled: rn_k_step_pool)
              stepSize = rn_da_reset(logStepSize, logStepSizeBar, avgError, shrinkageTarget, daIter);
          }
          RN_SYNC();
        }
#endif  // RN_MASS_POOL
      }
#endif
      if (A.mass_tuner == 1) {  // DiagonalMassMatrixTuner, MassMatrix.scala:147-164
        win_j += 1;
        if (A.adaptation == 1) {  // pooled extension: per-chain Welford statistics of the window (see rn_k_pool_reduce / rn_k_pool_apply)
          if (RN_IN_WINDOW(A, win_j)) {
            win_i += 1;
            // the chain's Welford mean / M2 over this window (combined over chains at the window end).  Not rn_variance_update:
            // the second difference re-reads q after the store of the mean, which that helper does not do.
            RN_FOR_LANES(i) {
              double mean = RN_AT(A.est_mean, i, c);
              const double od = w.q[i] - mean;
              mean += od / (double)win_i;
              RN_AT(A.est_mean, i, c) = mean;
              RN_AT(A.est_raw, i, c) += od * (w.q[i] - mean);
            }
            if (win_i == win_size) {
              win_i = 0;
              win_size = rn_d2i(win_size * A.win_expansion);
            }
          }
        } else if (RN_IN_WINDOW(A, win_j)) {
          win_i += 1;
          est_samples += 1;
          const bool window_end = (win_i == win_size);
          RN_FOR_LANES(i) {  // VarianceEstimator.update, MassMatrixEstimator.scala:69-83
            double mean = RN_AT(A.est_mean, i, c);
            const double oldDiff = w.q[i] - mean;
            mean += (oldDiff / (double)est_samples);
            const double newDiff = w.q[i] - mean;
            double raw = RN_AT(A.est_raw, i, c) + oldDiff * newDiff;
            if (window_end) {
              const double var = raw / (double)est_samples;
              if (var == 0.0) S.err |= 2;
              w.m[i] = var;
              RN_AT(A.mass, i, c) = var;
              mean = 0.0;
              raw = 0.0;
            }
            RN_AT(A.est_mean, i, c) = mean;
            RN_AT(A.est_raw, i, c) = raw;
          }
          if (window_end) {
            S.err |= (int)rn_group_or((unsigned)(S.err & 2), w.red);
            win_i = 0;
            win_size = rn_d2i(win_size * A.win_expansion);
            w.mass_kind = 1;
            if (A.step_tuner == 0 && !RN_STEP_POOL)  // stepSizeTuner.reset() (pooled: rn_k_step_pool)
              stepSize = rn_da_reset(logStepSize, logStepSizeBar, avgError, shrinkageTarget, daIter);
          }
          RN_SYNC();
        }
      }
    } else if (A.samples) {
      double* out = A.samples + (size_t)it * RN_N * (size_t)A.chains;
      RN_FOR_LANES(i) out[(size_t)i * (size_t)A.chains + c] = w.q[i];
    }
  }

  if (RN_LANE == 0) {
    if (A.phase == 0) {
      RN_AT(A.da, 0, c) = stepSize;
      if (A.step_tuner == 0) {
        RN_AT(A.da, 1, c) = logStepSize;
        RN_AT(A.da, 2, c) = logStepSizeBar;
        RN_AT(A.da, 3, c) = avgError;
        RN_AT(A.da, 4, c) = shrinkageTarget;
        A.da_iter[c] = daIter;
      }
    }
    if (A.sampler == 1) {
      A.ring_i[c] = ring_i;
      A.ring_full[c] = ring_full;
    }
    A.rng_seed[c] = rng.seed;
    A.rng_nng[c] = rng.nng;
    A.rng_have[c] = rng.have;
  }
  rn_store_stats(A, c, S);
}

// =============================================================================================================
RN_GLOBAL void rn_k_density(const double* RN_RESTRICT qin, double* RN_RESTRICT out, const double* data, int* err,
                            int chains, double* wpc_state = nullptr) {  // (null: placement 0, or the host emulation)
  const int c = (int)((blockIdx.x * blockDim.x + threadIdx.x) / RN_G);
  if (c >= chains) return;
  RnW w;
  rn_w_setup(w, rn_smem + (size_t)RN_GROUP * RN_WPC_SMEM_DOUBLES, RN_WPC_GSLICE(wpc_state, c));
  RN_FOR_LANES(i) w.q[i] = qin[(size_t)i * chains + c];
  RN_SYNC();
  int e = 0;
  double dens;
  rn_density(w.q, dens, w.g, w.scr RN_DENSITY_RED(w.red), data, e, w.tma);
  RN_SYNC();
  if (RN_LANE == 0) out[c] = dens;
  RN_FOR_LANES(i) out[(size_t)(i + 1) * chains + c] = w.g[i];
  if (e && RN_LANE == 0) atomicOr(err, e);
}

#endif  // RN_SAMPLER_WPC_CUH

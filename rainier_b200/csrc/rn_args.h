// rn_args.h -- kernel argument block shared verbatim by the host runtime (rn_runtime.cpp) and the device code
// (embedded in front of rn_sampler_common.cuh).  Plain C: only int / long long / double / pointers.
#ifndef RN_ARGS_H
#define RN_ARGS_H
#ifndef RN_PRELUDE_CUH
typedef long long rn_i64;
#endif

struct RnArgs {
  int chains;  // number of chains == leading dimension of every SoA array
  int pad0;
  // ---- chain state, [field][chains] ----
  double* params;   // [2N+1]: p(0..N-1), q(N..2N-1), U   (LeapFrog.scala:118-126)
  double* grad;     // [N] gradient of log-density at params.q
  rn_i64* rng_seed;
  double* rng_nng;
  int* rng_have;
  double* da;       // [5]: stepSize, logStepSize, logStepSizeBar, avgError, shrinkageTarget
  int* da_iter;
  double* mass;     // diagonal: [N] variances; dense: [N*N]
  double* chol;     // dense: packed upper Cholesky factor [N(N+1)/2]
  double* est_mean; // [N]
  double* est_raw;  // [N]
  double* est_cov;  // [N*N] (dense tuner)
  double* ring;     // EHMC trajectory-length ring [buf_size]
  int* ring_i;
  int* ring_full;
  // ---- stats (Stats.scala) ----
  rn_i64* st_grads;
  rn_i64* st_steps;
  int* st_iters;
  int* st_accepted;
  int* st_err;
  double* st_energy;   // [3]: energyVariance.mean, energyVariance.raw, energyTransitions2
  int* st_energy_n;
  double* st_rings;    // [3][stats_window]: stepSizes, acceptanceRates, gradsPerIteration
  int* st_ring_i;      // [3]
  int* st_ring_full;   // [3]
  // ---- data / outputs ----
  const double* data;
  double* samples;     // [n_iter][N][chains] or NULL
  double* trace;       // [n_iter][4][chains] or NULL (test instrumentation)
  // ---- configuration (uniform over chains) ----
  int sampler, n_steps, max_steps, min_steps, buf_size, step_tuner;
  double p_count, delta, static_step;
  int mass_tuner, mass_kind;     // mass_kind: MassMatrix in force at the start of this launch (0 id, 1 diag, 2 dense)
  int win_size, win_i, win_j, total_warmup, skip_first, skip_last, est_samples;
  double win_expansion;
  int stats_window;
  int n_iter;                    // iterations in this launch
  int phase;                     // 0 warmup, 1 sampling
  int adaptation;                // 0 per chain (reference semantics), 1 pooled over chains/ranks (extension)
  int tma;                       // warp-per-chain kernels: CTA-shared TMA data tiles allowed (see rn_sampler_wpc.cuh)
  int chain_begin;               // rn_k_iter works on chains [chain_begin, chain_end): rn_sample pipelines chain blocks
  int chain_end;                 //   against the device->host copy of the previous block
  int pad1;
  // pooled step-size adaptation (RN_STEP_POOL modules only, rn_sampler_common.cuh): rn_k_init adds into step_acc[0] (sum of
  // the chains' log2 initial step sizes) and step_acc[1] (chains); a warmup launch of one iteration adds its quantised
  // acceptance probabilities into *step_acc (the slot of that iteration)
  rn_i64* step_acc;
};

// argument block of rn_k_eval (rn_function.cuh): batched evaluation of a compiled function, generic addressing
struct RnEvalArgs {
  const double* x;
  double* out;
  long long count;
  long long in_inner, in_outer, in_pstride, in_estride;
  long long out_inner, out_outer, out_pstride, out_estride;
  int* err;  // bit 0: a lookup index fell outside its table at some point
};

// argument block of rn_k_lbfgs (rn_optimizer.cuh): batched multi-start L-BFGS, one thread per start
struct RnOptArgs {
  const double* x0;   // [N][starts] or NULL (every start at 0: Optimizer.scala:7)
  double* x;          // [N][starts]
  double* f;          // [starts]  -density at x
  int* info;          // [starts]  0 converged | bit 0 evaluation cap | bit 1 "dginit" | bit 2 lookup error
  int* evals;         // [starts]  density evaluations used
  const double* data;
  double eps;         // Optimizer.scala:13
  int starts;
  int max_evals;
};

#endif

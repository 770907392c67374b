/*
 * rainier_cuda.h -- the C ABI of librainier_cuda.so: the drop-in boundary for Rainier's HMC hot path.
 *
 * Every entry point replaces one seam of the reference (paths relative to the stripe/rainier tree):
 *
 *   rn_model_create    <- Compiler.compileTargets(group): ir.DataFunction
 *                         rainier-compute/src/main/scala/com/stripe/rainier/compute/Compiler.scala:14-20
 *                         (bytecode emitter ir/CompiledFunction.scala:42-120 replaced by a CUDA source emitter)
 *   rn_density_batch   <- DensityFunction.update / density / gradient
 *                         rainier-sampler/src/main/scala/com/stripe/rainier/sampler/DensityFunction.scala:3-8
 *                         as implemented by Model.density(), rainier-core/.../core/Model.scala:38-50
 *   rn_sample          <- Model.sample(config, nChains) -> Driver.sample per chain
 *                         rainier-core/.../core/Model.scala:13-24, rainier-sampler/.../sampler/Driver.scala:7-46
 *   rn_config          <- SamplerConfig + the built-in Sampler / StepSizeTuner / MassMatrixTuner classes
 *                         rainier-sampler/.../sampler/Sampler.scala:3-62, HMC.scala:3, EHMC.scala:3-6,
 *                         DualAvg.scala:3, MassMatrix.scala:120-181
 *   rn_chain_stats     <- Stats  rainier-sampler/.../sampler/Stats.scala:3-17
 *   rn_emit_source     <- rainier-decompile (debug dump of the generated code), Decompiler.scala:8-26
 *
 * Conventions: plain pointers and sizes only; the caller owns every host buffer; a handle owns its device
 * memory, CUDA module and stream and is freed only by the matching destroy; no C++ exception crosses the
 * ABI; every function returns RN_OK (0) or a negative RN_E_* code and leaves a message retrievable with
 * rn_last_error() (thread-local).  NaN/inf are *values* and propagate exactly as in the reference
 * (LeapFrog.scala:43-46,138-142); only a lookup index outside its table -- a NullPointerException thrown from
 * generated code in the reference (ir/MethodGenerator.scala:164-167) -- is an error (RN_E_LOOKUP).
 * A handle is not thread-safe (one stream); distinct handles may be used from distinct threads -- handles derived from the
 * same model handle -- samplers, rn_sample / rn_sample_predict / rn_optimize calls, diagnostics -- share its kernel and scratch
 * caches and serialise on the model's internal lock where they touch them.
 *
 * The CPU oracle (oracle/, test infrastructure only) exports the same symbols with an `rno_` prefix so the
 * parity tests can diff the two call for call.
 */
#ifndef RAINIER_CUDA_H
#define RAINIER_CUDA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- error codes ------------------------------------------------------------------------------------ */
enum {
  RN_OK = 0,
  RN_E_INVALID = -1,   /* bad argument / malformed RIR */
  RN_E_CUDA = -2,      /* CUDA driver / runtime failure (includes "no device": there is no CPU fallback) */
  RN_E_COMPILE = -3,   /* NVRTC rejected the emitted source (message holds the log) */
  RN_E_LOOKUP = -4,    /* a LookupIR index fell outside [low, low+len) on some chain */
  RN_E_UNSUPPORTED = -5,
  RN_E_NCCL = -6
};

/* ---- sampler configuration (POD mirror of SamplerConfig and friends) --------------------------------- */
enum { RN_SAMPLER_HMC = 0, RN_SAMPLER_EHMC = 1 };                  /* HMCSampler / EHMCSampler */
enum { RN_STEP_DUAL_AVG = 0, RN_STEP_STATIC = 1 };                 /* DualAvgTuner / StaticStepSize */
enum { RN_MASS_IDENTITY = 0, RN_MASS_DIAGONAL = 1, RN_MASS_DENSE = 2, RN_MASS_STATIC = 3 };
                                      /* IdentityMassMatrixTuner / DiagonalMassMatrixTuner /
                                         DenseMassMatrixTuner / StaticMassMatrix */
enum { RN_MATRIX_IDENTITY = 0, RN_MATRIX_DIAGONAL = 1, RN_MATRIX_DENSE = 2 }; /* MassMatrix ADT, MassMatrix.scala:3-32 */
enum { RN_ADAPT_PER_CHAIN = 0, RN_ADAPT_POOLED = 1 };
enum { RN_MATH_PARITY = 0, RN_MATH_FAST = 1 };
enum { RN_GRAD_AUTO = 0, RN_GRAD_SYMBOLIC = 1, RN_GRAD_ADJOINT = 2 };
/* kernel shape: one thread per chain (data-free / small models: state in registers, exact sequential row order) or one
 * warp per chain (streamed data: rows across lanes, shuffle reduction).  AUTO picks by rows and parameter count. */
enum { RN_BACKEND_AUTO = 0, RN_BACKEND_THREAD = 1, RN_BACKEND_WARP = 2 };

/* java.util.Random state (48-bit LCG + cached second Gaussian), so that a chain can continue a stream the
 * host already drew from (the reference shares one RNG between data synthesis and sampling,
 * rainier-test/.../core/SBCModel.scala:31-39). */
typedef struct rn_rng_state {
  int64_t seed48;           /* scrambled internal state, < 2^48 */
  double next_gaussian;     /* nextNextGaussian */
  int32_t have_next;        /* haveNextNextGaussian */
  int32_t reserved;
} rn_rng_state;

typedef struct rn_config {
  int32_t struct_size;      /* sizeof(rn_config), for forward compatibility */

  /* SamplerConfig, Sampler.scala:3-11,17-27 */
  int32_t iterations;        /* default 1000 */
  int32_t warmup_iterations; /* default 1000 */
  int32_t stats_window;      /* default 100 */

  /* sampler(): HMCSampler(nSteps) HMC.scala:3 | EHMCSampler(maxSteps,minSteps,bufSize,pCount) EHMC.scala:3-6 */
  int32_t sampler;           /* RN_SAMPLER_* */
  int32_t n_steps;           /* HMC */
  int32_t max_steps;         /* EHMC, default 1024 (DefaultConfig) */
  int32_t min_steps;         /* EHMC, default 1 */
  int32_t buf_size;          /* EHMC, default 100 */
  int32_t backend;           /* RN_BACKEND_AUTO (default) | RN_BACKEND_THREAD | RN_BACKEND_WARP, see below */
  double p_count;            /* EHMC, default 0.1 */

  /* stepSizeTuner(): DualAvgTuner(delta) DualAvg.scala:3 | StaticStepSize(stepSize) Sampler.scala:36-40 */
  int32_t step_size_tuner;   /* RN_STEP_* */
  int32_t step_adaptation;   /* extension: RN_ADAPT_PER_CHAIN (parity with the reference, default) or RN_ADAPT_POOLED:
                                one DualAvg state shared by all chains (and, when a communicator is attached, all
                                ranks), started at 2^(mean log2 of the chains' findReasonableStepSize) and updated
                                every warmup iteration with the chains' mean acceptance probability (exact integer
                                sums, DESIGN.md §3.2).  Independent of `adaptation`; needs DualAvgTuner */
  double delta;              /* default 0.8 */
  double static_step_size;

  /* massMatrixTuner(): MassMatrix.scala:120-181, Sampler.scala:47-50 */
  int32_t mass_tuner;        /* RN_MASS_* */
  int32_t initial_window_size; /* default 50 */
  double window_expansion;   /* default 1.5 */
  int32_t skip_first;        /* default 50 */
  int32_t skip_last;         /* default 50 */
  int32_t static_matrix;     /* RN_MATRIX_* when mass_tuner == RN_MASS_STATIC */
  int32_t trajectory_adaptation; /* extension, EHMCSampler only: RN_ADAPT_PER_CHAIN (parity with the reference, default: every
                                sampling iteration of a chain draws its length from its own ring of U-turn counts) or
                                RN_ADAPT_POOLED: warmup is unchanged; at the first sampling launch the histogram h[0..max_steps]
                                (int64) counts, over every chain (and, with a communicator attached, every rank), the ring
                                entries steps.sample() chooses from -- indices [0, ring_full ? buf_size : ring_i + 1), so a
                                ring that never filled offers slot 0, whose value is 0 -- and sampling iteration t (0 = the
                                first after warmup) of EVERY chain takes L_t leapfrog steps:
                                  T = sum h;  c[l] = h[0] + ... + h[l];  F = the 64-bit fingerprint of the counts (the
                                  checkpoints' word hash, rn_trajectory_lengths_sequence);
                                  z = splitmix64(F + (t + 1) * 0x9E3779B97F4A7C15), the finaliser z ^= z >> 30,
                                  z *= 0xBF58476D1CE4E5B9, z ^= z >> 27, z *= 0x94D049BB133111EB, z ^= z >> 31 (mod 2^64);
                                  r = mulhi64(z, T);  L_t = min { l : c[l] > r }.
                                No chain's RNG is consumed.  The first rn_sampler_run after warmup is a collective when a
                                communicator is attached.  max_steps <= 65536 in this mode */
  const double* static_matrix_elements; /* n (diagonal) or n*n (dense) doubles, shared by all chains */

  /* extensions (not in the reference) */
  int32_t adaptation;        /* RN_ADAPT_PER_CHAIN (parity with the reference, default) or RN_ADAPT_POOLED:
                                mass-matrix windows pool Welford statistics over all chains (and, when a
                                communicator is attached, all ranks).  RN_MASS_DIAGONAL pools the variances,
                                RN_MASS_DENSE the covariances (one shared matrix, factored once per window);
                                other tuners are refused */
  int32_t math_mode;         /* RN_MATH_PARITY: no FMA contraction, the reference's operation order;
                                RN_MATH_FAST: FMA contraction allowed */
  int32_t gradient_mode;     /* RN_GRAD_AUTO: use the RIR's symbolic gradient outputs when present, else adjoint */
  int32_t launch_iterations; /* iterations per kernel launch (0 = library default) */
  const rn_rng_state* rng_states; /* optional [chains]; overrides seeds when non-NULL */
  double* stats_rings;       /* optional host buffer [chains][3][stats_window]: the stepSizes, acceptanceRates
                                and gradsPerIteration ring buffers in RingBuffer slot order (Stats.scala:19-59) */
  double* diagnostics;       /* optional host buffer [n][2]: Trace.diagnostics (rHat, effectiveSampleSize per parameter,
                                core/Trace.scala:11-21) reduced on the device over all chains and iterations of this
                                call; with `samples == NULL` nothing but these numbers crosses PCIe */
} rn_config;

/* Stats.scala:3-17, one per chain, sampling phase (the reference resets stats after warmup, Driver.scala:31) */
typedef struct rn_chain_stats {
  int64_t gradient_evaluations; /* the reference's accounting: 2l+1 per takeSteps(l) (LeapFrog.scala:194-200) */
  int64_t leapfrog_steps;       /* integrator steps taken (l per takeSteps(l)); the throughput numerator */
  int32_t iterations;
  int32_t divergences;          /* never written by the reference (Stats.scala:6); always 0 */
  int32_t accepted;             /* accepted proposals (diagnostic, not in the reference) */
  int32_t error_flags;          /* bit 0: lookup index out of range */
  double step_size;             /* stepSizeTuner.stepSize used for sampling (Driver.scala:37) */
  double energy_mean;           /* energyVariance.mean(0) */
  double energy_raw;            /* energyVariance.raw(0) */
  double energy_transitions2;   /* bfmi = energy_transitions2 / energy_raw */
  int32_t energy_samples;
  int32_t reserved;
  int32_t ring_pos[3];          /* RingBuffer.i of stepSizes / acceptanceRates / gradsPerIteration */
  int32_t ring_full[3];
  double step_sizes_mean;       /* RingBuffer.mean semantics (Stats.scala:47-58) */
  double acceptance_rates_mean;
  double grads_per_iteration_mean;
  rn_rng_state rng;             /* RNG state after the last iteration */
  double gradient_time_ns_mean;  /* gradientTimes.mean / iterationTimes.mean (Stats.scala:8-9), read by the notebook's   */
  double iteration_time_ns_mean; /* HTMLProgress.scala:57,65: device time of the sampling launches / this chain's gradient */
                                 /* evaluations, and / iterations of the batch (all chains advance together)              */
} rn_chain_stats;

typedef struct rn_model rn_model;
typedef struct rn_sampler rn_sampler;
typedef struct rn_comm rn_comm;

/* fills *cfg with the reference's DefaultConfig (Sampler.scala:17-27) */
void rn_config_default(rn_config* cfg);

/* ---- model ------------------------------------------------------------------------------------------- */
/* rir/len: container of rainier_rir.h.  cols[i] (i < n_cols) are the column placeholders' data in input
 * order (input index n_params + i), col_rows[i] their lengths; copied to the device.  device: CUDA ordinal. */
int rn_model_create(const void* rir, size_t len, const double* const* cols, const int64_t* col_rows,
                    int n_cols, int device, rn_model** out);
int rn_model_nvars(const rn_model* m);
/* Device-side inlining (replaces TargetGroup.inlinable + PartialEvaluator.inline, compute/Target.scala:136-207,
 * compute/PartialEvaluator.scala:86-97): rn_model_create folds every SEPARABLE streamed target of a primal container into a
 * data-free polynomial -- the row sums of its column-only monomials are reduced on the device once -- so the caller sends the
 * streamed form and never runs the reference's inliner (RN_INLINE=0 disables).  Returns the number of targets folded;
 * *monomials / *rows (optional) = monomials summed and rows no longer streamed per gradient evaluation. */
int rn_model_inlined(const rn_model* m, int64_t* monomials, int64_t* rows);
/* tooling / tests (no device): the host halves of that step.  rn_inline_plan: number of separable targets of a primal
 * container; for target k of them its index, the number of column-only monomials and the RIR_FLAG_FUNCTION container that
 * evaluates them over the target's columns.  rn_inline_apply: the rewritten container given the monomials' row sums. */
int rn_inline_plan(const void* rir, size_t len, int k, int* n_targets, int* target_index, int64_t* n_monomials, void* fn_rir, size_t cap,
                   size_t* needed);
int rn_inline_apply(const void* rir, size_t len, const double* sums, size_t n_sums, void* out, size_t cap, size_t* needed);
/* q: host [chains][n];  out: host [chains][n+1] = density then gradient (Model.scala:48-49) */
int rn_density_batch(rn_model* m, const double* q, int chains, double* out);
/* debug: emitted CUDA source of the fused kernel for `cfg` (NUL-terminated).  Returns RN_OK and the needed
 * size (incl. NUL) in *needed; copies at most cap bytes. */
int rn_emit_source(rn_model* m, const rn_config* cfg, char* buf, size_t cap, size_t* needed);
/* debug/test: host image of the device data buffer exactly as rn_model_create uploads it -- per streamed target a
 * tile-major block [tile][column][32 rows] (one tile = one contiguous chunk = one TMA bulk copy).  cols as in
 * rn_model_create; *needed receives the size in doubles; image may be NULL to query it. */
int rn_model_pack_columns(const rn_model* m, const double* const* cols, double* image, size_t cap_doubles, size_t* needed);
/* debug/analysis: where the frozen DAG "really is a dense mat-vec" -- maximal sums of parameter x column products in the
 * streamed row bodies (the Translator's fold of a `Line` with column coefficients, compute/Translator.scala:91-125).
 * out = [dot products per gradient evaluation (summed over rows), their multiply-adds per gradient, terms of the longest
 * dot, distinct dots in the emitted row bodies]. */
int rn_model_dot_structure(rn_model* m, const rn_config* cfg, double out[4]);
/* debug/analysis: which streamed targets are separable -- their row sum is sum_k S_k * p_k(parameters) with S_k a row sum of
 * products of column-only values, the shape the reference's inliner folds into constants on the JVM
 * (compute/Target.scala:136-207, compute/PartialEvaluator.scala:86-97).  out = [streamed targets, separable among them,
 * atoms S_k, rows no longer streamed per gradient evaluation].  Analysis only (DESIGN.md 5b-4). */
int rn_model_separable_structure(rn_model* m, double out[4]);
/* debug: the compiled cubin of the same kernel (for cuobjdump -sass). */
int rn_emit_cubin(rn_model* m, const rn_config* cfg, void* buf, size_t cap, size_t* needed);
void rn_model_destroy(rn_model* m);

/* ---- one-call sampling (the path Model.sample lowers to) ------------------------------------------------ */
/* seeds[c]: chain c behaves exactly like a single-chain reference run with ScalaRNG(seeds[c]).
 * samples: host [chains][iterations][n].  mass: host [chains][n] (diagonal/identity: variances, identity = 1)
 * or [chains][n*n] (dense), may be NULL.  stats: host [chains], may be NULL. */
int rn_sample(rn_model* m, const rn_config* cfg, const int64_t* seeds, int chains, double* samples,
              double* mass, rn_chain_stats* stats);

/* ---- page-locked host buffers (optional) ----------------------------------------------------------------- */
/* The result of rn_sample is chains*iterations*n doubles -- at the headline size 1.08 GB per call -- so the
 * device->host copy dominates the call.  When `samples` points into page-locked memory the DMA engine writes it
 * directly; a pageable buffer is filled through a pinned staging ring plus host memcpy threads (about half the rate).
 * rn_host_alloc returns page-locked memory (the JVM side wraps it with NewDirectByteBuffer, see INTEGRATION.md);
 * rn_host_register page-locks a buffer the caller already owns (e.g. a long-lived direct ByteBuffer). */
int rn_host_alloc(int device, size_t bytes, void** out);
int rn_host_free(int device, void* p);
int rn_host_register(int device, void* p, size_t bytes);
int rn_host_unregister(int device, void* p);

/* ---- staged / device-resident sampling (what rn_sample is built from) ----------------------------------- */
int rn_sampler_create(rn_model* m, const rn_config* cfg, const int64_t* seeds, int chains, rn_sampler** out);
/* LeapFrog.initialize + Driver.warmup (Driver.scala:22,48-90) for `iterations` more warmup iterations
 * (first call also initializes); call until cfg->warmup_iterations are consumed or pass -1 for "all". */
int rn_sampler_warmup(rn_sampler* s, int iterations);
/* Driver.collectSamples (Driver.scala:92-119): `iterations` sampling iterations.  d_samples: device pointer
 * to [iterations][n][chains] doubles (chain fastest: coalesced), or NULL to discard samples. */
int rn_sampler_run(rn_sampler* s, int iterations, double* d_samples);
/* blocks until all queued work is done */
int rn_sampler_sync(rn_sampler* s);
/* current q of every chain -> host [chains][n] */
int rn_sampler_positions(rn_sampler* s, double* q);
int rn_sampler_stats(rn_sampler* s, rn_chain_stats* stats, double* mass, double* stats_rings);
/* Trace.diagnostics (rainier-core/.../core/Trace.scala:11-21,49-121): rHat and effective sample size per parameter
 * over a DEVICE-resident sample block, reduced on the device (only n*2 numbers cross PCIe).  layout 0 =
 * [iterations][n][chains] (as rn_sampler_run writes it), 1 = [chains][iterations][n].  out: host [n][2]. */
int rn_sampler_diagnostics(rn_sampler* s, const double* d_samples, int iterations, int layout, double* out);
/* Trace.thin(thin).diagnostics over every sampling iteration rn_sampler_run performs after this call, accumulated on
 * the device as the draws are produced: no sample block is kept, and rn_sampler_run may be given d_samples == NULL.
 * Warmup draws are never tracked.  Calling it again restarts the accumulation.  thin >= 1.
 * Kept draws are those whose index among the tracked draws is a multiple of thin (index 0: the first draw after this
 * call), whatever the split into rn_sampler_run calls; any split gives bit-identical results.
 * Device memory, independent of the number of iterations: the state, 201 doubles per (parameter, chain), and the finish's
 * scratch, 8 doubles per (parameter, chain), both allocated by the first call and freed by rn_sampler_destroy.  With
 * d_samples == NULL, rn_sampler_run also keeps a scratch of one launch's draws, launch_iterations * n * chains doubles
 * (cfg->launch_iterations, 0 = 1000): lower launch_iterations to bound it.  The accumulation launches are not counted by
 * rn_sampler_launches and their time is not in rn_chain_stats' time fields. */
int rn_sampler_track_diagnostics(rn_sampler* s, int thin);
/* out: host [n][2] = rHat, effectiveSampleSize over the tracked draws of every chain.  With a communicator attached this
 * covers every chain of every rank and is a collective: every rank calls it, and every rank gets the same numbers or
 * the same error code.  RN_E_INVALID: called before rn_sampler_track_diagnostics (on any rank), fewer than 2 chains in
 * total, fewer than 2 kept draws, or kept counts that differ between ranks.  Its two all-reduces are not counted by
 * rn_sampler_comm_stats. */
int rn_sampler_tracked_diagnostics(rn_sampler* s, double* out);
/* the CUstream the sampler launches on (for CUDA-event timing by the caller) */
void* rn_sampler_stream(rn_sampler* s);
/* number of kernel launches issued so far on this sampler */
int64_t rn_sampler_launches(const rn_sampler* s);
/* attach a communicator: pooled adaptation all-reduces over its ranks */
int rn_sampler_set_comm(rn_sampler* s, rn_comm* comm);
/* the collective of this path: ncclAllReduce calls issued by the pooled warmup so far and their summed device time in
 * microseconds (event pairs on the sampler's stream; synchronises it) */
int rn_sampler_comm_stats(rn_sampler* s, int64_t* calls, double* total_us);
/* pooled trajectory lengths (rn_config.trajectory_adaptation == RN_ADAPT_POOLED): the pooled histogram h[0..max_steps] over
 * every chain of every rank.  *n = max_steps + 1; counts (may be NULL) receives min(cap, *n) of them.  RN_E_INVALID in
 * per-chain mode and before the first sampling launch has built the histogram. */
int rn_sampler_trajectory_lengths(rn_sampler* s, int64_t* counts, int cap, int* n);
/* tooling / tests (no device): L_t of rn_config.trajectory_adaptation for t = t0 .. t0 + count - 1 given the histogram
 * counts[0..bins) (bins <= 65537, every count >= 0, a positive total) */
int rn_trajectory_lengths_sequence(const int64_t* counts, int bins, int64_t t0, int64_t count, int32_t* out);
void rn_sampler_destroy(rn_sampler* s);

/* ---- checkpoints of a staged sampler (byte format: rainier_ckpt.h; DESIGN.md 3.6) --------------------------------- */
/* Between API calls a chain's whole state is on the device: a checkpoint copies it out, and a restore in a fresh handle --
 * another process, another device -- continues with the same bits as the uninterrupted run (any split of a run into
 * rn_sampler_warmup / rn_sampler_run calls already gives the same bits, DESIGN.md 3.2).
 * rn_sampler_save: at any API boundary after rn_sampler_create (before the first warmup call, mid-warmup, mid-sampling);
 * synchronises the sampler's stream.  buf == NULL: only *needed.  A page-locked buf (rn_host_alloc / rn_host_register)
 * is written by DMA, a pageable one through the pinned staging ring of rn_sample's drain.  Device staging is bounded
 * (two buffers of at most 128 MB).
 * rn_sampler_restore: a new sampler whose chains are the blobs' chains, concatenated in order, with kernels built as
 * rn_sampler_create builds them for `cfg`.  RN_E_INVALID, naming the first differing item, when: a blob is truncated,
 * corrupted (checksum) or of another version; the model (fingerprint of its RIR and data) or n differs; a semantic
 * config field differs (sampler and its parameters, the tuners and their parameters, adaptation, step_adaptation,
 * trajectory_adaptation, math_mode, gradient_mode, stats_window, and warmup_iterations while warmup is unfinished); the resolved kernel shape
 * differs (the warp-per-chain placement may); several blobs disagree, or are concatenated where chains are not independent
 * (pooled adaptation before the end of warmup).  iterations, launch_iterations and the device may differ.
 * rn_checkpoint_info / rn_checkpoint_slice need no device.  A slice is chains [begin, end) as a blob of its own; refused
 * where chains are not independent, as above. */
/* (a struct tag only: the name is also the function's) */
struct rn_checkpoint_info {
  int32_t version;
  int32_t phase;          /* 0 created, 1 warming up, 2 warmup finished, 3 sampling */
  int64_t n, chains, chain_offset;
  int32_t warmup_iterations, warm_done;
  int32_t win_size, win_i, win_j, est_samples;
  int32_t mass_kind, track;
  int32_t track_thin, reserved;
  int64_t track_seen, track_kept;
  int32_t backend, wpc_k, mma, wpc_place; /* resolved shape: backend 0 thread per chain, 1 warp per chain */
  uint64_t fingerprint;
  uint64_t header_bytes, table_bytes, replicated_bytes, record_bytes, records_bytes, total_bytes;
};
int rn_sampler_save(rn_sampler* s, void* buf, size_t cap, size_t* needed);
int rn_sampler_restore(rn_model* m, const rn_config* cfg, const void* const* blobs, const size_t* lens, int n_blobs, rn_sampler** out);
int rn_checkpoint_info(const void* blob, size_t len, struct rn_checkpoint_info* out);
int rn_checkpoint_slice(const void* blob, size_t len, int64_t begin, int64_t end, void* out, size_t cap, size_t* needed);

/* ---- multi-GPU plumbing (one process per GPU; chains are sharded by the caller) ------------------------- */
/* NCCL unique id exchange is the caller's job (e.g. torch.distributed broadcast of the 128 bytes). */
int rn_comm_unique_id(char id[128]);
int rn_comm_create(const char id[128], int rank, int world, int device, rn_comm** out);
void rn_comm_destroy(rn_comm* c);

/* ---- compiled functions: posterior-predictive "requirements" (SURVEY.md 8f-2) ------------------------------ */
/* rn_function_create   <- Compiler.compile(inputs: Seq[ir.Param], outputs: Seq[(String, Real)]): ir.CompiledFunction
 *                         rainier-compute/.../compute/Compiler.scala:22-30, as called by Generator.prepare
 *                         (rainier-core/.../core/Generator.scala:59-94) for Trace.predict (core/Trace.scala:34-41)
 * rn_function_eval*    <- the `0.until(cf.numOutputs).foreach(i => reqValues(i) = CompiledFunction.output(cf, array,
 *                         globalBuf, i))` loop of Generator.scala:80-84 (ir/CompiledFunction.scala:122-140), for ALL
 *                         posterior draws in one launch instead of once per draw
 * rir: a RIR_FLAG_FUNCTION container (rainier_rir.h): n inputs (the model's parameters), m outputs (the generator's
 * requirements, at most Generator.MaxRequirements = 500).  math_mode: RN_MATH_PARITY | RN_MATH_FAST.  device -1:
 * emit/compile only.  The Scala side keeps Generator.get (the RNG-consuming closure) and feeds it the values. */
typedef struct rn_function rn_function;
enum { RN_LAYOUT_SAMPLER = 0, RN_LAYOUT_ROWS = 1 };
int rn_function_create(const void* rir, size_t len, int device, int math_mode, rn_function** out);
int rn_function_ninputs(const rn_function* f);
int rn_function_noutputs(const rn_function* f);
/* host buffers: x [count][n] -> out [count][m]; blocking.  RN_E_LOOKUP when a lookup index left its table. */
int rn_function_eval(rn_function* f, const double* x, int64_t count, double* out);
/* device-resident draws, asynchronous on `stream` (NULL: the function's own stream, rn_function_stream):
 *   RN_LAYOUT_SAMPLER: d_x [iterations][n][chains] exactly as rn_sampler_run wrote it -> d_out [chains][iterations][m]
 *                      (the order of Trace.predict: chains.flatMap(_.map(fn)))
 *   RN_LAYOUT_ROWS   : d_x [iterations*chains][n] -> d_out [iterations*chains][m]
 * rn_function_sync waits for the function's own stream and reports lookup errors of the evaluations since the last sync. */
int rn_function_eval_device(rn_function* f, const double* d_x, int layout, int64_t iterations, int64_t chains, double* d_out,
                            void* stream);
int rn_function_sync(rn_function* f);
void* rn_function_stream(rn_function* f);
int64_t rn_function_launches(const rn_function* f);
/* debug: emitted CUDA source / compiled cubin (as rn_emit_source / rn_emit_cubin); static fp64 op counts of one point:
 * out = [adds+multiplies+compares, transcendental and division-class calls] */
int rn_function_emit_source(rn_function* f, char* buf, size_t cap, size_t* needed);
int rn_function_emit_cubin(rn_function* f, void* buf, size_t cap, size_t* needed);
int rn_function_op_counts(const rn_function* f, double out[2]);
void rn_function_destroy(rn_function* f);
/* rn_sample_predict   <- object Model.sample(t, config): List[U] = model.sample(config).predict(gen)
 *                         (rainier-core/.../core/Model.scala:56-63): sampling and the requirement values of predict in one
 * call; the draws stay on the device and only chains*iterations*m doubles come back.  f: the generator's requirements over
 * the model's parameters.  predictions: host [chains][iterations][m] (Trace.predict's order).  mass, stats, cfg->diagnostics,
 * cfg->stats_rings as in rn_sample. */
int rn_sample_predict(rn_model* m, const rn_config* cfg, rn_function* f, const int64_t* seeds, int chains, double* predictions,
                      double* mass, rn_chain_stats* stats);

/* ---- posterior-predictive draws: the Generator.get half of Trace.predict ------------------------------------ */
/* rn_generator_*       <- `chains.flatMap(_.map(fn))` of Trace.predict (rainier-core/.../core/Trace.scala:34-41) with
 *                         fn = Generator.prepare's closure (core/Generator.scala:59-94): for every posterior draw the
 *                         generator's requirement values AND its RNG-consuming Generator.get, on the device, for the
 *                         built-in distributions (Continuous.scala, Discrete.scala), Real values, tuples, Seq/Vec and
 *                         repeat(k) with a constant k.
 * rir: a RIR_FLAG_FUNCTION | RIR_FLAG_GENERATOR container (rainier_rir.h): n inputs (the model's parameters), the slots as
 * the function's outputs, the plan; m_out doubles per draw (rn_generator_noutputs), discrete values as Java Longs stored as
 * doubles.  device -1: emit/compile only.  Always parity math.
 * Stream rule: chain c owns rng_states[c] and draws its iterations in order, exactly as the reference's predict over a Trace
 * holding chain c alone with an RNG in that state; the state after the last draw is written back.  Any split of the
 * iterations into calls gives the same bits.
 * Bounded work: every draw of a built-in distribution may make at most 2^24 RNG calls (rn_generate.cuh: RN_GEN_BUDGET), and a
 * plan at most 2^26 ops per draw (checked at create).  A chain whose draw would exceed the budget stops: that iteration and
 * all its later ones in the call are NaN, its state is where the failed draw stopped, and the call returns RN_E_INVALID
 * naming the first such chain and its iteration (outputs and states are still written; the other chains' draws are
 * unaffected).  RN_E_LOOKUP as rn_function_eval. */
typedef struct rn_generator rn_generator;
int rn_generator_create(const void* rir, size_t len, int device, rn_generator** out);
int rn_generator_ninputs(const rn_generator* g);
int rn_generator_noutputs(const rn_generator* g);
int rn_generator_nslots(const rn_generator* g);
/* host buffers, blocking: x [chains][iterations][n] -> out [chains][iterations][m_out]; rng_states [chains] in/out */
int rn_generator_eval(rn_generator* g, const double* x, int64_t iterations, int64_t chains, rn_rng_state* rng_states, double* out);
/* device-resident draws on `stream` (NULL: the generator's own stream), blocking; rng_states: host [chains] in/out
 *   RN_LAYOUT_SAMPLER: d_x [iterations][n][chains] as rn_sampler_run wrote it
 *   RN_LAYOUT_ROWS   : d_x [chains][iterations][n]
 * d_out: [chains][iterations][m_out] (Trace.predict's order) */
int rn_generator_eval_device(rn_generator* g, const double* d_x, int layout, int64_t iterations, int64_t chains,
                             rn_rng_state* rng_states, double* d_out, void* stream);
/* tooling / tests (no device): the error report of a call from rn_k_generate's per-chain error bits (bit 0: a draw exceeded
 * the budget) and first failing iterations -- RN_OK, or RN_E_INVALID naming the first failing chain and its iteration */
int rn_generator_report(const int32_t* err, const int64_t* err_iter, int64_t chains);
/* iterations per chunk of the slot scratch (0, the default: as many as fit in 256 MB); results do not depend on it */
int rn_generator_set_chunk(rn_generator* g, int64_t iterations);
int rn_generator_emit_source(rn_generator* g, char* buf, size_t cap, size_t* needed);
int rn_generator_emit_cubin(rn_generator* g, void* buf, size_t cap, size_t* needed);
void rn_generator_destroy(rn_generator* g);
/* rn_sample_generate   <- model.sample(config).predict(gen) (core/Model.scala:56-63) with the draws of `gen` on the device:
 * sampling, the slots and the predictive draws in one call; the posterior draws never leave the device.  Chain c's
 * generator stream starts where its sampling stream ended (the rng of rn_sampler_stats); stats[c].rng is the state after
 * the predictive draws.  out: host [chains][iterations][m_out].  mass, stats, cfg->diagnostics, cfg->stats_rings as in
 * rn_sample. */
int rn_sample_generate(rn_model* m, const rn_config* cfg, rn_generator* g, const int64_t* seeds, int chains, double* out,
                       double* mass, rn_chain_stats* stats);

/* ---- MAP optimisation: batched multi-start L-BFGS (SURVEY.md 8f-4) ------------------------------------------ */
/* rn_optimize          <- Optimizer.lbfgs(df: DensityFunction): Array[Double]
 *                         rainier-sampler/.../optimizer/Optimizer.scala:6-24 driving class LBFGS
 *                         (rainier-sampler/.../optimizer/LBFGS.java:42-190, mcsrch :240-383, mcstep :431-605),
 *                         the body of Model.optimize (rainier-core/.../core/Model.scala:26-30)
 * The reference optimises from the single start x = 0.  Here every start of a batch is one GPU thread that runs the whole
 * optimisation (density + gradient + line search + history) inside one kernel; start c with x0 = NULL (or a zero row) is
 * bit-identical to the reference's run (thread-per-start shape: n*(2*history+4) <= 4096 doubles per start).  Streamed models
 * and large n use one warp per start (rows across lanes, L-BFGS history in shared memory). */
typedef struct rn_optimize_config {
  int32_t struct_size;
  int32_t history;          /* m of new LBFGS(x, m, eps); Optimizer.scala:12 uses 5 */
  double eps;               /* terminate when ||g|| <= eps * max(1, ||x||); Optimizer.scala:13 uses 0.1 */
  int32_t max_evaluations;  /* per start; the reference loops without a cap -- a kernel needs one (default 10000) */
  int32_t math_mode;        /* RN_MATH_* */
  int32_t gradient_mode;    /* RN_GRAD_* */
  int32_t backend;          /* RN_BACKEND_AUTO | RN_BACKEND_THREAD (one thread per start: bit-identical to the reference's
                               run) | RN_BACKEND_WARP (one warp per start: streamed models, history in shared memory; sums in
                               tree order -> agreement to rounding) */
} rn_optimize_config;
void rn_optimize_config_default(rn_optimize_config* cfg);
/* x0: host [starts][n] or NULL (all starts at 0).  x: host [starts][n].  f: host [starts] = -density at x (what LBFGS
 * minimises), may be NULL.  info: host [starts], may be NULL: 0 converged, bit 0 evaluation cap reached, bit 1 the search
 * direction was not a descent direction (`throw new RuntimeException("dginit")`, LBFGS.java:253-254), bit 2 lookup index
 * out of range (then the call returns RN_E_LOOKUP).  evaluations: host [starts] density evaluations used, may be NULL. */
int rn_optimize(rn_model* m, const rn_optimize_config* cfg, const double* x0, int starts, double* x, double* f, int32_t* info,
                int32_t* evaluations);
int rn_optimize_emit_source(rn_model* m, const rn_optimize_config* cfg, char* buf, size_t cap, size_t* needed);
int rn_optimize_emit_cubin(rn_model* m, const rn_optimize_config* cfg, void* buf, size_t cap, size_t* needed);

const char* rn_last_error(void);
const char* rn_version(void);

#ifdef __cplusplus
}
#endif
#endif

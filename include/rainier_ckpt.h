/*
 * rainier_ckpt.h -- the byte format of a staged sampler's checkpoint (rn_sampler_save / rn_sampler_restore,
 * include/rainier_cuda.h; DESIGN.md 3.6).  Little-endian, no device pointers, versioned.  A blob is, in order:
 *
 *   1. rn_ckpt_header                                  (header_bytes)
 *   2. n_fields x rn_ckpt_field                        the record layout: fields in record order
 *   3. step_bytes: d_step, int64 [2 + warmup] with pooled step-size adaptation, else [1]; then
 *      pool_bytes: the pooled window buffer (doubles)   -- both shared by all chains, copied as they are; then
 *      reserved1 bytes: with pooled trajectory lengths (reserved0 = rn_config.trajectory_adaptation = RN_ADAPT_POOLED) the
 *      pooled histogram, int64 [max_steps + 1], once the first sampling launch has built it (0 bytes before, and always
 *      with per-chain lengths: such blobs are laid out exactly as without the extension)
 *   4. chains x record_bytes                           chain-major records: chain c's fields in table order, each its
 *                                                      elements back to back (8-byte fields first, then 4-byte ones,
 *                                                      padded to a multiple of 8 bytes)
 *   5. uint64 checksum of parts 1-4
 *
 * Because the records are chain-major, chains [b, e) are one contiguous byte range (rn_checkpoint_slice).
 */
#ifndef RAINIER_CKPT_H
#define RAINIER_CKPT_H

#include <stdint.h>

#define RN_CKPT_MAGIC "RNCKPT\0\1"
#define RN_CKPT_VERSION 1

/* field ids of the table; each is one array of the sampler's per-chain state (rn_args.h: RnArgs) */
enum {
  RN_CKPT_PARAMS = 1, /* [2n+1] p, q, U */
  RN_CKPT_GRAD,       /* [n] */
  RN_CKPT_RNG_SEED,   /* int64 */
  RN_CKPT_RNG_NNG,
  RN_CKPT_DA,         /* [5] DualAvg: stepSize, logStepSize, logStepSizeBar, avgError, shrinkageTarget */
  RN_CKPT_MASS,       /* [n] diagonal, [n*n] dense, [0] identity */
  RN_CKPT_CHOL,       /* [n(n+1)/2] dense */
  RN_CKPT_EST_MEAN,
  RN_CKPT_EST_RAW,
  RN_CKPT_EST_COV,
  RN_CKPT_RING,       /* [buf_size] EHMC trajectory lengths */
  RN_CKPT_ST_GRADS,   /* int64 */
  RN_CKPT_ST_STEPS,   /* int64 */
  RN_CKPT_ST_ENERGY,  /* [3] */
  RN_CKPT_ST_RINGS,   /* [3 * stats_window] */
  RN_CKPT_TRACK,      /* [201 * n] tracked diagnostics, element f * n + i (rn_diag.cuh) */
  RN_CKPT_RNG_HAVE,   /* int32 from here on */
  RN_CKPT_DA_ITER,
  RN_CKPT_RING_I,
  RN_CKPT_RING_FULL,
  RN_CKPT_ST_ERR,
  RN_CKPT_ST_ITERS,
  RN_CKPT_ST_ACCEPTED,
  RN_CKPT_ST_ENERGY_N,
  RN_CKPT_ST_RING_I,  /* [3] */
  RN_CKPT_ST_RING_FULL /* [3] */
};
enum { RN_CKPT_F64 = 0, RN_CKPT_I64 = 1, RN_CKPT_I32 = 2 };

typedef struct rn_ckpt_field {
  uint32_t id;   /* RN_CKPT_PARAMS .. */
  uint32_t type; /* RN_CKPT_F64 | RN_CKPT_I64 | RN_CKPT_I32 */
  uint64_t elems; /* per chain */
} rn_ckpt_field;

typedef struct rn_ckpt_header {
  char magic[8];
  uint32_t version;
  uint32_t header_bytes;
  uint64_t fingerprint; /* of the model: its RIR bytes and device data image */
  /* the semantic rn_config fields */
  int32_t sampler, n_steps, max_steps, min_steps, buf_size, step_size_tuner, step_adaptation, mass_tuner;
  double p_count, delta, static_step_size, window_expansion;
  int32_t initial_window_size, skip_first, skip_last, static_matrix, adaptation, math_mode, gradient_mode, stats_window,
      warmup_iterations, iterations;
  /* the resolved kernel shape (wpc_place is informational: a restore may use another placement) */
  int32_t backend, wpc_k, mma, mma_chains, wpc_place, mass_max, adjoint, fast, ehmc, step_pool, mass_pool,
          reserved0;  /* rn_config.trajectory_adaptation */
  int64_t n, chains, chain_offset; /* chain_offset: index of the first chain in the sampler that was saved */
  /* the sampler's host mirror */
  int32_t initialized, warm_done, stats_reset_for_sampling, win_size, win_i, win_j, est_samples, mass_kind;
  /* tracked diagnostics (rn_sampler_track_diagnostics) */
  int32_t track, track_thin;
  int64_t track_seen, track_kept;
  /* accumulated device times */
  double sampling_ms, track_ms;
  int64_t sampling_iterations;
  uint32_t n_fields, reserved1;  /* reserved1: bytes of the pooled trajectory-length histogram (part 3) */
  uint64_t step_bytes, pool_bytes, record_bytes;
} rn_ckpt_header;

#endif

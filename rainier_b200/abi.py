"""
ctypes mirror of include/rainier_cuda.h (the C ABI of librainier_cuda.so).  Field order and types must match
the header exactly; tests/test_abi.py checks sizeof() against the library's own rn_abi_sizes().
"""
import ctypes as C

RN_OK = 0
RN_E_INVALID, RN_E_CUDA, RN_E_COMPILE, RN_E_LOOKUP, RN_E_UNSUPPORTED, RN_E_NCCL = -1, -2, -3, -4, -5, -6

RN_SAMPLER_HMC, RN_SAMPLER_EHMC = 0, 1
RN_STEP_DUAL_AVG, RN_STEP_STATIC = 0, 1
RN_MASS_IDENTITY, RN_MASS_DIAGONAL, RN_MASS_DENSE, RN_MASS_STATIC = 0, 1, 2, 3
RN_MATRIX_IDENTITY, RN_MATRIX_DIAGONAL, RN_MATRIX_DENSE = 0, 1, 2
RN_ADAPT_PER_CHAIN, RN_ADAPT_POOLED = 0, 1
RN_MATH_PARITY, RN_MATH_FAST = 0, 1
RN_GRAD_AUTO, RN_GRAD_SYMBOLIC, RN_GRAD_ADJOINT = 0, 1, 2
RN_BACKEND_AUTO, RN_BACKEND_THREAD, RN_BACKEND_WARP = 0, 1, 2
RN_LAYOUT_SAMPLER, RN_LAYOUT_ROWS = 0, 1


class RngState(C.Structure):
    _fields_ = [("seed48", C.c_int64), ("next_gaussian", C.c_double), ("have_next", C.c_int32), ("reserved", C.c_int32)]


class Config(C.Structure):
    _fields_ = [
        ("struct_size", C.c_int32),
        ("iterations", C.c_int32),
        ("warmup_iterations", C.c_int32),
        ("stats_window", C.c_int32),
        ("sampler", C.c_int32),
        ("n_steps", C.c_int32),
        ("max_steps", C.c_int32),
        ("min_steps", C.c_int32),
        ("buf_size", C.c_int32),
        ("backend", C.c_int32),
        ("p_count", C.c_double),
        ("step_size_tuner", C.c_int32),
        ("step_adaptation", C.c_int32),
        ("delta", C.c_double),
        ("static_step_size", C.c_double),
        ("mass_tuner", C.c_int32),
        ("initial_window_size", C.c_int32),
        ("window_expansion", C.c_double),
        ("skip_first", C.c_int32),
        ("skip_last", C.c_int32),
        ("static_matrix", C.c_int32),
        ("trajectory_adaptation", C.c_int32),
        ("static_matrix_elements", C.POINTER(C.c_double)),
        ("adaptation", C.c_int32),
        ("math_mode", C.c_int32),
        ("gradient_mode", C.c_int32),
        ("launch_iterations", C.c_int32),
        ("rng_states", C.POINTER(RngState)),
        ("stats_rings", C.POINTER(C.c_double)),
        ("diagnostics", C.POINTER(C.c_double)),
    ]


class ChainStats(C.Structure):
    _fields_ = [
        ("gradient_evaluations", C.c_int64),
        ("leapfrog_steps", C.c_int64),
        ("iterations", C.c_int32),
        ("divergences", C.c_int32),
        ("accepted", C.c_int32),
        ("error_flags", C.c_int32),
        ("step_size", C.c_double),
        ("energy_mean", C.c_double),
        ("energy_raw", C.c_double),
        ("energy_transitions2", C.c_double),
        ("energy_samples", C.c_int32),
        ("reserved", C.c_int32),
        ("ring_pos", C.c_int32 * 3),
        ("ring_full", C.c_int32 * 3),
        ("step_sizes_mean", C.c_double),
        ("acceptance_rates_mean", C.c_double),
        ("grads_per_iteration_mean", C.c_double),
        ("rng", RngState),
        ("gradient_time_ns_mean", C.c_double),
        ("iteration_time_ns_mean", C.c_double),
    ]


class OptimizeConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("history", C.c_int32), ("eps", C.c_double), ("max_evaluations", C.c_int32),
                ("math_mode", C.c_int32), ("gradient_mode", C.c_int32), ("backend", C.c_int32)]


class CheckpointInfo(C.Structure):  # struct rn_checkpoint_info
    _fields_ = [("version", C.c_int32), ("phase", C.c_int32), ("n", C.c_int64), ("chains", C.c_int64), ("chain_offset", C.c_int64),
                ("warmup_iterations", C.c_int32), ("warm_done", C.c_int32), ("win_size", C.c_int32), ("win_i", C.c_int32),
                ("win_j", C.c_int32), ("est_samples", C.c_int32), ("mass_kind", C.c_int32), ("track", C.c_int32),
                ("track_thin", C.c_int32), ("reserved", C.c_int32), ("track_seen", C.c_int64), ("track_kept", C.c_int64),
                ("backend", C.c_int32), ("wpc_k", C.c_int32), ("mma", C.c_int32), ("wpc_place", C.c_int32),
                ("fingerprint", C.c_uint64), ("header_bytes", C.c_uint64), ("table_bytes", C.c_uint64),
                ("replicated_bytes", C.c_uint64), ("record_bytes", C.c_uint64), ("records_bytes", C.c_uint64),
                ("total_bytes", C.c_uint64)]


# the checkpoint byte format, include/rainier_ckpt.h
CKPT_MAGIC = b"RNCKPT\0\1"
CKPT_VERSION = 1
(CKPT_PARAMS, CKPT_GRAD, CKPT_RNG_SEED, CKPT_RNG_NNG, CKPT_DA, CKPT_MASS, CKPT_CHOL, CKPT_EST_MEAN, CKPT_EST_RAW, CKPT_EST_COV, CKPT_RING,
 CKPT_ST_GRADS, CKPT_ST_STEPS, CKPT_ST_ENERGY, CKPT_ST_RINGS, CKPT_TRACK, CKPT_RNG_HAVE, CKPT_DA_ITER, CKPT_RING_I, CKPT_RING_FULL,
 CKPT_ST_ERR, CKPT_ST_ITERS, CKPT_ST_ACCEPTED, CKPT_ST_ENERGY_N, CKPT_ST_RING_I, CKPT_ST_RING_FULL) = range(1, 27)
CKPT_F64, CKPT_I64, CKPT_I32 = 0, 1, 2


class CkptField(C.Structure):  # rn_ckpt_field
    _fields_ = [("id", C.c_uint32), ("type", C.c_uint32), ("elems", C.c_uint64)]


class CkptHeader(C.Structure):  # rn_ckpt_header
    _fields_ = [("magic", C.c_char * 8), ("version", C.c_uint32), ("header_bytes", C.c_uint32), ("fingerprint", C.c_uint64)] + \
        [(f, C.c_int32) for f in ("sampler", "n_steps", "max_steps", "min_steps", "buf_size", "step_size_tuner", "step_adaptation",
                                  "mass_tuner")] + \
        [(f, C.c_double) for f in ("p_count", "delta", "static_step_size", "window_expansion")] + \
        [(f, C.c_int32) for f in ("initial_window_size", "skip_first", "skip_last", "static_matrix", "adaptation", "math_mode",
                                  "gradient_mode", "stats_window", "warmup_iterations", "iterations", "backend", "wpc_k", "mma",
                                  "mma_chains", "wpc_place", "mass_max", "adjoint", "fast", "ehmc", "step_pool", "mass_pool",
                                  "reserved0")] + \
        [(f, C.c_int64) for f in ("n", "chains", "chain_offset")] + \
        [(f, C.c_int32) for f in ("initialized", "warm_done", "stats_reset_for_sampling", "win_size", "win_i", "win_j", "est_samples",
                                  "mass_kind", "track", "track_thin")] + \
        [("track_seen", C.c_int64), ("track_kept", C.c_int64), ("sampling_ms", C.c_double), ("track_ms", C.c_double),
         ("sampling_iterations", C.c_int64), ("n_fields", C.c_uint32), ("reserved1", C.c_uint32), ("step_bytes", C.c_uint64),
         ("pool_bytes", C.c_uint64), ("record_bytes", C.c_uint64)]

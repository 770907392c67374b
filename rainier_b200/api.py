"""
rainier_b200.api -- Python host side over the C ABI of librainier_cuda.so (include/rainier_cuda.h).

The reference's host side is Scala; no JVM toolchain exists in this image, so the same plugin surface is mirrored
here in Python with the reference's own names and argument meaning, so that tests and benchmarks read like the
reference's (rainier-sampler/src/main/scala/com/stripe/rainier/sampler/):

    SamplerConfig / DefaultConfig      Sampler.scala:3-27
    HMCSampler(nSteps)                 HMC.scala:3          HMC(warmIt, it, nSteps)            HMC.scala:26-33
    EHMCSampler(maxSteps, minSteps, bufSize, pCount)        EHMC.scala:3-6 ; EHMC(...)          EHMC.scala:64-73
    DualAvgTuner(delta), StaticStepSize(stepSize)           DualAvg.scala:3, Sampler.scala:36-40
    IdentityMassMatrixTuner, DiagonalMassMatrixTuner, DenseMassMatrixTuner, StaticMassMatrix
                                       MassMatrix.scala:120-181, Sampler.scala:47-50
    IdentityMassMatrix / DiagonalMassMatrix / DenseMassMatrix   MassMatrix.scala:3-32
    CudaModel.sample(config, nChains)  <- Model.sample (rainier-core/.../core/Model.scala:13-24)
    CudaModel.density()                <- Model.density(): DensityFunction (Model.scala:38-50)

Python is plumbing only: every number is produced by the CUDA path.  There is no CPU fallback -- when the
library or a GPU is missing the calls raise RainierCudaError.
"""
import ctypes as C
import os

import numpy as np

from . import abi
from .abi import ChainStats, Config, RngState

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class RainierCudaError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("rainier_cuda error %d: %s" % (code, msg))
        self.code = code


def lib():
    """Loads rainier_b200/librainier_cuda.so (built in-tree by __graft_entry__.build / csrc/Makefile)."""
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "librainier_cuda.so")
        if not os.path.exists(path):
            raise RainierCudaError(abi.RN_E_CUDA, "librainier_cuda.so is not built (run __graft_entry__.build()); "
                                   "there is no CPU fallback")
        L = C.CDLL(path)
        L.rn_last_error.restype = C.c_char_p
        L.rn_version.restype = C.c_char_p
        L.rn_config_default.argtypes = [C.POINTER(Config)]
        L.rn_abi_sizes.argtypes = [C.POINTER(C.c_int32)]
        L.rn_model_create.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int,
                                      C.c_int, C.POINTER(C.c_void_p)]
        L.rn_model_nvars.argtypes = [C.c_void_p]
        L.rn_model_pack_columns.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_model_destroy.argtypes = [C.c_void_p]
        L.rn_model_op_counts.argtypes = [C.c_void_p, C.POINTER(Config), C.POINTER(C.c_double)]
        L.rn_model_separable_structure.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        L.rn_model_dot_structure.argtypes = [C.c_void_p, C.POINTER(Config), C.POINTER(C.c_double)]
        L.rn_model_inlined.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.rn_inline_plan.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64), C.c_void_p,
                                     C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_inline_apply.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_density_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.rn_emit_source.argtypes = [C.c_void_p, C.POINTER(Config), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_emit_cubin.argtypes = [C.c_void_p, C.POINTER(Config), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_sample.argtypes = [C.c_void_p, C.POINTER(Config), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rn_sampler_create.argtypes = [C.c_void_p, C.POINTER(Config), C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        L.rn_sampler_warmup.argtypes = [C.c_void_p, C.c_int]
        L.rn_sampler_run.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.rn_sampler_sync.argtypes = [C.c_void_p]
        L.rn_sampler_positions.argtypes = [C.c_void_p, C.c_void_p]
        L.rn_sampler_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rn_sampler_diagnostics.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.rn_sampler_track_diagnostics.argtypes = [C.c_void_p, C.c_int]
        L.rn_sampler_tracked_diagnostics.argtypes = [C.c_void_p, C.c_void_p]
        L.rn_sampler_stream.argtypes = [C.c_void_p]
        L.rn_sampler_stream.restype = C.c_void_p
        L.rn_sampler_launches.argtypes = [C.c_void_p]
        L.rn_sampler_launches.restype = C.c_int64
        L.rn_sampler_destroy.argtypes = [C.c_void_p]
        L.rn_sampler_enable_trace.argtypes = [C.c_void_p]
        L.rn_sampler_read_trace.argtypes = [C.c_void_p, C.c_void_p]
        L.rn_sampler_set_comm.argtypes = [C.c_void_p, C.c_void_p]
        L.rn_sampler_comm_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_double)]
        L.rn_sampler_trajectory_lengths.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        L.rn_trajectory_lengths_sequence.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p]
        L.rn_comm_unique_id.argtypes = [C.c_char_p]
        L.rn_comm_create.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        L.rn_comm_destroy.argtypes = [C.c_void_p]
        L.rn_host_alloc.argtypes = [C.c_int, C.c_size_t, C.POINTER(C.c_void_p)]
        L.rn_host_free.argtypes = [C.c_int, C.c_void_p]
        L.rn_host_register.argtypes = [C.c_int, C.c_void_p, C.c_size_t]
        L.rn_host_unregister.argtypes = [C.c_int, C.c_void_p]
        L.rn_optimize_config_default.argtypes = [C.POINTER(abi.OptimizeConfig)]
        L.rn_optimize.argtypes = [C.c_void_p, C.POINTER(abi.OptimizeConfig), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p]
        L.rn_optimize_emit_source.argtypes = [C.c_void_p, C.POINTER(abi.OptimizeConfig), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_optimize_emit_cubin.argtypes = [C.c_void_p, C.POINTER(abi.OptimizeConfig), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_function_create.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        L.rn_function_ninputs.argtypes = [C.c_void_p]
        L.rn_function_noutputs.argtypes = [C.c_void_p]
        L.rn_function_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.rn_function_eval_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]
        L.rn_function_sync.argtypes = [C.c_void_p]
        L.rn_function_stream.argtypes = [C.c_void_p]
        L.rn_function_stream.restype = C.c_void_p
        L.rn_function_launches.argtypes = [C.c_void_p]
        L.rn_function_launches.restype = C.c_int64
        L.rn_function_emit_source.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_function_emit_cubin.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_function_op_counts.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        L.rn_function_destroy.argtypes = [C.c_void_p]
        L.rn_sample_predict.argtypes = [C.c_void_p, C.POINTER(Config), C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_void_p]
        L.rn_generator_create.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]
        L.rn_generator_ninputs.argtypes = [C.c_void_p]
        L.rn_generator_noutputs.argtypes = [C.c_void_p]
        L.rn_generator_nslots.argtypes = [C.c_void_p]
        L.rn_generator_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]
        L.rn_generator_eval_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                               C.c_void_p]
        L.rn_generator_set_chunk.argtypes = [C.c_void_p, C.c_int64]
        L.rn_generator_report.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.rn_generator_emit_source.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_generator_emit_cubin.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_generator_destroy.argtypes = [C.c_void_p]
        L.rn_sample_generate.argtypes = [C.c_void_p, C.POINTER(Config), C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_void_p]
        L.rn_sampler_save.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rn_sampler_restore.argtypes = [C.c_void_p, C.POINTER(Config), C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int,
                                         C.POINTER(C.c_void_p)]
        L.rn_checkpoint_info.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(abi.CheckpointInfo)]
        L.rn_checkpoint_slice.argtypes = [C.c_void_p, C.c_size_t, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        sizes = (C.c_int32 * 4)()
        L.rn_abi_sizes(sizes)
        if sizes[0] != C.sizeof(Config) or sizes[1] != C.sizeof(ChainStats) or sizes[2] != C.sizeof(RngState):
            raise RainierCudaError(abi.RN_E_INVALID, "ABI struct size mismatch between abi.py and librainier_cuda.so")
        _LIB = L
    return _LIB


def _check(rc):
    if rc != 0:
        raise RainierCudaError(rc, lib().rn_last_error().decode(errors="replace"))


class PinnedBuffer:
    """Page-locked host memory from rn_host_alloc, viewed as a numpy array: rn_sample DMAs results straight into it
    (the JVM analogue is a direct ByteBuffer over the same allocation, see INTEGRATION.md)."""

    def __init__(self, shape, device=0, dtype=np.float64):
        self.device = int(device)
        nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        p = C.c_void_p()
        _check(lib().rn_host_alloc(self.device, max(nbytes, 8), C.byref(p)))
        self.ptr = p.value
        self.array = np.ctypeslib.as_array((C.c_char * max(nbytes, 8)).from_address(self.ptr))[:nbytes].view(dtype).reshape(shape)

    def close(self):
        if getattr(self, "ptr", None):
            self.array = None
            lib().rn_host_free(self.device, self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ----------------------------------------------------------------------------------------------------------
# MassMatrix ADT  (sampler/MassMatrix.scala:3-32)
# ----------------------------------------------------------------------------------------------------------
class MassMatrix:
    pass


class _Identity(MassMatrix):
    def __repr__(self):
        return "IdentityMassMatrix"


IdentityMassMatrix = _Identity()


class DiagonalMassMatrix(MassMatrix):
    def __init__(self, elements):
        self.elements = np.asarray(elements, dtype=np.float64)
        if np.any(self.elements == 0.0):
            raise ValueError("requirement failed")  # MassMatrix.scala:8


class DenseMassMatrix(MassMatrix):
    def __init__(self, elements):
        self.elements = np.asarray(elements, dtype=np.float64).reshape(-1)
        if np.any(self.elements == 0.0):
            raise ValueError("requirement failed")  # MassMatrix.scala:16


# ----------------------------------------------------------------------------------------------------------
# samplers / tuners  (descriptors that lower to rn_config)
# ----------------------------------------------------------------------------------------------------------
class Sampler:
    pass


class HMCSampler(Sampler):
    def __init__(self, nSteps):
        self.nSteps = int(nSteps)


class EHMCSampler(Sampler):
    def __init__(self, maxSteps, minSteps=1, bufSize=100, pCount=0.1):
        self.maxSteps, self.minSteps, self.bufSize, self.pCount = int(maxSteps), int(minSteps), int(bufSize), float(pCount)


class StepSizeTuner:
    pass


class DualAvgTuner(StepSizeTuner):
    def __init__(self, delta):
        self.delta = float(delta)


class StaticStepSize(StepSizeTuner):
    def __init__(self, stepSize):
        self.stepSize = float(stepSize)


class MassMatrixTuner:
    pass


class IdentityMassMatrixTuner(MassMatrixTuner):
    pass


class DiagonalMassMatrixTuner(MassMatrixTuner):
    def __init__(self, initialWindowSize, windowExpansion, skipFirst, skipLast):
        self.initialWindowSize, self.windowExpansion = int(initialWindowSize), float(windowExpansion)
        self.skipFirst, self.skipLast = int(skipFirst), int(skipLast)


class DenseMassMatrixTuner(DiagonalMassMatrixTuner):
    pass


class StaticMassMatrix(MassMatrixTuner):
    def __init__(self, mass):
        self.mass = mass


class SamplerConfig:
    """sampler/Sampler.scala:3-11.  Subclass or pass keyword overrides, like `new DefaultConfig { override ... }`."""
    iterations = 1000
    warmupIterations = 1000
    statsWindow = 100

    def __init__(self, **overrides):
        for k, v in overrides.items():
            setattr(self, k, v)

    def stepSizeTuner(self):
        return getattr(self, "_stepSizeTuner", None) or DualAvgTuner(0.8)

    def massMatrixTuner(self):
        return getattr(self, "_massMatrixTuner", None) or DiagonalMassMatrixTuner(50, 1.5, 50, 50)

    def sampler(self):
        return getattr(self, "_sampler", None) or EHMCSampler(1024)

    # extensions of the CUDA path (not in the reference)
    mathMode = abi.RN_MATH_PARITY
    gradientMode = abi.RN_GRAD_AUTO
    adaptation = abi.RN_ADAPT_PER_CHAIN
    stepAdaptation = abi.RN_ADAPT_PER_CHAIN  # RN_ADAPT_POOLED: one DualAvg step size fitted to all chains' mean acceptance
    trajectoryAdaptation = abi.RN_ADAPT_PER_CHAIN  # RN_ADAPT_POOLED (EHMC): every chain samples with one shared length per
                                                    # iteration, drawn from the U-turn counts of all chains' warmups
    launchIterations = 0
    backend = abi.RN_BACKEND_AUTO


DefaultConfig = SamplerConfig


def make_config(iterations=1000, warmupIterations=1000, statsWindow=100, sampler=None, stepSizeTuner=None,
                massMatrixTuner=None, **ext):
    c = SamplerConfig(iterations=iterations, warmupIterations=warmupIterations, statsWindow=statsWindow, **ext)
    c._sampler, c._stepSizeTuner, c._massMatrixTuner = sampler, stepSizeTuner, massMatrixTuner
    return c


def HMC(warmIt, it, nSteps):  # HMC.scala:26-33
    return make_config(iterations=it, warmupIterations=warmIt, sampler=HMCSampler(nSteps))


def EHMC(warmIt, it, minSteps=1, numLengths=100):  # EHMC.scala:64-73
    return make_config(iterations=it, warmupIterations=warmIt, sampler=EHMCSampler(1000, minSteps, numLengths, 0.1))


def lower_config(config):
    """SamplerConfig -> (rn_config, keepalive).  A user-defined Sampler/tuner subclass cannot be lowered to the
    GPU and is an explicit error (no CPU fallback)."""
    c = Config()
    lib().rn_config_default(C.byref(c))
    keep = []
    c.iterations, c.warmup_iterations, c.stats_window = int(config.iterations), int(config.warmupIterations), int(config.statsWindow)
    s = config.sampler()
    if type(s) is HMCSampler:
        c.sampler, c.n_steps = abi.RN_SAMPLER_HMC, s.nSteps
    elif type(s) is EHMCSampler:
        c.sampler = abi.RN_SAMPLER_EHMC
        c.max_steps, c.min_steps, c.buf_size, c.p_count = s.maxSteps, s.minSteps, s.bufSize, s.pCount
    else:
        raise RainierCudaError(abi.RN_E_UNSUPPORTED, "only the built-in HMCSampler/EHMCSampler can be lowered to the GPU")
    t = config.stepSizeTuner()
    if type(t) is DualAvgTuner:
        c.step_size_tuner, c.delta = abi.RN_STEP_DUAL_AVG, t.delta
    elif type(t) is StaticStepSize:
        c.step_size_tuner, c.static_step_size = abi.RN_STEP_STATIC, t.stepSize
    else:
        raise RainierCudaError(abi.RN_E_UNSUPPORTED, "only DualAvgTuner/StaticStepSize can be lowered to the GPU")
    m = config.massMatrixTuner()
    if type(m) is IdentityMassMatrixTuner:
        c.mass_tuner = abi.RN_MASS_IDENTITY
    elif type(m) in (DiagonalMassMatrixTuner, DenseMassMatrixTuner):
        c.mass_tuner = abi.RN_MASS_DIAGONAL if type(m) is DiagonalMassMatrixTuner else abi.RN_MASS_DENSE
        c.initial_window_size, c.window_expansion = m.initialWindowSize, m.windowExpansion
        c.skip_first, c.skip_last = m.skipFirst, m.skipLast
    elif type(m) is StaticMassMatrix:
        c.mass_tuner = abi.RN_MASS_STATIC
        if m.mass is IdentityMassMatrix:
            c.static_matrix = abi.RN_MATRIX_IDENTITY
        else:
            c.static_matrix = abi.RN_MATRIX_DIAGONAL if isinstance(m.mass, DiagonalMassMatrix) else abi.RN_MATRIX_DENSE
            arr = np.ascontiguousarray(m.mass.elements, dtype=np.float64)
            keep.append(arr)
            c.static_matrix_elements = arr.ctypes.data_as(C.POINTER(C.c_double))
    else:
        raise RainierCudaError(abi.RN_E_UNSUPPORTED, "unknown MassMatrixTuner")
    c.math_mode, c.gradient_mode = int(config.mathMode), int(config.gradientMode)
    c.adaptation, c.launch_iterations = int(config.adaptation), int(config.launchIterations)
    c.step_adaptation = int(config.stepAdaptation)
    c.trajectory_adaptation = int(config.trajectoryAdaptation)
    c.backend = int(config.backend)
    return c, keep


# ----------------------------------------------------------------------------------------------------------
# Stats / Trace
# ----------------------------------------------------------------------------------------------------------
class Stats:
    """sampler/Stats.scala:3-17, rebuilt on the host from rn_chain_stats."""

    def __init__(self, st, rings=None):
        self.gradientEvaluations = st.gradient_evaluations
        self.leapfrogSteps = st.leapfrog_steps
        self.iterations = st.iterations
        self.divergences = st.divergences
        self.accepted = st.accepted
        self.stepSize = st.step_size
        self.energyTransitions2 = st.energy_transitions2
        self.energyVarianceRaw = st.energy_raw
        self.energyVarianceMean = st.energy_mean
        self.stepSizesMean = st.step_sizes_mean
        self.acceptanceRatesMean = st.acceptance_rates_mean
        self.gradsPerIterationMean = st.grads_per_iteration_mean
        self.gradientTimesMean = st.gradient_time_ns_mean    # Stats.gradientTimes.mean (ns), HTMLProgress.scala:65
        self.iterationTimesMean = st.iteration_time_ns_mean  # Stats.iterationTimes.mean (ns), HTMLProgress.scala:57
        self.rings = rings
        self.rng = (st.rng.seed48, st.rng.next_gaussian, st.rng.have_next)

    @property
    def bfmi(self):
        return self.energyTransitions2 / self.energyVarianceRaw


class Trace:
    """rainier-core/.../core/Trace.scala:6-9: chains[chain][iteration][variable], mass per chain, stats per chain."""

    def __init__(self, chains, mass, stats):
        self.chains, self.mass, self.stats = chains, mass, stats

    def requirements(self, function):
        """The device half of Trace.predict (core/Trace.scala:34-41): the values of a generator's requirements
        (Generator.prepare, core/Generator.scala:76-84) for every draw, in predict's order (chain-major), evaluated by
        one rn_function_eval call.  function: CudaFunction compiled from the requirements.  Returns
        [chains*iterations][m]; the host side applies Generator.get to each row."""
        c = np.ascontiguousarray(self.chains, dtype=np.float64)
        return function(c.reshape(-1, c.shape[-1]))

    def generate(self, generator, rng_states):
        """Trace.predict (core/Trace.scala:34-41) with the draws on the device: chain c continues rng_states[c] (one
        RngState, or a (seed48, next_gaussian, have_next) tuple, per chain).  Returns (draws [chains][iterations][m_out],
        the RngStates after the last draw)."""
        return generator(self.chains, rng_states)


# ----------------------------------------------------------------------------------------------------------
# compiled functions (posterior-predictive requirements)
# ----------------------------------------------------------------------------------------------------------
class CudaFunction:
    """Replaces Compiler.compile(inputs, outputs): CompiledFunction (compute/Compiler.scala:22-30) as Generator.prepare
    uses it (core/Generator.scala:59-94): RIR_FLAG_FUNCTION container -> emitted rn_function() + rn_k_eval, evaluated
    for all posterior draws at once."""

    def __init__(self, rir, device=0, fast=False):
        L = lib()
        self._rir = bytes(rir)
        h = C.c_void_p()
        _check(L.rn_function_create(self._rir, len(self._rir), int(device), abi.RN_MATH_FAST if fast else abi.RN_MATH_PARITY,
                                    C.byref(h)))
        self.h = h
        self.nInputs = L.rn_function_ninputs(h)
        self.nOutputs = L.rn_function_noutputs(h)
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            lib().rn_function_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __call__(self, x):
        """x: [count][nInputs] host array -> [count][nOutputs]"""
        x = np.ascontiguousarray(x, dtype=np.float64).reshape(-1, max(self.nInputs, 1))[:, : self.nInputs]
        x = np.ascontiguousarray(x)
        out = np.empty((x.shape[0], self.nOutputs), dtype=np.float64)
        _check(lib().rn_function_eval(self.h, x.ctypes.data, x.shape[0], out.ctypes.data))
        return out

    def eval_device(self, d_x, iterations, chains, d_out, layout=abi.RN_LAYOUT_SAMPLER, stream=None):
        """device pointers (ints); asynchronous -- call sync() before reading d_out"""
        _check(lib().rn_function_eval_device(self.h, C.c_void_p(d_x), layout, iterations, chains, C.c_void_p(d_out),
                                             C.c_void_p(stream) if stream else None))

    def sync(self):
        _check(lib().rn_function_sync(self.h))

    def stream(self):
        return lib().rn_function_stream(self.h)

    def launches(self):
        return lib().rn_function_launches(self.h)

    def emit_source(self):
        need = C.c_size_t()
        _check(lib().rn_function_emit_source(self.h, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _check(lib().rn_function_emit_source(self.h, buf, need.value, C.byref(need)))
        return buf.value.decode()

    def emit_cubin(self):
        need = C.c_size_t()
        _check(lib().rn_function_emit_cubin(self.h, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _check(lib().rn_function_emit_cubin(self.h, buf, need.value, C.byref(need)))
        return buf.raw

    def op_counts(self):
        out = (C.c_double * 2)()
        _check(lib().rn_function_op_counts(self.h, out))
        return {"flops": out[0], "special": out[1]}


def _rng_array(rng_states):
    states = [st if isinstance(st, RngState) else RngState(int(st[0]), float(st[1]), int(st[2]), 0) for st in rng_states]
    return (RngState * max(len(states), 1))(*states), len(states)


def generator_report(err, err_iter):
    """tooling / tests (no device): rn_generator_report -- raises RainierCudaError(RN_E_INVALID) naming the first chain whose
    error bit 0 (a draw over the RNG budget) is set, as rn_generator_eval does after its launches"""
    err = np.ascontiguousarray(err, dtype=np.int32)
    err_iter = np.ascontiguousarray(err_iter, dtype=np.int64)
    _check(lib().rn_generator_report(err.ctypes.data, err_iter.ctypes.data, len(err)))


class CudaGenerator:
    """The Generator.get half of Trace.predict on the device (rn_generator_*): a RIR_FLAG_GENERATOR container (built by
    rainier_b200.generate.lower_generator) -> the slots' rn_function() + rn_k_eval and the plan's rn_k_generate, one thread
    per chain continuing that chain's java.util.Random stream."""

    def __init__(self, rir, device=0):
        L = lib()
        self._rir = bytes(rir)
        h = C.c_void_p()
        _check(L.rn_generator_create(self._rir, len(self._rir), int(device), C.byref(h)))
        self.h = h
        self.nInputs = L.rn_generator_ninputs(h)
        self.nOutputs = L.rn_generator_noutputs(h)
        self.nSlots = L.rn_generator_nslots(h)
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            lib().rn_generator_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __call__(self, x, rng_states):
        """x: [chains][iterations][nInputs] host array; rng_states: one per chain.  Returns (out [chains][iterations][nOutputs],
        list of RngState after the draws)."""
        x = np.ascontiguousarray(x, dtype=np.float64)
        chains, iterations = x.shape[0], x.shape[1]
        arr, k = _rng_array(rng_states)
        if k != chains:
            raise ValueError("one rng state per chain")
        out = np.empty((chains, iterations, self.nOutputs), dtype=np.float64)
        _check(lib().rn_generator_eval(self.h, x.ctypes.data, iterations, chains, C.cast(arr, C.c_void_p), out.ctypes.data))
        return out, list(arr)[:chains]

    def eval_device(self, d_x, iterations, chains, rng_states, d_out, layout=abi.RN_LAYOUT_SAMPLER, stream=None):
        """device pointers (ints); blocking.  Returns the RngStates after the draws."""
        arr, k = _rng_array(rng_states)
        if k != chains:
            raise ValueError("one rng state per chain")
        _check(lib().rn_generator_eval_device(self.h, C.c_void_p(d_x), layout, iterations, chains, C.cast(arr, C.c_void_p),
                                              C.c_void_p(d_out), C.c_void_p(stream) if stream else None))
        return list(arr)[:chains]

    def set_chunk(self, iterations):
        _check(lib().rn_generator_set_chunk(self.h, int(iterations)))

    def emit_source(self):
        need = C.c_size_t()
        _check(lib().rn_generator_emit_source(self.h, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _check(lib().rn_generator_emit_source(self.h, buf, need.value, C.byref(need)))
        return buf.value.decode()

    def emit_cubin(self):
        need = C.c_size_t()
        _check(lib().rn_generator_emit_cubin(self.h, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _check(lib().rn_generator_emit_cubin(self.h, buf, need.value, C.byref(need)))
        return buf.raw


# ----------------------------------------------------------------------------------------------------------
# model
# ----------------------------------------------------------------------------------------------------------
class CudaModel:
    """Replaces Compiler.compileTargets(targetGroup) (compute/Compiler.scala:14-20): frozen DAG (RIR bytes) + data
    columns -> emitted, NVRTC-compiled sm_90a kernels."""

    def __init__(self, rir, cols=(), device=0):
        L = lib()
        self._rir = bytes(rir)
        self._cols = [np.ascontiguousarray(c, dtype=np.float64) for c in cols]
        n = len(self._cols)
        ptrs = (C.c_void_p * max(n, 1))(*[c.ctypes.data for c in self._cols])
        rows = (C.c_int64 * max(n, 1))(*[len(c) for c in self._cols])
        h = C.c_void_p()
        _check(L.rn_model_create(self._rir, len(self._rir), ptrs, rows, n, int(device), C.byref(h)))
        self.h = h
        self.nVars = L.rn_model_nvars(h)
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            lib().rn_model_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def pack_columns(self):
        """debug/test: host image of the device data buffer (tile-major [tile][column][32 rows] per streamed target)"""
        n = len(self._cols)
        ptrs = (C.c_void_p * max(n, 1))(*[c.ctypes.data for c in self._cols])
        need = C.c_size_t()
        _check(lib().rn_model_pack_columns(self.h, ptrs, None, 0, C.byref(need)))
        image = np.zeros(max(need.value, 1), dtype=np.float64)
        _check(lib().rn_model_pack_columns(self.h, ptrs, image.ctypes.data, need.value, C.byref(need)))
        return image

    # -- debug (the analogue of rainier-decompile) --
    def inlined(self):
        """(targets folded at create, monomials summed on the device, rows no longer streamed per gradient)"""
        mono, rows = C.c_int64(0), C.c_int64(0)
        n = lib().rn_model_inlined(self.h, C.byref(mono), C.byref(rows))
        return int(n), int(mono.value), int(rows.value)

    def emit_source(self, config=None):
        cfg = lower_config(config)[0] if config is not None else None
        need = C.c_size_t()
        _check(lib().rn_emit_source(self.h, C.byref(cfg) if cfg else None, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _check(lib().rn_emit_source(self.h, C.byref(cfg) if cfg else None, buf, need.value, C.byref(need)))
        return buf.value.decode()

    def emit_cubin(self, config=None):
        cfg = lower_config(config)[0] if config is not None else None
        need = C.c_size_t()
        _check(lib().rn_emit_cubin(self.h, C.byref(cfg) if cfg else None, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _check(lib().rn_emit_cubin(self.h, C.byref(cfg) if cfg else None, buf, need.value, C.byref(need)))
        return buf.raw

    def op_counts(self, config=None):
        cfg = lower_config(config)[0] if config is not None else None
        out = (C.c_double * 4)()
        _check(lib().rn_model_op_counts(self.h, C.byref(cfg) if cfg else None, out))
        return {"flops_invariant": out[0], "special_invariant": out[1], "flops_rows": out[2], "special_rows": out[3]}

    def separable_structure(self):
        """which streamed targets a device-side inliner could fold into constants (sufficient statistics)"""
        out = (C.c_double * 4)()
        _check(lib().rn_model_separable_structure(self.h, out))
        return {"streamed_targets": int(out[0]), "separable_targets": int(out[1]), "atoms": int(out[2]), "rows_removed": int(out[3])}

    def dot_structure(self, config=None):
        """where the DAG is a dense mat-vec: parameter x column dot products of the streamed row bodies"""
        cfg = lower_config(config)[0] if config is not None else None
        out = (C.c_double * 4)()
        _check(lib().rn_model_dot_structure(self.h, C.byref(cfg) if cfg else None, out))
        return {"dots_per_gradient": out[0], "dot_fmas_per_gradient": out[1], "longest_dot": int(out[2]), "distinct_dots": int(out[3])}

    # -- DensityFunction seam (sampler/DensityFunction.scala:3-8), batched --
    def density_batch(self, q):
        q = np.ascontiguousarray(q, dtype=np.float64).reshape(-1, self.nVars)
        out = np.empty((q.shape[0], self.nVars + 1), dtype=np.float64)
        _check(lib().rn_density_batch(self.h, q.ctypes.data, q.shape[0], out.ctypes.data))
        return out

    def density(self):
        model = self

        class _DF:  # DensityFunction
            nVars = model.nVars

            def update(self, vars):
                self._out = model.density_batch(np.asarray(vars, dtype=np.float64)[None, :])[0]

            @property
            def density(self):
                return self._out[0]

            def gradient(self, index):
                return self._out[index + 1]

        return _DF()

    # -- object Model.sample(t, config) = sample + predict (core/Model.scala:56-63) --
    def sample_predict(self, function, config=None, nChains=4, seeds=None, out=None):
        """model.sample(config).predict(gen) in one call: returns (predictions [chains][iterations][m], Trace without
        chains).  The draws stay on the device; only the requirement values cross PCIe."""
        config = config or SamplerConfig()
        cfg, keep = lower_config(config)
        if seeds is None:
            seeds = np.arange(nChains, dtype=np.int64) + 1
        seeds_a = np.ascontiguousarray(seeds, dtype=np.int64)
        nChains = len(seeds_a)
        n = self.nVars
        dense = cfg.mass_tuner == abi.RN_MASS_DENSE or (cfg.mass_tuner == abi.RN_MASS_STATIC and cfg.static_matrix == abi.RN_MATRIX_DENSE)
        pred = out if out is not None else np.empty((nChains, cfg.iterations, function.nOutputs), dtype=np.float64)
        mass = np.empty((nChains, n * n if dense else n), dtype=np.float64)
        stats = (ChainStats * nChains)()
        rings = np.zeros((nChains, 3, cfg.stats_window), dtype=np.float64)
        cfg.stats_rings = rings.ctypes.data_as(C.POINTER(C.c_double))
        _check(lib().rn_sample_predict(self.h, C.byref(cfg), function.h, seeds_a.ctypes.data, nChains, pred.ctypes.data,
                                       mass.ctypes.data, C.cast(stats, C.c_void_p)))
        return pred, Trace(None, mass, [Stats(stats[c], rings[c]) for c in range(nChains)])

    def sample_generate(self, generator, config=None, nChains=4, seeds=None, out=None):
        """model.sample(config).predict(gen) with the predictive draws on the device (rn_sample_generate): returns
        (draws [chains][iterations][m_out], Trace without chains).  Chain c's draws continue its sampling RNG stream;
        Trace.stats[c].rng is the state after them.  Only the predictive draws cross PCIe."""
        config = config or SamplerConfig()
        cfg, keep = lower_config(config)
        if seeds is None:
            seeds = np.arange(nChains, dtype=np.int64) + 1
        seeds_a = np.ascontiguousarray(seeds, dtype=np.int64)
        nChains = len(seeds_a)
        n = self.nVars
        dense = cfg.mass_tuner == abi.RN_MASS_DENSE or (cfg.mass_tuner == abi.RN_MASS_STATIC and cfg.static_matrix == abi.RN_MATRIX_DENSE)
        draws = out if out is not None else np.empty((nChains, cfg.iterations, generator.nOutputs), dtype=np.float64)
        mass = np.empty((nChains, n * n if dense else n), dtype=np.float64)
        stats = (ChainStats * nChains)()
        rings = np.zeros((nChains, 3, cfg.stats_window), dtype=np.float64)
        cfg.stats_rings = rings.ctypes.data_as(C.POINTER(C.c_double))
        _check(lib().rn_sample_generate(self.h, C.byref(cfg), generator.h, seeds_a.ctypes.data, nChains, draws.ctypes.data,
                                        mass.ctypes.data, C.cast(stats, C.c_void_p)))
        return draws, Trace(None, mass, [Stats(stats[c], rings[c]) for c in range(nChains)])

    # -- Model.optimize / Optimizer.lbfgs, batched over starts --
    @staticmethod
    def _optimize_config(m=5, eps=0.1, max_evals=10000, fast=False, gradient_mode=abi.RN_GRAD_AUTO, backend=abi.RN_BACKEND_AUTO):
        oc = abi.OptimizeConfig()
        lib().rn_optimize_config_default(C.byref(oc))
        oc.history, oc.eps, oc.max_evaluations = int(m), float(eps), int(max_evals)
        oc.math_mode = abi.RN_MATH_FAST if fast else abi.RN_MATH_PARITY
        oc.gradient_mode = gradient_mode
        oc.backend = backend
        return oc

    def optimize(self, x0=None, starts=1, **kw):
        """Optimizer.lbfgs(density()) (optimizer/Optimizer.scala:6-24; Model.optimize, core/Model.scala:26-30) for a batch
        of starts in one kernel.  x0: [starts][n] or None (every start at 0 = the reference's only start).  Returns
        dict(x [starts][n], f [starts] = -density, info [starts], evals [starts])."""
        oc = self._optimize_config(**kw)
        if x0 is not None:
            x0 = np.ascontiguousarray(x0, dtype=np.float64).reshape(-1, self.nVars)
            starts = x0.shape[0]
        x = np.empty((starts, self.nVars), dtype=np.float64)
        f = np.empty(starts, dtype=np.float64)
        info = np.empty(starts, dtype=np.int32)
        evals = np.empty(starts, dtype=np.int32)
        _check(lib().rn_optimize(self.h, C.byref(oc), x0.ctypes.data if x0 is not None else None, starts, x.ctypes.data,
                                 f.ctypes.data, info.ctypes.data, evals.ctypes.data))
        return {"x": x, "f": f, "info": info, "evals": evals}

    def emit_optimizer_source(self, **kw):
        oc = self._optimize_config(**kw)
        need = C.c_size_t()
        _check(lib().rn_optimize_emit_source(self.h, C.byref(oc), None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _check(lib().rn_optimize_emit_source(self.h, C.byref(oc), buf, need.value, C.byref(need)))
        return buf.value.decode()

    def emit_optimizer_cubin(self, **kw):
        oc = self._optimize_config(**kw)
        need = C.c_size_t()
        _check(lib().rn_optimize_emit_cubin(self.h, C.byref(oc), None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _check(lib().rn_optimize_emit_cubin(self.h, C.byref(oc), buf, need.value, C.byref(need)))
        return buf.raw

    # -- Model.sample --
    def sample(self, config=None, nChains=4, seeds=None, rng_states=None, dense_mass=None, out=None, diagnostics=False,
               keep_samples=True):
        """Model.sample(config, nChains) (core/Model.scala:13-24).  Chain c behaves exactly like a single-chain
        reference run with ScalaRNG(seeds[c]).  Returns a Trace with numpy arrays.  `out`: optional C-contiguous
        float64 array [chains][iterations][n] to receive the samples (e.g. PinnedBuffer(...).array)."""
        config = config or SamplerConfig()
        cfg, keep = lower_config(config)
        if rng_states is not None:
            nChains = len(rng_states)
            arr = (RngState * nChains)(*rng_states)
            cfg.rng_states = C.cast(arr, C.POINTER(RngState))
            seeds_a = np.zeros(nChains, dtype=np.int64)
        else:
            if seeds is None:
                seeds = np.arange(nChains, dtype=np.int64) + 1
            seeds_a = np.ascontiguousarray(seeds, dtype=np.int64)
            nChains = len(seeds_a)
        n = self.nVars
        dense = cfg.mass_tuner == abi.RN_MASS_DENSE or (cfg.mass_tuner == abi.RN_MASS_STATIC and cfg.static_matrix == abi.RN_MATRIX_DENSE)
        if out is not None:
            if out.shape != (nChains, cfg.iterations, n) or out.dtype != np.float64 or not out.flags.c_contiguous:
                raise ValueError("out must be a C-contiguous float64 array of shape (chains, iterations, n)")
            samples = out
        else:
            samples = np.empty((nChains, cfg.iterations, n), dtype=np.float64)
        mass = np.empty((nChains, n * n if dense else n), dtype=np.float64)
        stats = (ChainStats * nChains)()
        rings = np.zeros((nChains, 3, cfg.stats_window), dtype=np.float64)
        cfg.stats_rings = rings.ctypes.data_as(C.POINTER(C.c_double))
        diag = np.empty((n, 2), dtype=np.float64) if diagnostics else None
        if diagnostics:
            cfg.diagnostics = diag.ctypes.data_as(C.POINTER(C.c_double))
        _check(lib().rn_sample(self.h, C.byref(cfg), seeds_a.ctypes.data, nChains, samples.ctypes.data if keep_samples else None,
                               mass.ctypes.data, C.cast(stats, C.c_void_p)))
        tr = Trace(samples if keep_samples else None, mass, [Stats(stats[c], rings[c]) for c in range(nChains)])
        tr.diagnostics = diag  # [n][2] = rHat, effectiveSampleSize (Trace.diagnostics), reduced on the device
        return tr


def inline_plan(rir):
    """host half of the device-side inlining (rn_inline_plan): [(target index, n monomials, function-flavour RIR bytes)] for the
    separable streamed targets of a primal container"""
    rir = bytes(rir)
    nt = C.c_int(0)
    _check(lib().rn_inline_plan(rir, len(rir), -1, C.byref(nt), None, None, None, 0, None))
    out = []
    for k in range(nt.value):
        ti, nm, need = C.c_int(0), C.c_int64(0), C.c_size_t(0)
        _check(lib().rn_inline_plan(rir, len(rir), k, None, C.byref(ti), C.byref(nm), None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _check(lib().rn_inline_plan(rir, len(rir), k, None, None, None, buf, need.value, C.byref(need)))
        out.append((ti.value, nm.value, buf.raw))
    return out


def inline_apply(rir, sums):
    """the rewritten (data-free) container for the monomials' row sums (rn_inline_apply); sums: concatenated over targets"""
    rir = bytes(rir)
    s = np.ascontiguousarray(sums, dtype=np.float64)
    need = C.c_size_t(0)
    _check(lib().rn_inline_apply(rir, len(rir), s.ctypes.data, len(s), None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value)
    _check(lib().rn_inline_apply(rir, len(rir), s.ctypes.data, len(s), buf, need.value, C.byref(need)))
    return buf.raw


class Comm:
    """NCCL communicator of the library (rn_comm_*): used only by RN_ADAPT_POOLED's warmup-phase all-reduce.  The
    128-byte unique id is exchanged through torch.distributed (any backend), which is plumbing only."""

    def __init__(self, handle, rank, world):
        self.h, self.rank, self.world = handle, rank, world

    @staticmethod
    def from_torch_distributed(device):
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(), dist.get_world_size()
        buf = C.create_string_buffer(128)
        if rank == 0:
            _check(lib().rn_comm_unique_id(buf))
        t = torch.tensor(list(buf.raw), dtype=torch.uint8)
        if dist.get_backend() == "nccl":
            t = t.cuda(device)
        dist.broadcast(t, src=0)
        raw = bytes(t.cpu().tolist())
        h = C.c_void_p()
        _check(lib().rn_comm_create(raw, rank, world, int(device), C.byref(h)))
        return Comm(h, rank, world)

    def close(self):
        if getattr(self, "h", None):
            lib().rn_comm_destroy(self.h)
            self.h = None


def _blob_view(blob):
    """a bytes-like checkpoint (bytes, bytearray, memoryview, numpy array) as a flat uint8 array over the same memory"""
    a = blob if isinstance(blob, np.ndarray) else np.frombuffer(blob, dtype=np.uint8)
    if not a.flags.c_contiguous:
        raise ValueError("a checkpoint must be one contiguous buffer")
    return a.reshape(-1).view(np.uint8)


def checkpoint_info(blob):
    """rn_checkpoint_info: what a sampler checkpoint holds (no device needed), as a dict"""
    a = _blob_view(blob)
    info = abi.CheckpointInfo()
    _check(lib().rn_checkpoint_info(a.ctypes.data, a.nbytes, C.byref(info)))
    return {f: getattr(info, f) for f, _ in abi.CheckpointInfo._fields_ if f != "reserved"}


def trajectory_lengths_sequence(counts, t0, count):
    """tooling / tests (no device): rn_trajectory_lengths_sequence -- L_t of pooled trajectory lengths for t = t0 .. t0 + count - 1
    given the pooled histogram `counts` (the definition is in rainier_cuda.h, rn_config.trajectory_adaptation)"""
    h = np.ascontiguousarray(counts, dtype=np.int64)
    out = np.zeros(int(count), dtype=np.int32)
    _check(lib().rn_trajectory_lengths_sequence(h.ctypes.data, len(h), int(t0), int(count), out.ctypes.data))
    return out


def checkpoint_slice(blob, begin, end):
    """rn_checkpoint_slice: chains [begin, end) of a checkpoint as a checkpoint of their own (bytearray; no device needed)"""
    a = _blob_view(blob)
    need = C.c_size_t(0)
    _check(lib().rn_checkpoint_slice(a.ctypes.data, a.nbytes, int(begin), int(end), None, 0, C.byref(need)))
    out = bytearray(need.value)
    _check(lib().rn_checkpoint_slice(a.ctypes.data, a.nbytes, int(begin), int(end), (C.c_char * len(out)).from_buffer(out), len(out),
                                     C.byref(need)))
    return out


class CudaSampler:
    """Staged, device-resident sampling (what rn_sample is built from); used by bench.py and the parity tests."""

    def __init__(self, model, config, seeds=None, rng_states=None, trace=False):
        self.model = model
        self.cfg, self._keep = lower_config(config)
        if rng_states is not None:
            self.chains = len(rng_states)
            arr = (RngState * self.chains)(*rng_states)
            self._keep.append(arr)
            self.cfg.rng_states = C.cast(arr, C.POINTER(RngState))
            seeds_a = np.zeros(self.chains, dtype=np.int64)
        else:
            seeds_a = np.ascontiguousarray(seeds, dtype=np.int64)
            self.chains = len(seeds_a)
        h = C.c_void_p()
        _check(lib().rn_sampler_create(model.h, C.byref(self.cfg), seeds_a.ctypes.data, self.chains, C.byref(h)))
        self.h = h
        self._trace = trace
        if trace:
            _check(lib().rn_sampler_enable_trace(self.h))

    def set_comm(self, comm):
        self._comm = comm
        _check(lib().rn_sampler_set_comm(self.h, comm.h))

    def comm_stats(self):
        """(ncclAllReduce calls of the pooled warmup, their summed device time in microseconds)"""
        calls, us = C.c_int64(0), C.c_double(0.0)
        _check(lib().rn_sampler_comm_stats(self.h, C.byref(calls), C.byref(us)))
        return int(calls.value), float(us.value)

    def trajectory_lengths(self):
        """the pooled histogram of U-turn counts over every chain of every rank, int64 [max_steps + 1]
        (trajectoryAdaptation = RN_ADAPT_POOLED, after the first sampling launch)"""
        n = C.c_int(0)
        _check(lib().rn_sampler_trajectory_lengths(self.h, None, 0, C.byref(n)))
        out = np.zeros(n.value, dtype=np.int64)
        _check(lib().rn_sampler_trajectory_lengths(self.h, out.ctypes.data, n.value, C.byref(n)))
        return out

    def warmup(self, iterations=-1):
        _check(lib().rn_sampler_warmup(self.h, int(iterations)))

    def run(self, iterations, d_samples=None):
        """d_samples: device pointer (int) to [iterations][n][chains] float64, or None."""
        _check(lib().rn_sampler_run(self.h, int(iterations), C.c_void_p(d_samples) if d_samples else None))

    def sync(self):
        _check(lib().rn_sampler_sync(self.h))

    @property
    def stream(self):
        return lib().rn_sampler_stream(self.h)

    @property
    def launches(self):
        return lib().rn_sampler_launches(self.h)

    def diagnostics(self, d_samples, iterations, layout=0):
        """Trace.diagnostics (core/Trace.scala:11-21) of a device-resident sample block, reduced on the device.
        d_samples: device pointer; layout 0 = [iterations][n][chains], 1 = [chains][iterations][n].
        Returns an array [n][2] = (rHat, effectiveSampleSize)."""
        out = np.empty((self.model.nVars, 2), dtype=np.float64)
        _check(lib().rn_sampler_diagnostics(self.h, C.c_void_p(d_samples), int(iterations), int(layout), out.ctypes.data))
        return out

    def track_diagnostics(self, thin=1):
        """Trace.thin(thin).diagnostics over every sampling iteration run() performs from now on, accumulated on the device
        as the draws are produced (run() may then be given no sample block).  Calling it again restarts the accumulation."""
        _check(lib().rn_sampler_track_diagnostics(self.h, int(thin)))

    def tracked_diagnostics(self):
        """[n][2] = (rHat, effectiveSampleSize) over the tracked draws; with a communicator attached, over every chain of
        every rank (a collective: every rank calls it)"""
        out = np.empty((self.model.nVars, 2), dtype=np.float64)
        _check(lib().rn_sampler_tracked_diagnostics(self.h, out.ctypes.data))
        return out

    def positions(self):
        q = np.empty((self.chains, self.model.nVars), dtype=np.float64)
        _check(lib().rn_sampler_positions(self.h, q.ctypes.data))
        return q

    def stats(self):
        n = self.model.nVars
        stats = (ChainStats * self.chains)()
        dense = self.cfg.mass_tuner == abi.RN_MASS_DENSE or (self.cfg.mass_tuner == abi.RN_MASS_STATIC and self.cfg.static_matrix == abi.RN_MATRIX_DENSE)
        mass = np.empty((self.chains, n * n if dense else n), dtype=np.float64)
        rings = np.zeros((self.chains, 3, self.cfg.stats_window), dtype=np.float64)
        _check(lib().rn_sampler_stats(self.h, C.cast(stats, C.c_void_p), mass.ctypes.data, rings.ctypes.data))
        return [Stats(stats[c], rings[c]) for c in range(self.chains)], mass

    def save(self, out=None):
        """rn_sampler_save: the sampler's whole state as a checkpoint (DESIGN.md 3.6).  Returns a bytearray, or, with `out` (a
        uint8 numpy array of at least the size, e.g. PinnedBuffer(..., dtype=np.uint8).array: one DMA per chunk), the view of
        `out` that holds it."""
        need = C.c_size_t(0)
        _check(lib().rn_sampler_save(self.h, None, 0, C.byref(need)))
        if out is None:
            buf = bytearray(need.value)
            _check(lib().rn_sampler_save(self.h, (C.c_char * len(buf)).from_buffer(buf), len(buf), C.byref(need)))
            return buf
        a = _blob_view(out)
        if a.nbytes < need.value:
            raise ValueError("out holds %d bytes, the checkpoint needs %d" % (a.nbytes, need.value))
        _check(lib().rn_sampler_save(self.h, a.ctypes.data, a.nbytes, C.byref(need)))
        return a[:need.value]

    @classmethod
    def restore(cls, model, config, blobs, trace=False):
        """rn_sampler_restore: a new sampler whose chains are those of `blobs` (one checkpoint or a list), concatenated in
        order, continuing exactly where they were saved.  `config` must agree with the checkpoints' semantic fields; its
        iterations may be larger (extension).  trace=True records the per-iteration trace from the restore point on."""
        views = [_blob_view(b) for b in (blobs if isinstance(blobs, (list, tuple)) else [blobs])]
        self = cls.__new__(cls)
        self.model = model
        self.cfg, self._keep = lower_config(config)
        ptrs = (C.c_void_p * len(views))(*[v.ctypes.data for v in views])
        lens = (C.c_size_t * len(views))(*[v.nbytes for v in views])
        h = C.c_void_p()
        _check(lib().rn_sampler_restore(model.h, C.byref(self.cfg), ptrs, lens, len(views), C.byref(h)))
        self.h = h
        self.chains = sum(checkpoint_info(v)["chains"] for v in views)
        self.cfg.warmup_iterations = checkpoint_info(views[0])["warmup_iterations"]  # (may differ only once warmup has finished)
        self._trace = trace
        if trace:
            _check(lib().rn_sampler_enable_trace(self.h))
        return self

    def read_trace(self):
        total = self.cfg.warmup_iterations + self.cfg.iterations
        out = np.zeros((self.chains, total, 4), dtype=np.float64)
        _check(lib().rn_sampler_read_trace(self.h, out.ctypes.data))
        return out

    def close(self):
        if getattr(self, "h", None):
            lib().rn_sampler_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

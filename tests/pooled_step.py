"""
Test infrastructure for pooled step-size adaptation (rn_config.step_adaptation == RN_ADAPT_POOLED): the oracle's lockstep
restatement (tests/pooled_step_oracle.cpp, built on the unchanged per-chain oracle) and a host emulation of the runtime's
per-iteration orchestration (one warmup launch per iteration, the iteration's int64 acceptance sum, rn_k_step_pool) over
the kernel source the emitter produces.  Neither is part of the product.
"""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

from oracle.rainier_py.cachedir import private_dir
from rainier_b200.abi import ChainStats, Config

import host_emulation as he

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
Q_SCALE = 4294967296.0  # 2^32: quantum of the pooled acceptance probability
LN2 = 0.6931471805599453
_ORACLE = None


def _oracle_lib():
    global _ORACLE
    if _ORACLE is None:
        srcs = [os.path.join(_HERE, "pooled_step_oracle.cpp"), os.path.join(_ROOT, "oracle", "rainier_oracle.cpp"),
                os.path.join(_ROOT, "oracle", "jmath.h"), os.path.join(_ROOT, "include", "rainier_cuda.h"),
                os.path.join(_ROOT, "include", "rainier_rir.h")]
        key = hashlib.sha1(b"".join(open(p, "rb").read() for p in srcs)).hexdigest()[:16]
        so = os.path.join(private_dir("rno_pooled_step"), key + ".so")
        if not os.path.exists(so):
            tmp = so + ".tmp%d" % os.getpid()
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread", "-w", "-shared",
                            "-o", tmp, srcs[0], "-ldl"], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.rno_last_error.restype = C.c_char_p
        L.rno_model_create.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int, C.c_int,
                                       C.POINTER(C.c_void_p)]
        L.rno_model_destroy.argtypes = [C.c_void_p]
        L.rno_model_nvars.argtypes = [C.c_void_p]
        L.rno_sample_pooled_step.argtypes = [C.c_void_p, C.POINTER(Config), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p]
        _ORACLE = L
    return _ORACLE


def oracle_sample(rir, cols, cfg, seeds, dense_mass=False):
    """the lockstep oracle: dict(samples [chains][iters][n], mass, stats (rn_chain_stats), trace [chains][warm+iters][4])"""
    L = _oracle_lib()
    cols = [np.ascontiguousarray(c, dtype=np.float64) for c in cols]
    ptrs = (C.c_void_p * max(len(cols), 1))(*[c.ctypes.data for c in cols])
    rows = (C.c_int64 * max(len(cols), 1))(*[len(c) for c in cols])
    h = C.c_void_p()
    rir = bytes(rir)
    if L.rno_model_create(rir, len(rir), ptrs, rows, len(cols), 0, C.byref(h)) != 0:
        raise RuntimeError(L.rno_last_error().decode())
    try:
        n = L.rno_model_nvars(h)
        seeds = np.ascontiguousarray(seeds, dtype=np.int64)
        chains = len(seeds)
        samples = np.zeros((chains, cfg.iterations, n))
        mass = np.zeros((chains, n * n if dense_mass else n))
        stats = (ChainStats * chains)()
        trace = np.zeros((chains, cfg.warmup_iterations + cfg.iterations, 4))
        cfg.rng_states = None
        if L.rno_sample_pooled_step(h, C.byref(cfg), seeds.ctypes.data, chains, samples.ctypes.data, mass.ctypes.data,
                                    C.cast(stats, C.c_void_p), trace.ctypes.data) != 0:
            raise RuntimeError(L.rno_last_error().decode())
    finally:
        L.rno_model_destroy(h)
    return {"samples": samples, "mass": mass, "stats": stats, "trace": trace}


_POOLED_SHIM = r"""
// Host emulation of rn_sampler_warmup / run with pooled step-size adaptation: rn_k_init, then rn_k_step_pool(-1) on the sums
// K, C; every warmup iteration is one launch of the warmup kernel that adds into its int64 slot, followed by
// rn_k_step_pool(t, reset) -- rn_runtime.cpp: rn_sampler_warmup / run_phase / step_pool_apply.
extern "C" int emu_sample_pooled(const EmuCfg* c, const long long* seeds, int chains, const double* data, double* samples,
                                 double* trace, long long* out_stats, double* mass_out, int* mass_kind_out, double* da_out) {
  const size_t C = (size_t)chains, n = RN_N, W = (size_t)c->stats_window;
  std::vector<double> params((2 * n + 1) * C), grad(n * C), nng(C), da(5 * C), mass(n * n * C + 1), chol(n * (n + 1) / 2 * C + 1),
      emean(n * C + 1), eraw(n * C + 1), ecov(n * n * C + 1), ring((size_t)c->buf_size * C + 1), energy(3 * C), rings(3 * W * C);
  std::vector<long long> seed(C), grads(C), steps(C), acc(2 + (size_t)c->warmup, 0);
  std::vector<int> have(C), dait(C), ring_i(C), ring_full(C), err(C), iters(C), accepted(C), energy_n(C), sri(3 * C), srf(3 * C);
  RnArgs a;
  std::memset(&a, 0, sizeof(a));
  a.chains = chains;
  a.params = params.data(); a.grad = grad.data(); a.rng_seed = seed.data(); a.rng_nng = nng.data(); a.rng_have = have.data();
  a.da = da.data(); a.da_iter = dait.data(); a.mass = mass.data(); a.chol = chol.data(); a.est_mean = emean.data();
  a.est_raw = eraw.data(); a.est_cov = ecov.data(); a.ring = ring.data(); a.ring_i = ring_i.data(); a.ring_full = ring_full.data();
  a.st_err = err.data(); a.st_grads = grads.data(); a.st_steps = steps.data(); a.st_iters = iters.data();
  a.st_accepted = accepted.data(); a.st_energy = energy.data(); a.st_energy_n = energy_n.data(); a.st_rings = rings.data();
  a.st_ring_i = sri.data(); a.st_ring_full = srf.data(); a.data = data;
  a.sampler = c->sampler; a.n_steps = c->n_steps; a.max_steps = c->max_steps; a.min_steps = c->min_steps; a.buf_size = c->buf_size;
  a.step_tuner = c->step_tuner; a.p_count = c->p_count; a.delta = c->delta; a.static_step = c->static_step;
  a.mass_tuner = c->mass_tuner; a.total_warmup = c->warmup; a.skip_first = c->skip_first; a.skip_last = c->skip_last;
  a.win_expansion = c->win_expansion; a.stats_window = c->stats_window;
  a.chain_begin = 0; a.chain_end = chains;
#if defined(RN_TMA_STAGES) && RN_TMA_STAGES > 0
  a.tma = 1;
#endif
  for (size_t k = 0; k < C; k++) seed[k] = (seeds[k] ^ 0x5DEECE66DLL) & ((1LL << 48) - 1);
  auto launch = [&](void (*kern)(const RnArgs)) {
@LAUNCH@  };
  auto apply = [&](int t, int reset) {  // rn_k_step_pool, one chain per emulated thread
    blockDim.x = 1; gridDim.x = (unsigned)chains; threadIdx.x = 0;
    for (int k = 0; k < chains; k++) { blockIdx.x = (unsigned)k; rn_k_step_pool(a, (const rn_i64*)acc.data(), t, reset); }
  };
  a.mass_kind = 0;
  a.step_acc = (rn_i64*)acc.data();
  launch(rn_k_init);
  apply(-1, 0);
  int win_size = c->initial_window, win_i = 0, win_j = 0, est = 0, mass_kind = 0;
  if (c->mass_tuner == 3) mass_kind = c->static_kind;  // (diagonal / identity static matrices only in these tests)
  if (c->mass_tuner == 3 && c->static_kind == 1)
    for (size_t e = 0; e < n; e++)
      for (size_t k = 0; k < C; k++) mass[e * C + k] = c->static_elements[e];
  for (int t = 0; t < c->warmup; t++) {
    a.phase = 0; a.n_iter = 1; a.mass_kind = mass_kind; a.win_size = win_size; a.win_i = win_i; a.win_j = win_j; a.est_samples = est;
    a.trace = trace ? trace + (size_t)t * 4 * C : nullptr;
    a.step_acc = (rn_i64*)acc.data() + 2 + t;
    launch(RN_K_WARMUP);
    int closed = 0;
    if (c->mass_tuner == 1 || c->mass_tuner == 2) {  // rn_runtime.cpp: advance_window
      win_j += 1;
      if (!(win_j < c->skip_first || (c->warmup - win_j) < c->skip_last)) {
        win_i += 1; est += 1;
        if (win_i == win_size) { closed = 1; win_i = 0; win_size = (int)(win_size * c->win_expansion); mass_kind = c->mass_tuner; }
      }
    }
    apply(t, closed);
  }
  std::fill(grads.begin(), grads.end(), 0); std::fill(steps.begin(), steps.end(), 0); std::fill(iters.begin(), iters.end(), 0);
  std::fill(accepted.begin(), accepted.end(), 0); std::fill(energy.begin(), energy.end(), 0.0); std::fill(energy_n.begin(), energy_n.end(), 0);
  std::fill(rings.begin(), rings.end(), 0.0); std::fill(sri.begin(), sri.end(), 0); std::fill(srf.begin(), srf.end(), 0);
  if (c->iterations > 0) {
    a.phase = 1; a.n_iter = c->iterations; a.mass_kind = mass_kind; a.samples = samples;
    a.trace = trace ? trace + (size_t)c->warmup * 4 * C : nullptr;
    launch(rn_k_iter);
  }
  for (size_t k = 0; k < C; k++) {
    out_stats[k * 5 + 0] = grads[k]; out_stats[k * 5 + 1] = steps[k]; out_stats[k * 5 + 2] = accepted[k]; out_stats[k * 5 + 3] = seed[k];
    out_stats[k * 5 + 4] = err[k];
  }
  const size_t ne = mass_kind == 2 ? n * n : n;
  for (size_t e = 0; e < ne * C; e++) mass_out[e] = mass_kind == 0 ? 1.0 : mass[e];
  for (size_t e = 0; e < 5 * C; e++) da_out[e] = da[e];
  *mass_kind_out = mass_kind;
  return 0;
}
"""

_LAUNCH_TPC = ("    blockDim.x = 1; gridDim.x = (unsigned)chains; threadIdx.x = 0;\n"
               "    for (int k = 0; k < chains; k++) { blockIdx.x = (unsigned)k; kern(a); }\n")
_LAUNCH_WPC = ("    const int spc = c->chains_per_cta > 0 ? c->chains_per_cta : 1, nb = (chains + spc - 1) / spc;\n"
               "    for (int b = 0; b < nb; b++)\n"
               "      rn_emu_run_cta(b, nb, spc, (chains - b * spc) < spc ? (chains - b * spc) : spc, [&] { kern(a); });\n")


def _compile(src):
    assert "#define RN_STEP_POOL 1" in src
    wpc = "#define RN_BACKEND 1" in src
    launch = _LAUNCH_WPC if wpc else _LAUNCH_TPC
    full = (src + (he._WPC_SHIM if wpc else he._SHIM) + he._SAMPLER_SHIM.replace("@LAUNCH@", launch)
            + _POOLED_SHIM.replace("@LAUNCH@", launch))
    d = private_dir("rn_emul")
    key = hashlib.sha1(("pooled-step" + full).encode()).hexdigest()[:16]
    so = os.path.join(d, key + ".so")
    if not os.path.exists(so):
        cpp = os.path.join(d, key + ".cpp")
        with open(cpp, "w") as f:
            f.write(full)
        tmp = so + ".tmp%d" % os.getpid()
        subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-DRN_HOST_EMULATION", "-w", "-pthread", "-ffp-contract=off",
                        cpp, "-o", tmp], check=True)
        os.replace(tmp, so)
    return C.CDLL(so)


def emulate(src, cfg, seeds, model, chains_per_cta=1):
    """runs the emitted pooled-step kernels on the host; returns dict like host_emulation.sample plus `da` [chains][5]"""
    L = _compile(src)
    seeds = np.ascontiguousarray(seeds, dtype=np.int64)
    chains, n = len(seeds), model.nVars
    e = he.EmuCfg(cfg.sampler, cfg.n_steps, cfg.max_steps, cfg.min_steps, cfg.buf_size, cfg.step_size_tuner, cfg.p_count, cfg.delta,
                  cfg.static_step_size, cfg.mass_tuner, cfg.initial_window_size, cfg.skip_first, cfg.skip_last, cfg.window_expansion,
                  cfg.stats_window, cfg.warmup_iterations, cfg.iterations,
                  cfg.static_matrix if cfg.mass_tuner == 3 else 0, cfg.static_matrix_elements if cfg.mass_tuner == 3 else None,
                  int(chains_per_cta))
    it, tot = cfg.iterations, cfg.warmup_iterations + cfg.iterations
    samples = np.zeros((max(it, 1), n, chains))
    trace = np.zeros((max(tot, 1), 4, chains))
    stats = np.zeros((chains, 5), dtype=np.int64)
    mass = np.zeros((n * n, chains))
    da = np.zeros((5, chains))
    kind = C.c_int(0)
    data = model.pack_columns()
    L.emu_sample_pooled.argtypes = [C.POINTER(he.EmuCfg), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.POINTER(C.c_int), C.c_void_p]
    L.emu_sample_pooled(C.byref(e), seeds.ctypes.data, chains, data.ctypes.data, samples.ctypes.data, trace.ctypes.data,
                        stats.ctypes.data, mass.ctypes.data, C.byref(kind), da.ctypes.data)
    ne = n * n if kind.value == 2 else n
    return {"samples": np.ascontiguousarray(samples[:it].transpose(2, 0, 1)), "trace": np.ascontiguousarray(trace[:tot].transpose(2, 0, 1)),
            "stats": stats, "mass": np.ascontiguousarray(mass.reshape(-1)[: ne * chains].reshape(ne, chains).T), "mass_kind": kind.value,
            "da": np.ascontiguousarray(da.T)}


def _vec(which, x):
    from oracle.rainier_py.binding import lib
    x = np.ascontiguousarray(np.atleast_1d(x), dtype=np.float64)
    out = np.empty_like(x)
    lib().rno_vec_math(which, x.ctypes.data_as(C.c_void_p), None, out.ctypes.data_as(C.c_void_p), C.c_int64(len(x)))
    return out


def replay_steps(a, warmup, delta, closes, eps0):
    """Steps 2-4 of the pooled update replayed on the host from the log acceptance probabilities a[chain][t] of a trace, with
    the oracle's math (StrictMath exp / log, Java's pow).  closes: warmup iterations at which a mass window closed
    (stepSizeTuner.reset()).  Returns the step size each warmup iteration used and the final exp(logStepSizeBar)."""
    from oracle.rainier_py.binding import lib
    jpow = lib().rno_jpow
    exp = lambda x: float(_vec(0, x)[0])  # noqa: E731
    log = lambda x: float(_vec(1, x)[0])  # noqa: E731
    chains = a.shape[0]

    def apply(ss):  # DualAvg.apply, DualAvg.scala:80-90
        return {"logStepSize": log(ss), "logStepSizeBar": 0.0, "avgError": 0.0, "iteration": 0, "shrinkageTarget": log(10 * ss)}

    da, step, used = apply(eps0), eps0, []
    for t in range(warmup):
        used.append(step)
        q = np.rint(_vec(0, a[:, t]) * Q_SCALE).astype(np.int64)
        p = float(int(np.sum(q))) / (Q_SCALE * float(chains))
        da["iteration"] += 1
        it = float(da["iteration"])
        am = 1.0 / (it + 10)
        sm = jpow(it, -0.75)
        da["avgError"] = ((1.0 - am) * da["avgError"] + (am * (delta - p)))
        da["logStepSize"] = (da["shrinkageTarget"] - (da["avgError"] * float(np.sqrt(it)) / 0.05))
        da["logStepSizeBar"] = (sm * da["logStepSize"] + (1.0 - sm) * da["logStepSizeBar"])
        step = exp(da["logStepSize"])
        if t in closes:
            ss = exp(da["logStepSizeBar"])
            da, step = apply(ss), ss
    return np.array(used), exp(da["logStepSizeBar"])


def window_closes(cfg):
    """warmup iterations (0-based) at which WindowedMassMatrixTuner closes a window (rn_runtime.cpp: advance_window)"""
    if cfg.mass_tuner not in (1, 2):
        return set()
    out, size, i = set(), cfg.initial_window_size, 0
    for j in range(1, cfg.warmup_iterations + 1):
        if j < cfg.skip_first or (cfg.warmup_iterations - j) < cfg.skip_last:
            continue
        i += 1
        if i == size:
            out.add(j - 1)
            i, size = 0, int(size * cfg.window_expansion)
    return out

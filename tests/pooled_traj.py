"""
Test infrastructure for pooled EHMC trajectory lengths (rn_config.trajectory_adaptation == RN_ADAPT_POOLED): an independent
restatement of the draw L_t defined in rainier_cuda.h, the histogram a sampler pools from its chains' rings, and a reader of
the chain records of a checkpoint (include/rainier_ckpt.h).  None of it is part of the product.
"""
import ctypes as C

import numpy as np

from rainier_b200 import abi

M64 = (1 << 64) - 1
FNV_BASIS, FNV_PRIME = 1469598103934665603, 1099511628211


def fingerprint(h):
    """the 64-bit fingerprint F of the counts: four interleaved FNV-1a-style lanes over the int64 words, then the lanes and the
    byte length folded in (the checkpoints' word hash)"""
    words = [int(x) & M64 for x in np.asarray(h, dtype=np.int64)]
    lanes = [FNV_BASIS, FNV_BASIS ^ 1, FNV_BASIS ^ 2, FNV_BASIS ^ 3]
    for i, w in enumerate(words):
        lanes[i & 3] = ((lanes[i & 3] ^ w) * FNV_PRIME) & M64
    r = (FNV_BASIS * FNV_PRIME) & M64  # no tail bytes: the words are whole
    for v in lanes:
        r = ((r ^ v) * FNV_PRIME) & M64
    return ((r ^ (len(words) * 8)) * FNV_PRIME) & M64


def splitmix64(x):
    z = x & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def lengths(h, t0, count):
    """L_t for t = t0 .. t0 + count - 1: z = splitmix64(F + (t + 1) * 0x9E3779B97F4A7C15), r = mulhi64(z, T),
    L_t = min { l : c[l] > r }"""
    h = np.asarray(h, dtype=np.int64)
    cum = np.cumsum(h)
    T, F = int(cum[-1]), fingerprint(h)
    out = np.empty(count, dtype=np.int64)
    for k in range(count):
        r = (splitmix64(F + (t0 + k + 1) * 0x9E3779B97F4A7C15) * T) >> 64
        out[k] = int(np.searchsorted(cum, r, side="right"))
    return out


def ring_histogram(ring, ring_i, ring_full, max_steps):
    """the pooled histogram of rings [chains][buf_size]: entries [0, ring_full ? buf_size : ring_i + 1) of every chain"""
    h = np.zeros(max_steps + 1, dtype=np.int64)
    for c in range(len(ring)):
        k = ring.shape[1] if ring_full[c] else ring_i[c] + 1
        np.add.at(h, ring[c, :k].astype(np.int64), 1)
    return h


def checkpoint_records(blob):
    """(header, {field id: [chains][elems] array}, the replicated section's bytes) of a checkpoint"""
    b = bytes(blob)
    h = abi.CkptHeader.from_buffer_copy(b[:C.sizeof(abi.CkptHeader)])
    off = C.sizeof(abi.CkptHeader)
    fields = [abi.CkptField.from_buffer_copy(b[off + k * C.sizeof(abi.CkptField):]) for k in range(h.n_fields)]
    rep = off + h.n_fields * C.sizeof(abi.CkptField)
    rec = rep + h.step_bytes + h.pool_bytes + h.reserved1
    R = h.record_bytes
    raw = np.frombuffer(b, dtype=np.uint8, count=h.chains * R, offset=rec).reshape(h.chains, R)
    out, at = {}, 0
    for f in fields:
        dt = {abi.CKPT_F64: np.float64, abi.CKPT_I64: np.int64, abi.CKPT_I32: np.int32}[f.type]
        nb = f.elems * np.dtype(dt).itemsize
        out[f.id] = raw[:, at:at + nb].copy().view(dt).reshape(h.chains, f.elems)
        at += nb
    return h, out, b[rep:rec]


def checkpoint_histogram(blob):
    """the pooled histogram a checkpoint carries (None before the first sampling launch built it)"""
    h, _, rep = checkpoint_records(blob)
    if h.reserved1 == 0:
        return None
    return np.frombuffer(rep[len(rep) - h.reserved1:], dtype=np.int64).copy()


def checkpoint_ring_histogram(blob):
    """the histogram of a checkpoint's chains' rings, restated from the records"""
    h, rec, _ = checkpoint_records(blob)
    return ring_histogram(rec[abi.CKPT_RING], rec[abi.CKPT_RING_I][:, 0], rec[abi.CKPT_RING_FULL][:, 0], h.max_steps)


# ---------------------------------------------------------------------------------------------------------------------
# The oracle's restatement (tests/pooled_traj_oracle.cpp) and a host emulation of the runtime's orchestration over the
# emitted kernel source
# ---------------------------------------------------------------------------------------------------------------------
import hashlib  # noqa: E402
import os  # noqa: E402
import subprocess  # noqa: E402

from oracle.rainier_py.cachedir import private_dir  # noqa: E402
from rainier_b200.abi import ChainStats, Config  # noqa: E402

import host_emulation as he  # noqa: E402

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_ORACLE = None


def _oracle_lib():
    global _ORACLE
    if _ORACLE is None:
        srcs = [os.path.join(_HERE, "pooled_traj_oracle.cpp"), os.path.join(_ROOT, "oracle", "rainier_oracle.cpp"),
                os.path.join(_ROOT, "oracle", "jmath.h"), os.path.join(_ROOT, "include", "rainier_cuda.h"),
                os.path.join(_ROOT, "include", "rainier_rir.h")]
        key = hashlib.sha1(b"".join(open(p, "rb").read() for p in srcs)).hexdigest()[:16]
        so = os.path.join(private_dir("rno_pooled_traj"), key + ".so")
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
        L.rno_sample_pooled_traj.argtypes = [C.c_void_p, C.POINTER(Config), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p]
        _ORACLE = L
    return _ORACLE


def oracle_sample(rir, cols, cfg, seeds):
    """dict(samples [chains][iters][n], mass [chains][n], stats (rn_chain_stats), trace [chains][warm+iters][4], hist)"""
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
        mass = np.zeros((chains, n))
        stats = (ChainStats * chains)()
        trace = np.zeros((chains, cfg.warmup_iterations + cfg.iterations, 4))
        hist = np.zeros(cfg.max_steps + 1, dtype=np.int64)
        cfg.rng_states = None
        if L.rno_sample_pooled_traj(h, C.byref(cfg), seeds.ctypes.data, chains, samples.ctypes.data, mass.ctypes.data,
                                    C.cast(stats, C.c_void_p), trace.ctypes.data, hist.ctypes.data) != 0:
            raise RuntimeError(L.rno_last_error().decode())
    finally:
        L.rno_model_destroy(h)
    return {"samples": samples, "mass": mass, "stats": stats, "trace": trace, "hist": hist}


_TRAJ_SHIM = r"""
// Host emulation of rn_sampler_warmup / run with pooled trajectory lengths (rn_runtime.cpp: traj_build / run_phase): rn_k_init,
// one warmup launch, rn_k_traj_hist over each emulated rank's chains into that rank's histogram, their sum (the all-reduce), the
// prefix sums and the word hash, then the sampling iterations in two launches (the second starts at t = split).
static unsigned long long emu_hash(const std::vector<long long>& h) {
  const unsigned long long basis = 1469598103934665603ull, prime = 1099511628211ull;
  unsigned long long lane[4] = {basis, basis ^ 1, basis ^ 2, basis ^ 3};
  for (size_t i = 0; i < h.size(); i++) lane[i & 3] = (lane[i & 3] ^ (unsigned long long)h[i]) * prime;
  unsigned long long r = basis * prime;
  for (int l = 0; l < 4; l++) r = (r ^ lane[l]) * prime;
  return (r ^ (unsigned long long)(h.size() * 8)) * prime;
}
extern "C" int emu_sample_traj(const EmuCfg* c, const long long* seeds, int chains, const double* data, double* samples,
                               double* trace, long long* out_stats, double* mass_out, int ranks, int split, long long* rank_hists,
                               long long* hist) {
  const size_t C = (size_t)chains, n = RN_N, W = (size_t)c->stats_window, B = (size_t)c->max_steps + 1;
  std::vector<double> params((2 * n + 1) * C), grad(n * C), nng(C), da(5 * C), mass(n * n * C + 1), chol(n * (n + 1) / 2 * C + 1),
      emean(n * C + 1), eraw(n * C + 1), ecov(n * n * C + 1), ring((size_t)c->buf_size * C + 1), energy(3 * C), rings(3 * W * C);
  std::vector<long long> seed(C), grads(C), steps(C), h(B, 0), cum(B);
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
  a.mass_kind = 0;
  launch(rn_k_init);
  int win_size = c->initial_window, win_i = 0, win_j = 0, est = 0, mass_kind = 0;
  if (c->warmup > 0) {
    a.phase = 0; a.n_iter = c->warmup; a.mass_kind = 0; a.win_size = win_size; a.win_i = 0; a.win_j = 0; a.est_samples = 0;
    a.trace = trace;
    launch(RN_K_WARMUP);
    if (c->mass_tuner == 1)
      for (int k = 0; k < c->warmup; k++) {
        win_j += 1;
        if (win_j < c->skip_first || (c->warmup - win_j) < c->skip_last) continue;
        win_i += 1; est += 1;
        if (win_i == win_size) { win_i = 0; win_size = (int)(win_size * c->win_expansion); mass_kind = 1; }
      }
  }
  std::fill(grads.begin(), grads.end(), 0); std::fill(steps.begin(), steps.end(), 0); std::fill(iters.begin(), iters.end(), 0);
  std::fill(accepted.begin(), accepted.end(), 0); std::fill(energy.begin(), energy.end(), 0.0); std::fill(energy_n.begin(), energy_n.end(), 0);
  std::fill(rings.begin(), rings.end(), 0.0); std::fill(sri.begin(), sri.end(), 0); std::fill(srf.begin(), srf.end(), 0);
  for (int r = 0; r < ranks; r++) {  // dist.chain_block: the first chains % ranks ranks hold one chain more
    const int base = chains / ranks, extra = chains % ranks;
    const int lo = r * base + (r < extra ? r : extra), hi = lo + base + (r < extra ? 1 : 0);
    a.traj_hist = (rn_i64*)(rank_hists + (size_t)r * B);
    blockDim.x = 1; gridDim.x = (unsigned)chains; threadIdx.x = 0;
    for (int k = lo; k < hi; k++) { blockIdx.x = (unsigned)k; rn_k_traj_hist(a); }
    for (size_t l = 0; l < B; l++) h[l] += rank_hists[(size_t)r * B + l];
  }
  long long run = 0;
  for (size_t l = 0; l < B; l++) cum[l] = run += h[l];
  std::memcpy(hist, h.data(), B * 8);
  a.traj_cum = (const rn_i64*)cum.data(); a.traj_total = cum.back(); a.traj_fp = (rn_i64)emu_hash(h); a.traj_bins = (int)B;
  for (int part = 0; part < 2; part++) {
    const int t0 = part ? split : 0, k = part ? c->iterations - split : split;
    if (k <= 0) continue;
    a.phase = 1; a.n_iter = k; a.mass_kind = mass_kind; a.traj_t0 = t0;
    a.samples = samples + (size_t)t0 * n * C;
    a.trace = trace ? trace + (size_t)(c->warmup + t0) * 4 * C : nullptr;
    launch(rn_k_iter);
  }
  for (size_t k = 0; k < C; k++) {
    out_stats[k * 5 + 0] = grads[k]; out_stats[k * 5 + 1] = steps[k]; out_stats[k * 5 + 2] = accepted[k]; out_stats[k * 5 + 3] = seed[k];
    out_stats[k * 5 + 4] = err[k];
  }
  for (size_t e = 0; e < n * C; e++) mass_out[e] = mass_kind == 0 ? 1.0 : mass[e];
  return 0;
}
"""


def _compile(src):
    assert "#define RN_TRAJ_POOL 1" in src
    wpc = "#define RN_BACKEND 1" in src
    launch = ("    const int spc = c->chains_per_cta > 0 ? c->chains_per_cta : 1, nb = (chains + spc - 1) / spc;\n"
              "    for (int b = 0; b < nb; b++)\n"
              "      rn_emu_run_cta(b, nb, spc, (chains - b * spc) < spc ? (chains - b * spc) : spc, [&] { kern(a); });\n") if wpc else \
        ("    blockDim.x = 1; gridDim.x = (unsigned)chains; threadIdx.x = 0;\n"
         "    for (int k = 0; k < chains; k++) { blockIdx.x = (unsigned)k; kern(a); }\n")
    full = (src + (he._WPC_SHIM if wpc else he._SHIM) + he._SAMPLER_SHIM.replace("@LAUNCH@", launch)
            + _TRAJ_SHIM.replace("@LAUNCH@", launch))
    d = private_dir("rn_emul")
    key = hashlib.sha1(("pooled-traj" + full).encode()).hexdigest()[:16]
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


def emulate(src, cfg, seeds, model, chains_per_cta=1, ranks=1, split=None):
    """runs the emitted RN_TRAJ_POOL kernels on the host; dict like host_emulation.sample plus `hist` and `rank_hists`"""
    L = _compile(src)
    seeds = np.ascontiguousarray(seeds, dtype=np.int64)
    chains, n = len(seeds), model.nVars
    e = he.EmuCfg(cfg.sampler, cfg.n_steps, cfg.max_steps, cfg.min_steps, cfg.buf_size, cfg.step_size_tuner, cfg.p_count, cfg.delta,
                  cfg.static_step_size, cfg.mass_tuner, cfg.initial_window_size, cfg.skip_first, cfg.skip_last, cfg.window_expansion,
                  cfg.stats_window, cfg.warmup_iterations, cfg.iterations, 0, None, int(chains_per_cta))
    it, tot = cfg.iterations, cfg.warmup_iterations + cfg.iterations
    samples = np.zeros((max(it, 1), n, chains))
    trace = np.zeros((max(tot, 1), 4, chains))
    stats = np.zeros((chains, 5), dtype=np.int64)
    mass = np.zeros((n, chains))
    B = cfg.max_steps + 1
    rank_hists = np.zeros((ranks, B), dtype=np.int64)
    hist = np.zeros(B, dtype=np.int64)
    data = model.pack_columns()
    L.emu_sample_traj.argtypes = [C.POINTER(he.EmuCfg), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.emu_sample_traj(C.byref(e), seeds.ctypes.data, chains, data.ctypes.data, samples.ctypes.data, trace.ctypes.data,
                      stats.ctypes.data, mass.ctypes.data, int(ranks), int(it if split is None else split), rank_hists.ctypes.data,
                      hist.ctypes.data)
    return {"samples": np.ascontiguousarray(samples[:it].transpose(2, 0, 1)), "trace": np.ascontiguousarray(trace[:tot].transpose(2, 0, 1)),
            "stats": stats, "mass": np.ascontiguousarray(mass.T), "hist": hist, "rank_hists": rank_hists}

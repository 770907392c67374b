"""
Test infrastructure for the generator flavour (rn_generator_*, rn_generate.cuh):

  * run_plan: a Python executor of a RIR_FLAG_GENERATOR plan (include/rainier_rir.h) -- the reference semantics of the wire
    format, written from Continuous.scala / Discrete.scala like the closures of oracle/rainier_py/core.py, with Java's D2L /
    D2I conversions and Long arithmetic instead of Python ints, fdlibm log / exp / pow (oracle/jmath.h) and the per-draw RNG
    budget of rn_generate.cuh;
  * emulate: the emitted generator source compiled for the host (-DRN_HOST_EMULATION) and run one "thread" at a time through
    the same chunked rn_k_eval + rn_k_generate sequence rn_generator_eval_device launches;
  * fdlibm: a context manager that points the jlog / jexp / jpow of core.py's closures and compute.py's Evaluator at fdlibm.
"""
import contextlib
import ctypes as C
import hashlib
import math
import os
import struct
import subprocess

import numpy as np

from oracle.rainier_py import compute, core
from oracle.rainier_py.binding import JRandom, RngState
from oracle.rainier_py.cachedir import private_dir
from oracle.rainier_py.compute import jd2i
from rainier_b200 import generate as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUDGET = 1 << 24  # rn_generate.cuh: RN_GEN_BUDGET
NAN = float("nan")

_JMATH = None


def _jmath():
    global _JMATH
    if _JMATH is None:
        src = ('#include "%s"\nextern "C" double j_log(double x) { return rno::strict_log(x); }\n'
               'extern "C" double j_exp(double x) { return rno::strict_exp(x); }\n'
               'extern "C" double j_pow(double x, double y) { return rno::strict_pow(x, y); }\n') % os.path.join(ROOT, "oracle", "jmath.h")
        d = private_dir("rn_emul")
        so = os.path.join(d, "jmath_" + hashlib.sha1((src + open(os.path.join(ROOT, "oracle", "jmath.h")).read()).encode()).hexdigest()[:16] + ".so")
        if not os.path.exists(so):
            cpp = so[:-3] + ".cpp"
            with open(cpp, "w") as f:
                f.write(src)
            subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-w", cpp, "-o", so], check=True)
        L = C.CDLL(so)
        for name, n in (("j_log", 1), ("j_exp", 1), ("j_pow", 2)):
            getattr(L, name).restype = C.c_double
            getattr(L, name).argtypes = [C.c_double] * n
        _JMATH = L
    return _JMATH


def jlog(x):
    return _jmath().j_log(x)


def jexp(x):
    return _jmath().j_exp(x)


def jpow(x, y):
    return _jmath().j_pow(x, y)


@contextlib.contextmanager
def fdlibm():
    """core.py's generator closures and compute.py's Evaluator with Java's Math.log / exp / pow pinned to fdlibm (as the
    device path and the compiled functions are)"""
    saved = [(m, m.jlog, m.jexp, m.jpow) for m in (core, compute)]
    for m in (core, compute):
        m.jlog, m.jexp, m.jpow = jlog, jexp, jpow
    try:
        yield
    finally:
        for m, a, b, c in saved:
            m.jlog, m.jexp, m.jpow = a, b, c


def d2l(v):
    if v != v:
        return 0
    if v >= 9.223372036854775807e18:
        return (1 << 63) - 1
    if v <= -9.223372036854775808e18:
        return -(1 << 63)
    return int(v)


def wrap64(n):
    return ((n + (1 << 63)) % (1 << 64)) - (1 << 63)


def _div(a, b):
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def _sqrt(a):
    with np.errstate(all="ignore"):
        return float(np.sqrt(np.float64(a)))


def _floor(a):
    return float(np.floor(np.float64(a)))


def _mul(a, b):
    with np.errstate(all="ignore"):
        return float(np.float64(a) * np.float64(b))


class _Budget(Exception):
    pass


class _Draws:
    def __init__(self, rand):
        self.r, self.calls = rand, 0

    def u(self):
        if self.calls >= BUDGET:
            raise _Budget()
        self.calls += 1
        return self.r.nextDouble()

    def n(self):
        if self.calls >= BUDGET:
            raise _Budget()
        self.calls += 1
        return self.r.nextGaussian()


def _gamma_mt(D, a):
    while True:
        d = a - 1.0 / 3.0
        c = _div(1.0 / 3.0, _sqrt(d))
        x = D.n()
        v = 1.0 + c * x
        while v <= 0:
            x = D.n()
            v = 1.0 + c * x
        v3 = v * v * v
        u = D.u()
        if (u < 1 - 0.0331 * x * x * x * x) or (jlog(u) < 0.5 * x * x + d * (1 - v3 + jlog(v3))):
            return d * v3


def _gamma(D, a):
    if a < 1:
        u = D.u()
        return _mul(_gamma_mt(D, a + 1), jpow(u, _div(1.0, a)))
    return _gamma_mt(D, a)


def _geometric(D, q):
    u = D.u()
    return d2l(_floor(_div(jlog(u), jlog(1 - q))))


def _log_factorial(n):
    x = float(wrap64(n + 1))
    return ((x - 0.5) * jlog(x)) - x + (0.5 * jlog(2 * math.pi))


def _poisson(D, lam):
    if lam < 30.0:
        l = jexp(-lam)
        if l >= 1.0:
            return 0
        k, p = 0, 1.0
        while p > l:
            k += 1
            p *= D.u()
        return k - 1
    c = 0.767 - _div(3.36, lam)
    beta = _div(math.pi, _sqrt(3.0 * lam))
    alpha = beta * lam
    k = jlog(c) - lam - jlog(beta)
    while True:
        u = D.u()
        x = _div(alpha - jlog(_div(1.0 - u, u)), beta)
        n = d2l(_floor(x + 0.5))
        if n >= 0:
            v = D.u()
            y = alpha - beta * x
            lhs = y + jlog(_div(v, jpow(1.0 + jexp(y), 2)))
            rhs = k + float(n) * jlog(lam) - _log_factorial(n)
            if lhs <= rhs:
                return n


def _binomial(D, p, k, pk, kp, sd, cdf0):
    if k >= 100 and k * p <= 10:
        return min(_poisson(D, pk), d2l(k))
    if k >= 100 and k * p >= 9 and k * (1.0 - p) >= 9:
        z = D.n()
        return min(max(d2l(z * sd + kp), 0), d2l(k))
    count = 0
    for _ in range(jd2i(k)):
        if cdf0 >= D.u():
            count += 1
    return count


def _negbinomial(D, p, n, q, mean, sd):
    if p < _div(-100, n) + 1 and p > _div(100, n) - .25:
        z = D.n()
        return max(d2l(z * sd + mean), 0)
    total = 0
    for _ in range(max(d2l(n), 0)):
        total = wrap64(total + _geometric(D, q))
    return total


def parse(rir):
    """-> (ops [(kind, slots, k)], m_out, n_slots) of a generator container"""
    n_nodes, n_targets, n_lookup = struct.unpack_from("<I", rir, 16)[0], struct.unpack_from("<I", rir, 20)[0], struct.unpack_from("<I", rir, 24)[0]
    assert n_targets == 1
    off = 32 + 32 * n_nodes + ((4 * n_lookup + 7) & ~7)
    n_out = struct.unpack_from("<I", rir, off + 16)[0]
    off += 24 + ((4 * n_out + 7) & ~7)
    n_ops, m_out = struct.unpack_from("<2I", rir, off)[:2]
    off += G.GEN_HEADER.size
    ops = []
    for i in range(n_ops):
        f = G.GEN_OP.unpack_from(rir, off + i * G.GEN_OP.size)
        ops.append((f[0], list(f[1:7]), f[8]))
    return ops, m_out, n_out


def run_plan(rir, slot_rows, state):
    """One chain: slot_rows [iterations][n_slots] (the function's outputs at the chain's draws, in iteration order), state: the
    chain's RngState.  Returns (out [iterations][m_out], RngState after the draws, first iteration whose draw exceeded the
    budget or None).  Like rn_k_generate, the chain stops at a draw that exceeds the budget."""
    ops, m, _ = parse(rir)
    match, stack = {}, []
    for i, (kind, _, _) in enumerate(ops):
        if kind == G.REPEAT:
            stack.append(i)
        elif kind == G.END:
            match[stack.pop()] = i
    rand = JRandom()
    rand.set_state(state)
    D = _Draws(rand)
    out = np.zeros((len(slot_rows), m))
    first_bad = None
    for t, s in enumerate(slot_rows):
        s = [float(x) for x in s]
        row, st = [], {"v": 0.0}

        def draw(f, *a):
            D.calls = 0
            return float(f(D, *a))

        def run(i0, i1):
            i = i0
            while i < i1:
                kind, sl, k = ops[i]
                v = st["v"]
                if kind == G.REPEAT:
                    for _ in range(k):
                        run(i + 1, match[i])
                    i = match[i] + 1
                    continue
                if kind == G.NORMAL:
                    v = draw(lambda D: D.n())
                elif kind == G.CAUCHY:
                    v = draw(lambda D: _div(D.n(), D.n()))
                elif kind == G.LAPLACE:
                    def lap(D):
                        u = D.u() - 0.5
                        sgn = 1.0 if u > 0 else (-1.0 if u < 0 else u)
                        return sgn * -1 * jlog(1 - (2 * abs(u)))
                    v = draw(lap)
                elif kind == G.UNIFORM:
                    v = draw(lambda D: D.u())
                elif kind == G.GAMMA:
                    v = draw(_gamma, s[sl[0]])
                elif kind == G.BETA:
                    x = draw(_gamma, s[sl[0]])
                    y = draw(_gamma, s[sl[1]])
                    v = _div(x, x + y)
                elif kind == G.SCALE:
                    v = _mul(v, s[sl[0]])
                elif kind == G.TRANSLATE:
                    v = v + s[sl[0]]
                elif kind == G.EXP:
                    v = jexp(v)
                elif kind == G.EMIT:
                    row.append(v)
                elif kind == G.BERNOULLI:
                    v = draw(lambda D, p: 1 if D.u() <= p else 0, s[sl[0]])
                elif kind == G.GEOMETRIC:
                    v = draw(_geometric, s[sl[0]])
                elif kind == G.POISSON:
                    v = draw(_poisson, s[sl[0]])
                elif kind == G.BINOMIAL:
                    v = draw(_binomial, *[s[j] for j in sl[:6]])
                elif kind == G.NEGBINOMIAL:
                    v = draw(_negbinomial, *[s[j] for j in sl[:5]])
                elif kind == G.VALUE:
                    v = s[sl[0]]
                st["v"] = v
                i += 1

        try:
            run(0, len(ops))
        except _Budget:  # the chain stops: this iteration and the later ones are NaN, the RNG stays where the draw stopped
            out[t:] = NAN
            first_bad = t
            break
        out[t] = row
    return out, rand_state(rand), first_bad


def rand_state(rand):
    return RngState(rand.seed, rand.next_next, 1 if rand.have_next else 0, 0)


# ---- host emulation of the emitted source -------------------------------------------------------------------------------
_SHIM = r"""
#include <vector>
// Host emulation of rn_generator_eval_device (rn_runtime.cpp: generator_run): per chunk of iterations one rn_k_eval launch
// (CTAs of 128 "threads") into the [iteration][slot][chain] scratch, then one rn_k_generate launch (one "thread" per chain).
extern "C" void emu_generate(const double* x, int layout, long long I, long long C, RnRngState* rng, double* out, int* err,
                             long long* err_iter, int* lookup, long long chunk) {
  const long long n = RN_N, M = RN_M;
  for (long long c = 0; c < C; c++) { err[c] = 0; err_iter[c] = -1; }
  *lookup = 0;
  std::vector<double> slots((size_t)(chunk * M * C) + 1);
  for (long long t0 = 0; t0 < I; t0 += chunk) {
    const long long cnt = chunk < I - t0 ? chunk : I - t0;
    RnEvalArgs e;
    e.count = cnt * C;
    if (layout == 0) { e.x = x + t0 * n * C; e.in_inner = C; e.in_outer = n * C; e.in_pstride = 1; e.in_estride = C; }
    else { e.x = x + t0 * n; e.in_inner = C; e.in_outer = n; e.in_pstride = I * n; e.in_estride = 1; }
    e.out = slots.data(); e.out_inner = C; e.out_outer = M * C; e.out_pstride = 1; e.out_estride = C;
    e.err = lookup;
    const unsigned ge = (unsigned)((e.count + 127) / 128 < 3 ? (e.count + 127) / 128 : 3);
    blockDim.x = 128; gridDim.x = ge;
    for (unsigned b = 0; b < ge; b++)
      for (unsigned t = 0; t < 128; t++) { blockIdx.x = b; threadIdx.x = t; rn_k_eval(e); }
    RnGenArgs a;
    a.slots = slots.data(); a.out = out; a.rng = rng; a.err = err; a.err_iter = err_iter;
    a.chains = C; a.t0 = t0; a.t1 = t0 + cnt; a.iterations = I;
    const unsigned gg = (unsigned)((C + 127) / 128);
    gridDim.x = gg;
    for (unsigned b = 0; b < gg; b++)
      for (unsigned t = 0; t < 128; t++) { blockIdx.x = b; threadIdx.x = t; rn_k_generate(a); }
  }
}
"""


def _compile(src):
    d = private_dir("rn_emul")
    key = hashlib.sha1((src + _SHIM).encode()).hexdigest()[:16]
    so = os.path.join(d, "gen_" + key + ".so")
    if not os.path.exists(so):
        cpp = so[:-3] + ".cpp"
        with open(cpp, "w") as f:
            f.write(src + _SHIM)
        subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-DRN_HOST_EMULATION", "-w", "-ffp-contract=off", cpp, "-o", so],
                       check=True)
    L = C.CDLL(so)
    L.emu_generate.argtypes = [C.c_void_p, C.c_int, C.c_longlong, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_longlong]
    return L


def emulate(src, x, states, m_out, layout="rows", chunk=None):
    """Runs the emitted generator source on the host.  layout "rows": x [chains][iterations][n]; "sampler": x
    [iterations][n][chains].  Returns (out [chains][iterations][m_out], RngStates after, err [chains], err_iter [chains])."""
    L = _compile(src)
    x = np.ascontiguousarray(x, dtype=np.float64)
    if layout == "rows":
        chains, iters = x.shape[0], x.shape[1]
    else:
        iters, chains = x.shape[0], x.shape[2]
    arr = (RngState * chains)(*[RngState(s.seed48, s.next_gaussian, s.have_next, 0) for s in states])
    out = np.full((chains, iters, m_out), np.nan)
    err = np.zeros(chains, dtype=np.int32)
    err_iter = np.zeros(chains, dtype=np.int64)
    lookup = C.c_int(0)
    L.emu_generate(x.ctypes.data, 1 if layout == "rows" else 0, iters, chains, C.cast(arr, C.c_void_p), out.ctypes.data,
                   err.ctypes.data, err_iter.ctypes.data, C.byref(lookup), int(chunk or max(iters, 1)))
    assert lookup.value == 0
    return out, list(arr), err, err_iter

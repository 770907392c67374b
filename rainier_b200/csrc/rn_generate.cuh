// rn_generate.cuh -- hand-written half of the generator flavour: the posterior-predictive draws of Trace.predict
// (rainier-core/.../core/Trace.scala:34-41), i.e. `Generator.get(rng, evaluator)` for every posterior draw, on the device.
//
// One thread per chain.  The reference draws from ONE java.util.Random stream per chain, in iteration order, and the number
// of RNG calls a draw makes depends on the data (rejection loops, Poisson's product loop, the Binomial repeat), so a chain's
// stream cannot be split: the parallelism is the chains.  Every chain runs the same plan, so the control flow of the emitted
// rn_generate() is warp-uniform except where the reference's own loops run a data-dependent number of times.
//
// The distributions restate rainier-core/.../core/Continuous.scala and Discrete.scala line for line, in the same evaluation
// order; Math.log / exp / pow are fdlibm (rn_log / rn_exp / rn_pow in parity mode), Math.sqrt / floor and division IEEE, no
// FMA contraction (the generator flavour is always compiled with --fmad=false).
//
// Bounded work: some parameter values make the reference loop forever or nearly so (Poisson.large with lambda = NaN or inf,
// a Binomial repeat or a NegativeBinomial geometric sum over a huge count, ...).  Every draw of a built-in distribution (a
// Beta counts as its two Gamma draws) may make at most RN_GEN_BUDGET RNG calls (standardUniform or standardNormal); the call
// that would exceed it is not made.  The chain then stops for the rest of the call: the outputs of that iteration and of
// every later one are NaN, no further RNG call is made (the returned state is where the failed draw stopped), the chain gets
// error bit 0 and rn_generator_eval fails with RN_E_INVALID naming the chain and iteration.  So a call costs at most one
// over-budget draw per chain, and other chains are unaffected.  One over-budget draw is 2^24 RNG calls in one thread: in the
// host emulation (-O1, one x86 core) 0.06 s for a Binomial repeat and 0.8 s for Poisson.large with lambda = NaN (fdlibm
// log / exp / pow per iteration); not measured on the device, where one thread runs slower than a CPU core.
#ifndef RN_GENERATE_CUH
#define RN_GENERATE_CUH

#define RN_GEN_BUDGET (1 << 24)

// the per-op draws are called from straight-line emitted code, once per op of the plan: out of line, so that a plan of a
// thousand draws compiles to a thousand calls rather than a thousand inlined rejection loops
#ifdef RN_HOST_EMULATION
#define RN_GEN_OP static
#else
#define RN_GEN_OP __device__ __noinline__
#endif

struct RnGen {
  RnRng r;
  int calls;  // RNG calls of the current distribution draw
  int bad;    // a draw of the current iteration exceeded RN_GEN_BUDGET
};

RN_DEVICE rn_i64 rn_g_d2l(double v) {  // D2L: NaN -> 0, saturating, truncating
  if (v != v) return 0;
  if (v >= 9223372036854775807.0) return (rn_i64)0x7fffffffffffffffLL;
  if (v <= -9223372036854775808.0) return (rn_i64)(-0x7fffffffffffffffLL - 1);
  return (rn_i64)v;
}
RN_DEVICE bool rn_g_uniform(RnGen& g, double& u) {
  if (g.calls >= RN_GEN_BUDGET) return false;
  g.calls++;
  u = rn_uniform(g.r);
  return true;
}
RN_DEVICE bool rn_g_normal(RnGen& g, double& z) {
  if (g.calls >= RN_GEN_BUDGET) return false;
  g.calls++;
  z = rn_normal(g.r);
  return true;
}
RN_DEVICE double rn_g_fail(RnGen& g) {
  g.bad = 1;
  return RN_NAN;
}
#define RN_G_U(x) \
  do {                                            \
    if (!rn_g_uniform(g, x)) return rn_g_fail(g); \
  } while (0)
#define RN_G_N(x) \
  do {                                           \
    if (!rn_g_normal(g, x)) return rn_g_fail(g); \
  } while (0)

// ---- continuous (Continuous.scala) ----
RN_GEN_OP double rn_g_normal_draw(RnGen& g) {  // :63-67
  double z;
  RN_G_N(z);
  return z;
}
RN_GEN_OP double rn_g_cauchy(RnGen& g) {  // :72-77, numerator first
  double a, b;
  RN_G_N(a);
  RN_G_N(b);
  return a / b;
}
RN_GEN_OP double rn_g_laplace(RnGen& g) {  // :85-88
  double u;
  RN_G_U(u);
  u = u - 0.5;
  const double sgn = u > 0.0 ? 1.0 : (u < 0.0 ? -1.0 : u);  // Math.signum
  return sgn * -1 * rn_log(1 - (2 * fabs(u)));
}
RN_GEN_OP double rn_g_uniform_draw(RnGen& g) {
  double u;
  RN_G_U(u);
  return u;
}
RN_DEVICE double rn_g_gamma_mt(RnGen& g, double a) {  // Gamma.standard's generate, :125-144 (the tail recursion as a loop)
  for (;;) {
    const double d = a - 1.0 / 3.0;
    const double c = (1.0 / 3.0) / sqrt(d);
    double x, v, u;
    RN_G_N(x);
    v = 1.0 + c * x;
    while (v <= 0) {
      RN_G_N(x);
      v = 1.0 + c * x;
    }
    const double v3 = v * v * v;
    RN_G_U(u);
    if ((u < 1 - 0.0331 * x * x * x * x) || (rn_log(u) < 0.5 * x * x + d * (1 - v3 + rn_log(v3)))) return d * v3;
  }
}
RN_GEN_OP double rn_g_gamma(RnGen& g, double a) {  // :114-122: for a < 1, u is drawn before the recursive generate
  g.calls = 0;
  if (a < 1) {
    double u;
    RN_G_U(u);
    return rn_g_gamma_mt(g, a + 1) * rn_pow(u, 1.0 / a);
  }
  return rn_g_gamma_mt(g, a);
}
RN_GEN_OP double rn_g_beta(RnGen& g, double a, double b) {  // :162-168: Gamma(a, 1) zip Gamma(b, 1) map x / (x + y)
  const double x = rn_g_gamma(g, a);  // (the Scale(1) injection multiplies by 1.0: the identity)
  if (g.bad) return x;
  const double y = rn_g_gamma(g, b);
  return x / (x + y);
}

// ---- discrete (Discrete.scala); the Long result is returned as a double ----
RN_DEVICE double rn_g_bernoulli(RnGen& g, double p) {  // :43-48
  double u;
  RN_G_U(u);
  return u <= p ? 1.0 : 0.0;
}
RN_DEVICE double rn_g_geometric_draw(RnGen& g, double q) {  // :64-69
  double u;
  RN_G_U(u);
  return (double)rn_g_d2l(floor(rn_log(u) / rn_log(1 - q)));
}
RN_DEVICE double rn_g_poisson_small(RnGen& g, double lambda) {  // :142-153
  const double l = rn_exp(-lambda);
  if (l >= 1.0) return 0.0;
  int k = 0;
  double p = 1.0;
  while (p > l) {
    k += 1;
    double u;
    RN_G_U(u);
    p *= u;
  }
  return (double)(k - 1);
}
RN_DEVICE double rn_g_log_factorial(rn_i64 n) {  // :182-185 ((n + 1) wraps like a Long)
  const double x = (double)(rn_i64)((unsigned long long)n + 1ULL);
  return ((x - 0.5) * rn_log(x)) - x + (0.5 * rn_log(2 * 3.141592653589793));
}
RN_DEVICE double rn_g_poisson_large(RnGen& g, double lambda) {  // :156-178
  const double c = 0.767 - 3.36 / lambda;
  const double beta = 3.141592653589793 / sqrt(3.0 * lambda);
  const double alpha = beta * lambda;
  const double k = rn_log(c) - lambda - rn_log(beta);
  for (;;) {
    double u;
    RN_G_U(u);
    const double x = (alpha - rn_log((1.0 - u) / u)) / beta;
    const rn_i64 n = rn_g_d2l(floor(x + 0.5));
    if (n >= 0) {
      double v;
      RN_G_U(v);
      const double y = alpha - beta * x;
      const double lhs = y + rn_log(v / rn_pow(1.0 + rn_exp(y), 2));
      const double rhs = k + (double)n * rn_log(lambda) - rn_g_log_factorial(n);
      if (lhs <= rhs) return (double)n;
    }
  }
}
RN_DEVICE double rn_g_poisson_draw(RnGen& g, double lambda) {  // :128-134
  return lambda < 30.0 ? rn_g_poisson_small(g, lambda) : rn_g_poisson_large(g, lambda);
}
RN_GEN_OP double rn_g_bernoulli_op(RnGen& g, double p) { g.calls = 0; return rn_g_bernoulli(g, p); }
RN_GEN_OP double rn_g_geometric(RnGen& g, double p) { g.calls = 0; return rn_g_geometric_draw(g, p); }
RN_GEN_OP double rn_g_poisson(RnGen& g, double lambda) { g.calls = 0; return rn_g_poisson_draw(g, lambda); }
// Binomial, :203-228.  s: p, k, p*k, k*p, (k*p*(1-p)).pow(0.5), p + 0 (the first entry of Multinomial's categorical CDF)
RN_GEN_OP double rn_g_binomial(RnGen& g, double p, double k, double pk, double kp, double sd, double cdf0) {
  g.calls = 0;
  if (k >= 100 && k * p <= 10) {  // Poisson(p * k) zip k map x.min(k.toLong)
    const double x = rn_g_poisson_draw(g, pk);
    if (x != x) return x;
    const rn_i64 kl = rn_g_d2l(k), xl = rn_g_d2l(x);
    return (double)(xl < kl ? xl : kl);
  }
  if (k >= 100 && k * p >= 9 && k * (1.0 - p) >= 9) {  // Normal(k * p, sd) zip k map x.toLong.max(0).min(k.toLong)
    double z;
    RN_G_N(z);
    rn_i64 x = rn_g_d2l(z * sd + kp);
    x = x > 0 ? x : 0;
    const rn_i64 kl = rn_g_d2l(k);
    return (double)(x < kl ? x : kl);
  }
  // Multinomial(true -> p, false -> 1 - p, k): categorical.repeat(k.toInt), counting `true`: cdf(true) >= u
  const int n = rn_d2i(k);
  int count = 0;
  for (int i = 0; i < n; i++) {
    double u;
    RN_G_U(u);
    if (cdf0 >= u) count++;
  }
  return (double)count;
}
// NegativeBinomial, :87-108.  s: p, n, 1-p, n*p/(1-p), (n*p).pow(1/2)/(1-p)
RN_GEN_OP double rn_g_negbinomial(RnGen& g, double p, double n, double q, double mean, double sd) {
  g.calls = 0;
  if (p < -100 / n + 1 && p > 100 / n - .25) {  // Normal(mean, sd) map _.toLong.max(0)
    double z;
    RN_G_N(z);
    const rn_i64 x = rn_g_d2l(z * sd + mean);
    return (double)(x > 0 ? x : 0);
  }
  const rn_i64 m = rn_g_d2l(n);  // (1L to n.toLong).map(Geometric(1 - p).get).sum, wrapping like Long
  unsigned long long total = 0;
  for (rn_i64 i = 1; i <= m; i++) {
    const double x = rn_g_geometric_draw(g, q);
    if (x != x) return x;
    total += (unsigned long long)rn_g_d2l(x);
  }
  return (double)(rn_i64)total;
}

// the emitted plan: one draw of one chain.  Slot j of this draw is s[j * ss]; writes RN_MOUT doubles to o; returns at once
// when a distribution draw exceeds the budget (g.bad).
RN_DEVICE void rn_generate(RnGen& g, const double* RN_RESTRICT s, const long long ss, double* RN_RESTRICT o);

// RnGenArgs: rn_gen_args.h.  Chains [0, chains), iterations [t0, t1) of a call of `iterations`; the slot values of those
// iterations are slots[(t - t0) * RN_M * chains + j * chains + c] (rn_k_eval's output, chain-adjacent), the draws go to
// out[(c * iterations + t) * RN_MOUT + .] (Trace.predict's order).
RN_GLOBAL void rn_k_generate(const RnGenArgs A) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= A.chains) return;
  RnRngState st = A.rng[c];
  RnGen g;
  g.r.seed = st.seed48;
  g.r.nng = st.next_gaussian;
  g.r.have = st.have_next;
  g.calls = 0;
  int err = A.err[c];
  long long first = A.err_iter[c];
  for (long long t = A.t0; t < A.t1; t++) {
    double* o = A.out + (c * A.iterations + t) * (long long)RN_MOUT;
    if (!(err & 1)) {
      g.bad = 0;
      rn_generate(g, A.slots + (t - A.t0) * (long long)RN_M * A.chains + c, A.chains, o);
      if (!g.bad) continue;
      err |= 1;  // the chain stops here (see the head of this file)
      first = t;
    }
    for (long long j = 0; j < RN_MOUT; j++) o[j] = RN_NAN;
  }
  st.seed48 = g.r.seed;
  st.next_gaussian = g.r.nng;
  st.have_next = g.r.have;
  A.rng[c] = st;
  A.err[c] = err;
  A.err_iter[c] = first;
}

#endif  // RN_GENERATE_CUH

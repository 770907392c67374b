// rn_optimizer.cuh -- hand-written: batched multi-start MAP optimisation, one thread (or one warp) per start (SURVEY.md 8f-4).
//
// Replaces the loop of Optimizer.lbfgs (rainier-sampler/.../optimizer/Optimizer.scala:6-24) -- `df.update(x)`; negate
// density and gradient; `complete = lb(f, g)` -- together with the reverse-communication L-BFGS it drives
// (rainier-sampler/.../optimizer/LBFGS.java: two-loop recursion :62-190, More-Thuente line search mcsrch :240-383,
// safeguarded step mcstep :431-605).  The reference runs ONE start (x = 0) and crosses the DensityFunction interface once
// per evaluation; here every thread owns one start and runs the whole optimisation -- density, gradient, line search,
// history update -- without leaving the kernel: the emitted rn_density() is inlined, the history (2m vectors) lives in
// thread-local memory (n*(2m+1)+2m doubles; L1-resident for the small models the thread-per-chain shape serves).
//
// Arithmetic follows the reference operation for operation (sequential dot products, the same association in every
// expression, Math.min/max with Java's NaN and signed-zero rules, no FMA contraction in parity mode), so a start is
// bit-identical to `new LBFGS(x, m, eps)` driven by the CPU oracle.  `throw new RuntimeException("dginit")`
// (LBFGS.java:253-254) becomes info bit 1; the reference has no evaluation cap, a kernel needs one (info bit 0).
#ifndef RN_OPTIMIZER_CUH
#define RN_OPTIMIZER_CUH

// Two shapes share this source (like the samplers):
//   RN_BACKEND 0, one THREAD per start: vectors in thread-local memory, every sum sequential -> bit-identical to the oracle.
//   RN_BACKEND 1, one WARP per start (streamed models / many parameters): the start's vectors (x, g, diag and the 2m-vector
//     history) live in the warp's shared-memory slice and are updated lane-strided; dot products are per-lane partial sums
//     + a shuffle butterfly (all lanes hold the same total), scalars and the whole line-search logic are replicated and
//     identical in all lanes, so control flow stays warp-uniform.  Sums become trees -> agreement with the oracle to
//     rounding (and the emitted rn_density() itself sums rows in tree order there), not bit for bit.
//   A lane only ever re-reads vector elements it wrote itself (same striding everywhere); the one cross-lane hand-off is
//   x -> rn_density(), fenced by RN_LB_SYNC().
#ifndef RN_LBFGS_M
#define RN_LBFGS_M 5  // Optimizer.scala:12
#endif
#if RN_BACKEND == 1
#define RN_LB_LANE ((int)(threadIdx.x % RN_G))
#define RN_LB_FOR_N(i, count) for (int i = RN_LB_LANE; i < (count); i += RN_G)
#define RN_LB_REDUCE(s, red) rn_lb_group_sum(s, red)
#define RN_LB_SYNC() RN_SYNC()
#else
#define RN_LB_FOR_N(i, count) for (int i = 0; i < (count); i++)
#define RN_LB_REDUCE(s, red) (s)
#define RN_LB_SYNC()
#endif
#define RN_LB_FOR(i) RN_LB_FOR_N(i, RN_N)
#define RN_LB_W (RN_N * (2 * RN_LBFGS_M + 1) + 2 * RN_LBFGS_M)
#define RN_LB_ISPT (RN_N + 2 * RN_LBFGS_M)
#define RN_LB_IYPT (RN_LB_ISPT + RN_N * RN_LBFGS_M)

#if RN_BACKEND == 1
// Sum over the RN_G = 32*RN_WPC_K threads that own a start; every thread receives the same total.  One warp: shuffle
// butterfly.  K warps (a start whose state is so large that one warp per start would leave the SM nearly empty): the warps'
// totals meet in K doubles of the start's shared-memory slice and are added in one fixed order by every thread.
RN_DEVICE double rn_lb_group_sum(double x, double* red) {
  x = rn_warp_sum(x);
#if RN_WPC_K > 1
  if ((threadIdx.x & 31) == 0) red[(threadIdx.x % RN_G) >> 5] = x;
  RN_SYNC();
  x = red[0];
  for (int k = 1; k < RN_WPC_K; k++) x = x + red[k];
  RN_SYNC();
#else
  (void)red;
#endif
  return x;
}
#endif

RN_DEVICE double rn_jmin(double a, double b) {  // java.lang.Math.min: NaN wins, -0.0 < 0.0
  if (a != a) return a;
  if (b != b) return b;
  if (a == 0.0 && b == 0.0) return (rn_d2ll(a) < 0) ? a : b;
  return a <= b ? a : b;
}
RN_DEVICE double rn_jmax(double a, double b) {
  if (a != a) return a;
  if (b != b) return b;
  if (a == 0.0 && b == 0.0) return (rn_d2ll(a) < 0) ? b : a;
  return a >= b ? a : b;
}
RN_DEVICE double rn_max3(double a, double b, double c) { return a < b ? (b < c ? c : b) : (a < c ? c : a); }

struct RnLbfgs {
  double *x, *diag, *w;  // [RN_N], [RN_N], [RN_LB_W]: thread-local arrays (backend 0) or the start's shared-memory slice
  double* red;           // backend 1 with K warps per start: K doubles of cross-warp reduction scratch
  double eps, stp, stp1, ys, yy;
  int iter, point, npt, info, nfev, bound;
  // line-search state
  double dginit, dgtest, finit, stmin, stmax, width, width1, fx, dgx, fy, dgy, stx, sty;
  int infoc, brackt, stage1;
};

RN_DEVICE double rn_lb_dot(const RnLbfgs& S, const double* a, const double* b) {  // ddot, unit strides: a sequential sum (backend 0)
  double s = 0.0;
  RN_LB_FOR(i) s = s + a[i] * b[i];
  (void)S;
  return RN_LB_REDUCE(s, S.red);
}
RN_DEVICE void rn_lb_axpy(double da, const double* a, double* y) {  // daxpy; a zero factor leaves y untouched
  if (da == 0.0) return;
  RN_LB_FOR(i) y[i] = y[i] + da * a[i];
}

RN_DEVICE void rn_lb_init(RnLbfgs& S, double* x, double* diag, double* w, double* red, double eps) {
  S.red = red;
  S.x = x;
  S.diag = diag;
  S.w = w;
  S.eps = eps;
  RN_LB_FOR_N(i, RN_LB_W) S.w[i] = 0.0;
  RN_LB_FOR(i) S.diag[i] = 1.0;
  S.iter = S.point = S.npt = S.info = S.nfev = S.bound = 0;
  S.stp = S.stp1 = S.ys = S.yy = 0.0;
  S.dginit = S.dgtest = S.finit = S.stmin = S.stmax = S.width = S.width1 = 0.0;
  S.fx = S.dgx = S.fy = S.dgy = S.stx = S.sty = 0.0;
  S.infoc = S.brackt = S.stage1 = 0;
}

// mcstep: new trial step from the interval [stx, sty] and the trial point (stp, fp, dp).  fx/dx/fy/dy are the caller's
// (possibly modified-function) copies.
RN_DEVICE void rn_lb_step(RnLbfgs& S, double& fx, double& dx, double& fy, double& dy, const double fp, const double dp) {
  double stp = S.stp, stx = S.stx, sty = S.sty;
  S.infoc = 0;
  if ((S.brackt && (stp <= rn_jmin(stx, sty) || stp >= rn_jmax(stx, sty))) || dx * (stp - stx) >= 0.0 || S.stmax < S.stmin) return;
  const double sgnd = dp * (dx / fabs(dx));
  double theta, s, gamma, p, q, r, stpc, stpq, stpf;
  bool bound;
  if (fp > fx) {  // higher function value: the minimum is bracketed
    S.infoc = 1;
    bound = true;
    theta = 3 * (fx - fp) / (stp - stx) + dx + dp;
    s = rn_max3(fabs(theta), fabs(dx), fabs(dp));
    const double ts = theta / s;
    gamma = s * sqrt(ts * ts - (dx / s) * (dp / s));
    if (stp < stx) gamma = -gamma;
    p = (gamma - dx) + theta;
    q = ((gamma - dx) + gamma) + dp;
    r = p / q;
    stpc = stx + r * (stp - stx);
    stpq = stx + ((dx / ((fx - fp) / (stp - stx) + dx)) / 2) * (stp - stx);
    stpf = (fabs(stpc - stx) < fabs(stpq - stx)) ? stpc : stpc + (stpq - stpc) / 2;
    S.brackt = 1;
  } else if (sgnd < 0.0) {  // lower value, derivatives of opposite sign: bracketed
    S.infoc = 2;
    bound = false;
    theta = 3 * (fx - fp) / (stp - stx) + dx + dp;
    s = rn_max3(fabs(theta), fabs(dx), fabs(dp));
    const double ts = theta / s;
    gamma = s * sqrt(ts * ts - (dx / s) * (dp / s));
    if (stp > stx) gamma = -gamma;
    p = (gamma - dp) + theta;
    q = ((gamma - dp) + gamma) + dx;
    r = p / q;
    stpc = stp + r * (stx - stp);
    stpq = stp + (dp / (dp - dx)) * (stx - stp);
    stpf = (fabs(stpc - stp) > fabs(stpq - stp)) ? stpc : stpq;
    S.brackt = 1;
  } else if (fabs(dp) < fabs(dx)) {  // lower value, same sign, derivative shrinks
    S.infoc = 3;
    bound = true;
    theta = 3 * (fx - fp) / (stp - stx) + dx + dp;
    s = rn_max3(fabs(theta), fabs(dx), fabs(dp));
    const double ts = theta / s;
    gamma = s * sqrt(rn_jmax(0.0, ts * ts - (dx / s) * (dp / s)));
    if (stp > stx) gamma = -gamma;
    p = (gamma - dp) + theta;
    q = (gamma + (dx - dp)) + gamma;
    r = p / q;
    if (r < 0.0 && gamma != 0.0)
      stpc = stp + r * (stx - stp);
    else if (stp > stx)
      stpc = S.stmax;
    else
      stpc = S.stmin;
    stpq = stp + (dp / (dp - dx)) * (stx - stp);
    if (S.brackt)
      stpf = (fabs(stp - stpc) < fabs(stp - stpq)) ? stpc : stpq;
    else
      stpf = (fabs(stp - stpc) > fabs(stp - stpq)) ? stpc : stpq;
  } else {  // lower value, same sign, derivative does not shrink
    S.infoc = 4;
    bound = false;
    if (S.brackt) {
      theta = 3 * (fp - fy) / (sty - stp) + dy + dp;
      s = rn_max3(fabs(theta), fabs(dy), fabs(dp));
      const double ts = theta / s;
      gamma = s * sqrt(ts * ts - (dy / s) * (dp / s));
      if (stp > sty) gamma = -gamma;
      p = (gamma - dp) + theta;
      q = ((gamma - dp) + gamma) + dy;
      r = p / q;
      stpc = stp + r * (sty - stp);
      stpf = stpc;
    } else if (stp > stx) {
      stpf = S.stmax;
    } else {
      stpf = S.stmin;
    }
  }
  if (fp > fx) {
    sty = stp;
    fy = fp;
    dy = dp;
  } else {
    if (sgnd < 0.0) {
      sty = stx;
      fy = fx;
      dy = dx;
    }
    stx = stp;
    fx = fp;
    dx = dp;
  }
  stpf = rn_jmin(S.stmax, stpf);
  stpf = rn_jmax(S.stmin, stpf);
  stp = stpf;
  if (S.brackt && bound) {
    if (sty > stx)
      stp = rn_jmin(stx + 0.66 * (sty - stx), stp);
    else
      stp = rn_jmax(stx + 0.66 * (sty - stx), stp);
  }
  S.stp = stp;
  S.stx = stx;
  S.sty = sty;
}

// mcsrch, reverse communication: S.info == -1 on return means "evaluate at S.x and call again".  Returns false when the
// search direction is not a descent direction (the reference throws).
RN_DEVICE bool rn_lb_search(RnLbfgs& S, const double f, const double* g) {
  const double GTOL = 0.9, STPMIN = 1e-20, STPMAX = 1e20, XTOL = 1e-16, FTOL = 0.0001, P5 = 0.5, P66 = 0.66, XTRAPF = 4;
  const int MAXFEV = 20;
  const double* dir = S.w + RN_LB_ISPT + S.point * RN_N;
  if (S.info != -1) {
    S.infoc = 1;
    S.dginit = rn_lb_dot(S, g, dir);
    if (S.dginit >= 0) return false;
    S.brackt = 0;
    S.stage1 = 1;
    S.nfev = 0;
    S.finit = f;
    S.dgtest = FTOL * S.dginit;
    S.width = STPMAX - STPMIN;
    S.width1 = S.width / P5;
    RN_LB_FOR(j) S.diag[j] = S.x[j];
    S.stx = 0;
    S.fx = S.finit;
    S.dgx = S.dginit;
    S.sty = 0;
    S.fy = S.finit;
    S.dgy = S.dginit;
  }
  for (;;) {
    if (S.info != -1) {
      if (S.brackt) {
        S.stmin = rn_jmin(S.stx, S.sty);
        S.stmax = rn_jmax(S.stx, S.sty);
      } else {
        S.stmin = S.stx;
        S.stmax = S.stp + XTRAPF * (S.stp - S.stx);
      }
      S.stp = rn_jmax(S.stp, STPMIN);
      S.stp = rn_jmin(S.stp, STPMAX);
      if ((S.brackt && (S.stp <= S.stmin || S.stp >= S.stmax)) || S.nfev >= MAXFEV - 1 || S.infoc == 0 ||
          (S.brackt && S.stmax - S.stmin <= XTOL * S.stmax))
        S.stp = S.stx;
      RN_LB_FOR(j) S.x[j] = S.diag[j] + S.stp * dir[j];
      S.info = -1;
      return true;
    }
    S.info = 0;
    S.nfev = S.nfev + 1;
    const double dg = rn_lb_dot(S, g, dir);
    const double ftest1 = S.finit + S.stp * S.dgtest;
    if ((S.brackt && (S.stp <= S.stmin || S.stp >= S.stmax)) || S.infoc == 0) S.info = 6;
    if (S.stp == STPMAX && f <= ftest1 && dg <= S.dgtest) S.info = 5;
    if (S.stp == STPMIN && (f > ftest1 || dg >= S.dgtest)) S.info = 4;
    if (S.nfev >= MAXFEV) S.info = 3;
    if (S.brackt && S.stmax - S.stmin <= XTOL * S.stmax) S.info = 2;
    if (f <= ftest1 && fabs(dg) <= GTOL * (-S.dginit)) S.info = 1;
    if (S.info != 0) return true;
    if (S.stage1 && f <= ftest1 && dg >= rn_jmin(FTOL, GTOL) * S.dginit) S.stage1 = 0;
    if (S.stage1 && f <= S.fx && f > ftest1) {  // first stage: work on the modified function
      const double fm = f - S.stp * S.dgtest;
      double fxm = S.fx - S.stx * S.dgtest;
      double fym = S.fy - S.sty * S.dgtest;
      const double dgm = dg - S.dgtest;
      double dgxm = S.dgx - S.dgtest;
      double dgym = S.dgy - S.dgtest;
      rn_lb_step(S, fxm, dgxm, fym, dgym, fm, dgm);
      S.fx = fxm + S.stx * S.dgtest;
      S.fy = fym + S.sty * S.dgtest;
      S.dgx = dgxm + S.dgtest;
      S.dgy = dgym + S.dgtest;
    } else {
      rn_lb_step(S, S.fx, S.dgx, S.fy, S.dgy, f, dg);
    }
    if (S.brackt) {
      if (fabs(S.sty - S.stx) >= P66 * S.width1) S.stp = S.stx + P5 * (S.sty - S.stx);
      S.width1 = S.width;
      S.width = fabs(S.sty - S.stx);
    }
  }
}

// LBFGS.apply: 0 = evaluate at S.x and call again, 1 = converged, 2 = "dginit"
RN_DEVICE int rn_lb_apply(RnLbfgs& S, const double f, const double* g) {
  double* w = S.w;
  bool whole = false;
  if (S.iter == 0) {
    RN_LB_FOR(i) w[RN_LB_ISPT + i] = -g[i] * S.diag[i];
    const double gnorm = sqrt(rn_lb_dot(S, g, g));
    S.stp1 = 1 / gnorm;
    whole = true;
  }
  for (;;) {
    if (whole) {
      S.iter = S.iter + 1;
      S.info = 0;
      S.bound = S.iter - 1;
      if (S.iter != 1) {
        if (S.iter > RN_LBFGS_M) S.bound = RN_LBFGS_M;
        S.ys = rn_lb_dot(S, w + RN_LB_IYPT + S.npt, w + RN_LB_ISPT + S.npt);
        S.yy = rn_lb_dot(S, w + RN_LB_IYPT + S.npt, w + RN_LB_IYPT + S.npt);
        const double h0 = S.ys / S.yy;
        RN_LB_FOR(i) S.diag[i] = h0;
        int cp = S.point;
        if (S.point == 0) cp = RN_LBFGS_M;
        w[RN_N + cp - 1] = 1 / S.ys;
        RN_LB_FOR(i) w[i] = -g[i];
        cp = S.point;
        for (int k = 0; k < S.bound; k++) {  // backward pass over the history
          cp = cp - 1;
          if (cp == -1) cp = RN_LBFGS_M - 1;
          const double sq = rn_lb_dot(S, w + RN_LB_ISPT + cp * RN_N, w);
          const int inmc = RN_N + RN_LBFGS_M + cp;
          w[inmc] = w[RN_N + cp] * sq;
          rn_lb_axpy(-w[inmc], w + RN_LB_IYPT + cp * RN_N, w);
        }
        RN_LB_FOR(i) w[i] = S.diag[i] * w[i];
        for (int k = 0; k < S.bound; k++) {  // forward pass
          const double yr = rn_lb_dot(S, w + RN_LB_IYPT + cp * RN_N, w);
          double beta = w[RN_N + cp] * yr;
          beta = w[RN_N + RN_LBFGS_M + cp] - beta;
          rn_lb_axpy(beta, w + RN_LB_ISPT + cp * RN_N, w);
          cp = cp + 1;
          if (cp == RN_LBFGS_M) cp = 0;
        }
        RN_LB_FOR(i) w[RN_LB_ISPT + S.point * RN_N + i] = w[i];
      }
      S.nfev = 0;
      S.stp = 1;
      if (S.iter == 1) S.stp = S.stp1;
      RN_LB_FOR(i) w[i] = g[i];
    }
    if (!rn_lb_search(S, f, g)) return 2;
    if (S.info == -1) return 0;
    S.npt = S.point * RN_N;
    RN_LB_FOR(i) {
      w[RN_LB_ISPT + S.npt + i] = S.stp * w[RN_LB_ISPT + S.npt + i];
      w[RN_LB_IYPT + S.npt + i] = g[i] - w[i];
    }
    S.point = S.point + 1;
    if (S.point == RN_LBFGS_M) S.point = 0;
    const double gnorm = sqrt(rn_lb_dot(S, g, g));
    double xnorm = sqrt(rn_lb_dot(S, S.x, S.x));
    xnorm = rn_jmax(1.0, xnorm);
    if (gnorm / xnorm <= S.eps) return 1;
    whole = true;
  }
}

#define S_X_ARRAY(a) (*reinterpret_cast<double (*)[RN_N]>(a))  // the thread-per-chain density takes array references
// =============================================================================================================
// rn_k_lbfgs: x0 [N][starts] (NULL: all starts at 0, the reference's only start) -> x [N][starts], f [starts] = -density
// at x, info [starts] (bit 0 evaluation cap reached, bit 1 "dginit", bit 2 lookup error), evals [starts]
// =============================================================================================================
#if RN_BACKEND == 1
// slices of one start, by placement (RN_WPC_PLACE, as for the samplers: rn_sampler_wpc.cuh):
//   0  shared: x | gradient | g = -gradient | diag | w | scratch of the emitted density | K reduction slots
//   1  global: x | gradient | g | diag | w | density scratch  shared: K reduction slots | the density's reduction slots
#if RN_WPC_PLACE == 0
#define RN_OPT_SMEM_DOUBLES (4 * RN_N + RN_LB_W + RN_WPC_SCRATCH + RN_WPC_K)
#define RN_OPT_GLOBAL_DOUBLES 0
#else
#define RN_OPT_SMEM_DOUBLES (RN_WPC_K + RN_WPC_RED_DOUBLES)
#define RN_OPT_GLOBAL_DOUBLES ((4LL * RN_N + RN_LB_W + RN_WPC_SCRATCH + 15) / 16 * 16)
#endif
#ifdef RN_OPT_EXPECT_SMEM  // what rn_runtime.cpp:get_opt_kernel allocates per start; a mismatch is a slice overrun on the device
static_assert(RN_OPT_SMEM_DOUBLES == RN_OPT_EXPECT_SMEM, "rn_optimize: launcher and kernel disagree on the shared-memory slice of a start");
#endif
#ifdef RN_OPT_EXPECT_GLOBAL
static_assert(RN_OPT_GLOBAL_DOUBLES == RN_OPT_EXPECT_GLOBAL, "rn_optimize: launcher and kernel disagree on the global-memory slice of a start");
#endif
#ifdef RN_HOST_EMULATION
static double rn_smem[1 << 17];  // one emulated start at a time
#if RN_WPC_PLACE != 0  // ... with its global slice here (tests/host_emulation.py passes no slice array)
static double rn_emu_wpc_state[(size_t)RN_OPT_GLOBAL_DOUBLES * 8];
#endif
#else
extern __shared__ __align__(128) double rn_smem[];
#endif
#endif

RN_GLOBAL void rn_k_lbfgs(const RnOptArgs A) {
#if RN_BACKEND == 1
  const int c = (int)((blockIdx.x * blockDim.x + threadIdx.x) / RN_G);
  if (c >= A.starts) return;  // the whole group leaves together
  double* sbase = rn_smem + (size_t)RN_GROUP * RN_OPT_SMEM_DOUBLES;
#if RN_WPC_PLACE == 0
  double* base = sbase;
  double* scr = base + 4 * RN_N + RN_LB_W;
  double* red = scr + RN_WPC_SCRATCH;
#else
#ifdef RN_HOST_EMULATION
  double* base = rn_emu_wpc_state + (size_t)RN_GROUP * (size_t)RN_OPT_GLOBAL_DOUBLES;
#else
  double* base = A.wpc_state + (size_t)c * (size_t)RN_OPT_GLOBAL_DOUBLES;
#endif
  double* scr = base + 4 * RN_N + RN_LB_W;
  double* red = sbase;
#endif
  double *x = base, *grad = base + RN_N, *g = base + 2 * RN_N, *diag = base + 3 * RN_N, *w = base + 4 * RN_N;
  RnTma tma;  // the CTA-shared tile pipeline stays off: starts take different numbers of evaluations
  tma.on = 0;
  tma.seq = 0;
  tma.nthreads = 0;
  tma.stage = nullptr;
  tma.full = nullptr;
#else
  const int c = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (c >= A.starts) return;
  double x[RN_N], grad[RN_N], g[RN_N], diag[RN_N], w[RN_LB_W];
  double* red = nullptr;
#endif
  RnLbfgs S;
  rn_lb_init(S, x, diag, w, red, A.eps);
  RN_LB_FOR(i) x[i] = A.x0 ? A.x0[(size_t)i * A.starts + c] : 0.0;
  int evals = 0, info = 0, err = 0;
  double f = RN_NAN;
  for (;;) {
    if (evals >= A.max_evals) {
      info = 1;
      break;
    }
    double dens;
    RN_LB_SYNC();  // x was written lane-strided; the density reads all of it in every lane
#if RN_BACKEND == 1
    rn_density(x, dens, grad, scr RN_DENSITY_RED(red + RN_WPC_K), A.data, err, tma);  // df.update(x), Optimizer.scala:15 (ends with a group barrier)
#else
    rn_density(S_X_ARRAY(x), dens, S_X_ARRAY(grad), A.data, err);  // df.update(x), Optimizer.scala:15
#endif
    evals++;
    f = dens * -1;
    RN_LB_FOR(i) g[i] = grad[i] * -1;
    const int r = rn_lb_apply(S, f, g);
    if (r == 1) break;
    if (r == 2) {
      info = 2;
      break;
    }
  }
  if (err & 1) info |= 4;
  RN_LB_FOR(i) A.x[(size_t)i * A.starts + c] = x[i];
#if RN_BACKEND == 1
  if (RN_LB_LANE != 0) return;
#endif
  A.f[c] = f;
  A.info[c] = info;
  A.evals[c] = evals;
}

#endif  // RN_OPTIMIZER_CUH

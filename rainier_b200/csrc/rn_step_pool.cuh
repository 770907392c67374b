// rn_step_pool.cuh -- pooled step-size adaptation (rn_config.step_adaptation == RN_ADAPT_POOLED; an extension, not
// reference semantics).  Compiled in only when the emitter defines RN_STEP_POOL, so per-chain modules are unchanged.
//
// Let C be the number of chains over all ranks.  Every quantity that crosses chains is an exact integer sum, so the
// result depends neither on chain order, CTA shape, the order of the atomics nor on how chains are split over ranks:
//   init    chain c's findReasonableStepSize ends at 2^k_c (k_c counted, clamped to [-1075, 1024]);
//           K = sum k_c, eps0 = exp(ln2 * K / C); every chain's DualAvg becomes DualAvg.apply(delta, eps0)
//   warmup  iteration t: q_c = rint(exp(a_c) * 2^32), Q_t = sum q_c, P_t = Q_t / (2^32 C); every chain applies
//           DualAvg.update with newAcceptanceProb = P_t (DualAvg.scala:58-77), then -- if a mass window closed --
//           stepSizeTuner.reset() (Driver.scala:67-80), so every chain's copy of the DualAvg state is bit-identical.
// In this mode a warmup launch covers one iteration: the sampler kernels add their terms into the iteration's int64 slot
// (rn_pool_add), the host all-reduces the slot across ranks, and rn_k_step_pool applies the update
// (rn_step_pool_apply.cuh).  The emitter writes this file after the prelude and rn_step_pool_apply.cuh after the sampler
// kernels, into RN_STEP_POOL modules only.
#ifndef RN_STEP_POOL_CUH
#define RN_STEP_POOL_CUH

#define RN_POOL_Q_SCALE 4294967296.0 /* 2^32: quantum of the pooled acceptance probability */

// rint(p * 2^32) of this chain's acceptance probability p = exp(a) in [0, 1]
RN_DEVICE rn_i64 rn_pool_quantise(double p) { return (rn_i64)rint(p * RN_POOL_Q_SCALE); }

// *slot += v, exactly.  The converged lanes of the warp sum their terms first (three 22-bit limbs: a sum of 32 limbs fits 32
// bits; two's complement makes the limb sum of signed terms exact modulo 2^64) and one of them issues the atomic.  Any split
// of the chains into atomics gives the same integer.
RN_DEVICE void rn_pool_add(rn_i64* slot, rn_i64 v) {
#ifdef RN_HOST_EMULATION
  __atomic_fetch_add(slot, v, __ATOMIC_RELAXED);  // emulated warps of one CTA run as concurrent host threads
#else
  const unsigned long long u = (unsigned long long)v;
  const unsigned mask = __activemask();
  const unsigned l0 = __reduce_add_sync(mask, (unsigned)(u & 0x3FFFFFull));
  const unsigned l1 = __reduce_add_sync(mask, (unsigned)((u >> 22) & 0x3FFFFFull));
  const unsigned l2 = __reduce_add_sync(mask, (unsigned)(u >> 44));
  if ((int)(threadIdx.x & 31) == __ffs(mask) - 1)
    atomicAdd((unsigned long long*)slot, (unsigned long long)l0 + ((unsigned long long)l1 << 22) + ((unsigned long long)l2 << 44));
#endif
}

#endif  // RN_STEP_POOL_CUH

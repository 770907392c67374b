// rn_gen_args.h -- kernel argument block of rn_k_generate (rn_generate.cuh), shared verbatim by the host runtime
// (rn_runtime.cpp) and the device code (embedded in front of rn_generate.cuh).  Kept apart from rn_args.h so that the
// sources of the other flavours do not change.  Plain C: only int / long long / double / pointers.
#ifndef RN_GEN_ARGS_H
#define RN_GEN_ARGS_H

// java.util.Random state, laid out as rn_rng_state (rainier_cuda.h)
struct RnRngState {
  long long seed48;
  double next_gaussian;
  int have_next;
  int reserved;
};

// posterior-predictive draws, one thread per chain
struct RnGenArgs {
  const double* slots;  // [t1 - t0][RN_M][chains]: the plan's slot values (rn_k_eval's output)
  double* out;          // [chains][iterations][RN_MOUT]
  RnRngState* rng;      // [chains], read at the start of a launch and written back at its end
  int* err;             // [chains] bit 0: a draw exceeded RN_GEN_BUDGET RNG calls
  long long* err_iter;  // [chains] iteration of the first such draw
  long long chains, t0, t1, iterations;
};

#endif

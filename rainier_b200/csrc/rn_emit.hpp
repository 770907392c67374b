// rn_emit.hpp -- CUDA source emitter: Program -> one self-contained translation unit (prelude + emitted
// rn_density() + hand-written sampler kernels).  Replaces the reference's JVM bytecode emitter
// (rainier-compute/.../ir/CompiledFunction.scala:42-120 and the *Generator classes).
#pragma once
#include <string>

#include "rn_graph.hpp"

namespace rn {

struct EmitOptions {
  int backend = 0;        // 0 = thread per chain, 1 = warp per chain (rows across lanes)
  bool fast_math = false; // strength-reduce constant powers beyond what Math.pow itself special-cases
  int mass_max = 0;       // 0 identity only, 1 + diagonal, 2 + dense
  bool enable_ehmc = false;
  bool step_pool = false; // pooled step-size adaptation (rn_sampler_common.cuh): RN_STEP_POOL kernels
  bool mass_pool = false; // pooled dense mass windows (rn_sampler_common.cuh): RN_MASS_POOL kernels
  bool traj_pool = false; // pooled EHMC trajectory lengths (rn_sampler_common.cuh): RN_TRAJ_POOL kernels
  bool tpc_restore = false; // thread per chain: the iteration's restore point in shared memory (RN_TS_RESTORE, rn_sampler.cuh)
  int tma_stages = 0;     // warp per chain: shared-memory stages of the CTA-shared data-tile pipeline (0 = off)
  int wpc_k = 1;          // warp per chain: warps owning one chain (1, 2, 4 or 8; > 1 for chains with a large state)
  int wpc_place = 0;      // warp per chain: where a chain's state lives (RN_WPC_PLACE): 0 all in shared memory, 1 the chain
                          // vectors and the density scratch in global memory (the reduction slots stay in shared memory)
  std::vector<uint64_t> target_base;  // per target: element offset of its tile-major [tile][column][pitch] block in the data buffer
  std::vector<int> target_pitch;      // per target: doubles between consecutive columns of a tile (32 rows + padding; empty = 32).
                                      // 36 where the chain-batched DMMA path may run: X^T fragments are then bank-conflict free
  bool mma = false;       // warp per chain: chain-batched fp64 tensor-core contraction of the row bodies' dot products (see
                          // Emitter::mma_block); needs full CTAs of mma_chains chains (= warps, wpc_k == 1)
  int expect_slice_doubles = 0;  // the launcher's shared-memory doubles per chain / start (checked against the kernel's own layout at compile time)
  long long expect_global_doubles = -1;  // the launcher's global-memory state doubles per chain / start (likewise; -1 = unchecked)
  int interleave = 8;     // independent dataflow components of a row body (unrolled observations) emitted round-robin at a time
  int mma_chains = 8;     // 8 or 16: chains (warps) per CTA on that path -- 16 = two groups of 8 chains whose warps pair up on
                          // a dot's column block (twice the warps per SM for the same shared memory)
  int pitch(size_t t) const { return t < target_pitch.size() && target_pitch[t] > 0 ? target_pitch[t] : 32; }
};
// pitch a model should be packed with: 36 for streamed targets whose row body holds parameter x column dot products
std::vector<int> default_pitches(const Program& P);

// the generated rn_density() only
std::string emit_density(const Program& P, const EmitOptions& opt);
// full translation unit
std::string emit_source(const Program& P, const EmitOptions& opt);
// function flavour (Program from build_function): prelude + emitted rn_function() + rn_function.cuh (rn_k_eval); only
// opt.fast_math is read
std::string emit_function_source(const Program& P, const EmitOptions& opt);
// generator flavour (build_generator): the function flavour's rn_function() + rn_k_eval (the slots), rn_generate.cuh and the
// plan emitted as straight-line rn_generate() (REPEAT as a counted loop).  Parity math only.
std::string emit_generator_source(const Program& P, const GeneratorPlan& G);
// optimizer flavour: prelude + emitted thread-per-chain rn_density() + rn_optimizer.cuh (rn_k_lbfgs, `history` = the m of
// new LBFGS(x, m, eps)); reads opt.fast_math and opt.target_base
std::string emit_optimizer_source(const Program& P, const EmitOptions& opt, int history);
// shared-memory needs of the warp-per-chain kernels: doubles per warp (chain vectors + density scratch) and doubles of
// the largest data tile (n_cols * 32 over the streamed targets; 0 when nothing is streamed)
struct WpcSizes {
  int per_warp_doubles = 0;  // per CHAIN (its wpc_k warps share the slice), shared memory in placement opt.wpc_place:
                             // 0 vector_doubles + scratch_doubles, 1 red_doubles
  long long global_doubles = 0;  // per chain in global memory (RN_WPC_GLOBAL_DOUBLES): 0, or vectors + scratch; 128-byte multiple
  int vector_doubles = 0;    // the sampler's chain vectors (q, p, gradient, mass, EHMC snapshot, dense work vectors)
  int scratch_doubles = 0;   // the emitted density's part of it (RN_WPC_SCRATCH): tables, scatter slots, reduction scratch
  int red_doubles = 0;       // the cross-warp reduction slots inside that scratch (RN_WPC_RED_DOUBLES; 0 when wpc_k == 1)
  int tile_doubles = 0;
  bool mma_ok = false;       // every streamed target with full tiles can take the chain-batched DMMA path
  int mma_shared_doubles = 0;  // CTA-shared doubles of that path: 8 per-warp column-block regions + the reduction scratch
  int reg_accumulators = 0;    // accumulators the row bodies keep in registers (decides the row functions' default, see rn_emit.cpp)
};
WpcSizes wpc_sizes(const Program& P, const EmitOptions& opt);

}  // namespace rn

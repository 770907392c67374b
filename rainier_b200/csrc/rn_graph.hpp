// rn_graph.hpp -- the frozen Real DAG as the CUDA emitter sees it.
//
// Input: an RIR container (include/rainier_rir.h), i.e. the flat form of what the reference hands to its
// bytecode emitter (rainier-compute/.../compute/Compiler.scala:22-30 -> ir/CompiledFunction.scala:42-120).
// Output: a `Program`: straight-line SSA split into the regions the fused kernel needs
//   INV_FWD   nodes that depend on parameters/constants only          (evaluated once per gradient)
//   ROW_FWD_t nodes that depend on target t's columns                  (evaluated once per row of t)
//   ROW_BWD_t per-row reverse sweep of target t (adjoint mode only)
//   INV_BWD   reverse sweep through the invariant part (adjoint mode only)
// plus the accumulator slots that connect them.
//
// Two gradient modes:
//   symbolic : the RIR carries the reference's own symbolic gradient outputs (compute/Gradient.scala:8-69);
//              every target has n+1 outputs that are accumulated exactly like ir/DataFunction.scala:48-84.
//   adjoint  : the RIR carries primal outputs only; adjoints are derived here by reverse mode over the SSA
//              (rules mirror compute/Gradient.scala:71-152 so values agree to rounding), with a two-level
//              sweep so that a Lookup over a large parameter table becomes a scatter-add instead of the
//              reference's O(table) one-hot columns (SURVEY.md 7.3-3).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/rainier_rir.h"

namespace rn {

enum Kind : uint8_t {
  K_INPUT = 0,   // a = input index (parameter or column)
  K_CONST = 1,   // value
  K_UNARY = 2,   // op = RIR_U_* or U_NEG..; a
  K_BINARY = 3,  // op = RIR_B_*; a, b
  K_LOOKUP = 4,  // a = index, b = offset in lookup_refs, c = len, d = low
  K_SELEQ = 5,   // (d2i(val[a]) == d) ? val[b] : val[c]          (adjoint of Lookup)
  K_ACC = 6,     // reads accumulator slot a (total over rows/targets)  (adjoint mode, INV_BWD region)
};
enum ExtUnary : uint8_t { U_NEG = 32, U_RECIP = 33, U_SQRT = 34 };

enum Region : uint8_t { R_INV_FWD = 0, R_ROW_FWD = 1, R_ROW_BWD = 2, R_INV_BWD = 3 };

struct Node {
  uint8_t kind = K_CONST;
  uint8_t op = 0;
  uint8_t region = R_INV_FWD;
  int32_t target = -1;  // for ROW_* regions
  int32_t a = 0, b = 0, c = 0, d = 0;
  double value = 0.0;
};

// `acc[slot] += val[node]` executed once per row of `target` (or once, for data-free targets)
struct AccStmt {
  int32_t slot;
  int32_t node;
};
// dynamic scatter: `acc[slot_base + (d2i(val[index]) - low)] += val[node]`
struct ScatterStmt {
  int32_t slot_base, len, low;
  int32_t index_node;
  int32_t node;
};

// A row-variant dot product `base + sum_j q[param_j] * column_j` -- the Translator's left fold of a `Line` whose
// coefficients are observation columns (compute/Translator.scala:91-125), e.g. x.dot(betas) of a regression.  These are
// the places where the frozen DAG "really is a dense mat-vec" (over all rows: X*beta; over all chains: a GEMM), the
// candidates of the chain-batched DMMA contraction (DESIGN.md 5b-1).  Found by find_dots(); analysis only so far.
struct DotInfo {
  int32_t node = -1;                 // the ADD node holding the complete sum
  int32_t base = -1;                 // first operand of the fold when it is not itself a param*column product, else -1
  std::vector<int32_t> params;       // parameter index of every term, in fold order
  std::vector<int32_t> columns;      // column input index of every term
};

struct TargetInfo {
  uint64_t n_rows = 0;
  uint32_t first_input = 0, n_cols = 0;
  std::vector<int32_t> outputs;        // node ids (n+1 in symbolic mode, 1 in adjoint mode)
  std::vector<int32_t> row_fwd;        // ROW_FWD nodes, topological
  std::vector<int32_t> row_bwd;        // ROW_BWD nodes, emission order
  std::vector<AccStmt> row_acc;        // per-row accumulations
  std::vector<ScatterStmt> row_scatter;
  std::vector<DotInfo> dots;           // maximal param x column dot products of the row body (>= 2 terms)
  bool streamed() const { return n_cols > 0 && n_rows > 0; }
};

struct Program {
  uint32_t n_params = 0, n_inputs = 0;
  bool symbolic = true;
  std::vector<Node> nodes;
  std::vector<int32_t> lookup_refs;
  std::vector<TargetInfo> targets;
  std::vector<int32_t> inv_fwd;        // topological
  std::vector<AccStmt> inv_acc;        // accumulations done once (data-free targets), in target order
  std::vector<int32_t> inv_bwd;        // emission order (adjoint mode)
  // accumulator slots.  symbolic: slots [0, n+1) = DataFunction's outputs.  adjoint: slot 0 = density, slots
  // >=1 are frontier adjoints; grad_nodes[i] is the INV_BWD node holding d/dq_i.
  int32_t n_slots = 0;
  std::vector<int32_t> grad_nodes;
  std::vector<uint8_t> slot_row_accumulated;  // slot receives per-row contributions (needs cross-lane reduce)
  bool has_lookup = false;                    // any K_LOOKUP / K_SELEQ / scatter (error flag needed)
  // function flavour (RIR_FLAG_FUNCTION, build_function): the m output nodes of Compiler.compile(inputs, outputs);
  // every needed node sits in inv_fwd, there are no targets, slots or gradients
  std::vector<int32_t> fn_outputs;
  // static op counts per gradient evaluation (for the roofline; DESIGN.md): fp64 adds/muls/fmas are counted
  // as flops, transcendental calls separately.
  struct Counts {
    double flops_inv = 0, special_inv = 0;
    std::vector<double> flops_row, special_row;  // per target, per row
  } counts;
};

// returns empty string on success, else an error message
std::string build_program(const void* rir, size_t len, bool want_adjoint, bool fast_math, Program& out);

// Separability analysis of the streamed targets (analysis only; DESIGN.md 5b-4, SURVEY.md 8f-5): can the row sum of a
// target's primal output be written as sum_k S_k * p_k(parameters) with S_k = sum over rows of a product of at most
// `max_degree` column-only sub-expressions ("atoms")?  That is the shape the reference's inliner folds into constants on the
// JVM (compute/Target.scala:136-207 decides, compute/PartialEvaluator.scala:86-97 folds) -- here decided on the SSA form by
// carrying a polynomial over column-only atoms through ADD / SUB / MUL / constant powers and refusing any other operation on
// a node that mixes parameters and columns (the reference's `nonlinearOp` on a `combination`).  More general than the
// reference's rule: squares are expanded regardless of the number of terms (the reference stops at 5 additive terms,
// compute/LogLineOps.scala:43-66), so a Gaussian regression on any number of covariates is separable: its atoms are the
// entries of X^T X, X^T y and y^T y.
struct SeparableInfo {
  int streamed_targets = 0;
  int separable_targets = 0;
  int64_t atoms = 0;          // distinct products of column-only nodes over the separable targets (the S_k to reduce)
  int64_t rows_removed = 0;   // rows that would no longer be streamed per gradient evaluation
};
SeparableInfo analyze_separable(const Program& P, int max_degree = 2, int max_atoms = 4096);

// RIR_FLAG_FUNCTION containers: Compiler.compile(inputs, outputs): CompiledFunction (compute/Compiler.scala:22-30) --
// m named outputs over n_params inputs, forward evaluation only (Generator.prepare's "requirements",
// core/Generator.scala:59-94).  Fills nodes / lookup_refs / inv_fwd (nodes some output needs, topological) /
// fn_outputs / counts.flops_inv, special_inv.
std::string build_function(const void* rir, size_t len, Program& out);

// RIR_FLAG_GENERATOR containers: the function of build_function (its outputs are the plan's slots) followed by the
// generator plan of rainier_rir.h.  Every op kind, slot index, REPEAT count and nesting, and m_out are validated here.
struct GeneratorPlan {
  std::vector<rir_gen_op> ops;
  uint32_t m_out = 0;
};
std::string build_generator(const void* rir, size_t len, Program& fn, GeneratorPlan& plan);

}  // namespace rn

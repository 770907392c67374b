/*
 * rainier_rir.h -- "RIR": the frozen-DAG wire format handed across the drop-in boundary.
 *
 * The reference never serializes its compute DAG: `Compiler.compile` hands an in-memory
 * `Seq[ir.Param]` + `Seq[(String, ir.Expr)]` to the JVM-bytecode emitter
 * (rainier-compute/.../compute/Compiler.scala:22-30, ir/CompiledFunction.scala:42-120) and wraps it
 * in `ir.DataFunction(cf, numParamInputs, numOutputs, data)` (compute/Compiler.scala:14-20,
 * ir/DataFunction.scala:13-30).  RIR is a 1:1 flat encoding of exactly that hand-off:
 *
 *   - the closed sum type of ir/IR.scala:3-23 (Param / Const / VarDef+VarRef / BinaryIR / UnaryIR /
 *     LookupIR / SeqIR) flattened into an SSA node array in definition order.  A `VarDef(sym, rhs)`
 *     becomes the node that computes `rhs`; every `VarRef(sym)` becomes that node's index; `SeqIR`
 *     (evaluate-first-then-second, ir/ExprMethodGenerator.scala:57-63) disappears because node order
 *     already is evaluation order.  The reference guarantees defs precede refs
 *     ("VarRef was used before its VarDef" is a hard error, compute/Translator.scala:178-179), so the
 *     array is topologically sorted by construction: operands always have smaller indices.
 *   - ops of ir/Ops.scala:3-37.
 *   - `DataFunction`'s layout: inputs = nVars parameters then every target's column placeholders
 *     (compute/Target.scala:38-41); per target a row count and a list of output node ids
 *     (compute/Target.scala:50-56).
 *
 * Two flavours travel in the same container:
 *   RIR_FLAG_GRADIENT set   : every target carries nVars+1 outputs [density, d/dq_0 .. d/dq_{n-1}],
 *                             i.e. what `Compiler.compileTargets` produces today (symbolic gradient,
 *                             compute/Gradient.scala:8-69).  The CPU oracle consumes this flavour and the
 *                             CUDA emitter accepts it too ("symbolic" gradient mode).
 *   RIR_FLAG_GRADIENT clear : every target carries 1 output (the primal log-density); the CUDA emitter
 *                             derives adjoints itself (reverse mode over the SSA array).  This is the
 *                             flavour the Scala wrapper sends (SURVEY.md §7.3-3).
 *
 * All integers little-endian; all structs packed as declared (natural alignment, no padding surprises:
 * every struct size is a multiple of 8).
 */
#ifndef RAINIER_RIR_H
#define RAINIER_RIR_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RIR_MAGIC 0x31524952u /* "RIR1" */
#define RIR_VERSION 1u

#define RIR_FLAG_GRADIENT 1u
/* RIR_FLAG_FUNCTION: the container is the hand-off of the OTHER compile seam, `Compiler.compile(inputs: Seq[ir.Param],
 * outputs: Seq[(String, Real)]): ir.CompiledFunction` (compute/Compiler.scala:22-30) as Generator.prepare uses it for the
 * "requirements" of a posterior-predictive generator (core/Generator.scala:59-94, called from Trace.predict,
 * core/Trace.scala:34-41): n_inputs == n_params (parameters only, no columns), n_targets == 1 with n_rows == 0,
 * n_cols == 0 and n_outputs == m >= 1 arbitrary output nodes ("req0".."req{m-1}").  No gradient, no accumulation:
 * output j of a point is the value of node outputs[j].  Consumed by rn_function_create (rainier_cuda.h). */
#define RIR_FLAG_FUNCTION 2u
/* RIR_FLAG_GENERATOR (only together with RIR_FLAG_FUNCTION): the container also carries a posterior-predictive generator
 * plan -- the `Generator.get(rng, evaluator)` half of Trace.predict (core/Trace.scala:34-41) for the built-in
 * distributions.  The function's m outputs are the plan's "slots": every Real a draw reads.  Consumed by
 * rn_generator_create (rainier_cuda.h).  The plan section follows the target block (see the file layout below). */
#define RIR_FLAG_GENERATOR 4u

/* node kinds */
enum {
  RIR_INPUT = 0,  /* a = input index: [0,n_params) parameters, then column placeholders  (ir.Param) */
  RIR_CONST = 1,  /* value                                                                (ir.Const) */
  RIR_UNARY = 2,  /* op = RIR_U_*, a = operand node                                       (UnaryIR)  */
  RIR_BINARY = 3, /* op = RIR_B_*, a = left node, b = right node                          (BinaryIR) */
  RIR_LOOKUP = 4  /* a = index node, b = offset into lookup_refs, c = table length, d = low (LookupIR) */
};

/* binary ops, ir/Ops.scala:3-23.  Subtract/Divide exist in the reference's op set but its Translator never
 * emits them (compute/Translator.scala:154-156); they are encoded for completeness. */
enum { RIR_B_ADD = 0, RIR_B_MUL = 1, RIR_B_SUB = 2, RIR_B_DIV = 3, RIR_B_POW = 4, RIR_B_COMPARE = 5 };

/* unary ops, ir/Ops.scala:25-37 */
enum {
  RIR_U_EXP = 0,
  RIR_U_LOG = 1,
  RIR_U_ABS = 2,
  RIR_U_NOOP = 3,
  RIR_U_SIN = 4,
  RIR_U_COS = 5,
  RIR_U_TAN = 6,
  RIR_U_ASIN = 7,
  RIR_U_ACOS = 8,
  RIR_U_ATAN = 9
};

typedef struct rir_header {
  uint32_t magic;         /* RIR_MAGIC */
  uint32_t version;       /* RIR_VERSION */
  uint32_t n_params;      /* nVars: number of sampled parameters (DataFunction.numParamInputs) */
  uint32_t n_inputs;      /* n_params + total number of column placeholders (cf.numInputs) */
  uint32_t n_nodes;
  uint32_t n_targets;     /* prior + one per likelihood (compute/Target.scala:73-79) */
  uint32_t n_lookup_refs; /* total entries in the lookup-ref side table */
  uint32_t flags;         /* RIR_FLAG_* */
} rir_header; /* 32 bytes */

typedef struct rir_node {
  uint8_t kind; /* RIR_INPUT .. RIR_LOOKUP */
  uint8_t op;   /* RIR_B_* or RIR_U_* */
  uint16_t reserved0;
  int32_t a;
  int32_t b;
  int32_t c;
  int32_t d;
  int32_t reserved1;
  double value; /* RIR_CONST only; IEEE-754 bits incl. +-inf */
} rir_node; /* 32 bytes */

typedef struct rir_target {
  uint64_t n_rows;      /* rows streamed per evaluation; 0 = data-free target (evaluated once) */
  uint32_t first_input; /* index of this target's first column placeholder in the input vector */
  uint32_t n_cols;      /* number of column placeholders (columns ++ gradientColumns) */
  uint32_t n_outputs;   /* n_params+1 if RIR_FLAG_GRADIENT else 1 */
  uint32_t reserved;
  /* followed by n_outputs x uint32_t output node ids, padded to a multiple of 8 bytes */
} rir_target; /* 24 bytes + outputs */

/*
 * Generator plan (RIR_FLAG_GENERATOR).  One draw runs the ops in order over one register `v` (a double) and writes m_out
 * doubles, in the order of the EMIT ops.  Discrete draws leave a Java Long in v (stored as a double); every double -> long
 * conversion is the JVM's D2L (NaN -> 0, saturating), double -> int is D2I.  Slot fields name function outputs
 * ([0, n_outputs)); fields a kind does not read must be -1.  The arithmetic of every op restates the reference
 * (core/Continuous.scala, core/Discrete.scala) in its own evaluation order.
 */
enum {
  RIR_G_NORMAL = 0,       /* v = RNG.standardNormal                                                  Continuous.scala:63-67   */
  RIR_G_CAUCHY = 1,       /* v = standardNormal / standardNormal (numerator drawn first)             :72-77           */
  RIR_G_LAPLACE = 2,      /* u = standardUniform - 0.5; v = signum(u) * -1 * log(1 - 2|u|)           :82-89           */
  RIR_G_UNIFORM = 3,      /* v = standardUniform                                                     :204-218         */
  RIR_G_GAMMA = 4,        /* v = Gamma.standard(slot[0]) draw (Marsaglia-Tsang; a < 1 draws u first) :114-144         */
  RIR_G_BETA = 5,         /* x = Gamma(slot[0], 1), y = Gamma(slot[1], 1) draws; v = x / (x + y)     :162-184         */
  RIR_G_SCALE = 6,        /* v = v * slot[0]                              (Injection.scala:48-66 fastForwards) */
  RIR_G_TRANSLATE = 7,    /* v = v + slot[0]                              (Injection.scala:71-86)              */
  RIR_G_EXP = 8,          /* v = exp(v)                                   (Injection.scala:91-107)             */
  RIR_G_EMIT = 9,         /* out[next] = v                                                                     */
  RIR_G_BERNOULLI = 10,   /* slot[0] = p                                                             Discrete.scala:38-52   */
  RIR_G_GEOMETRIC = 11,   /* slot[0] = p                                                             :59-73           */
  RIR_G_POISSON = 12,     /* slot[0] = lambda (small below 30, large otherwise)                      :122-186         */
  RIR_G_BINOMIAL = 13,    /* slots p, k, p*k, k*p, (k*p*(1-p)).pow(0.5), p + 0 (the categorical CDF)  :194-228        */
  RIR_G_NEGBINOMIAL = 14, /* slots p, n, 1-p, n*p/(1-p), (n*p).pow(1/2)/(1-p)                         :81-108          */
  RIR_G_VALUE = 15,       /* v = slot[0]                                  (Generator.real, a Real as ToGenerator) */
  RIR_G_REPEAT = 16,      /* run the ops up to the matching END k times   (Generator.repeat with a constant k)  */
  RIR_G_END = 17
};
#define RIR_G_MAX_SLOTS 6
#define RIR_G_MAX_DEPTH 8 /* REPEAT nesting */

typedef struct rir_gen_header {
  uint32_t n_ops;
  uint32_t m_out;    /* doubles per draw: the EMITs, each multiplied by the k of every enclosing REPEAT; at most 2^24.
                        Ops executed per draw (likewise multiplied, one more per repetition) are at most 2^26 */
  uint32_t reserved[2];
} rir_gen_header; /* 16 bytes */

typedef struct rir_gen_op {
  uint32_t kind;                  /* RIR_G_* */
  int32_t slot[RIR_G_MAX_SLOTS];  /* function output indices, -1 where unused */
  uint32_t reserved;
  int64_t k;                      /* RIR_G_REPEAT: repetitions, 0 <= k <= INT32_MAX; 0 otherwise */
} rir_gen_op; /* 40 bytes */

/*
 * File layout:
 *   rir_header
 *   rir_node      nodes[n_nodes]
 *   int32_t       lookup_refs[n_lookup_refs]   (padded to a multiple of 8 bytes)
 *   n_targets x { rir_target, uint32_t outputs[n_outputs] (padded to 8) }
 *   RIR_FLAG_GENERATOR only: rir_gen_header, rir_gen_op ops[n_ops]
 */

#ifdef __cplusplus
}
#endif
#endif

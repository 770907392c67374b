// rn_graph.cpp -- RIR -> Program (see rn_graph.hpp).
#include "rn_graph.hpp"

#include <cmath>
#include <cstring>
#include <algorithm>
#include <functional>
#include <map>
#include <set>

namespace rn {

namespace {

struct Builder {
  Program& P;
  bool fast;
  std::vector<int> dep;       // -1 invariant, t = row-variant of target t
  std::vector<char> active;   // depends on a parameter
  explicit Builder(Program& p, bool f) : P(p), fast(f) {}

  int add(const Node& n, int d, bool act) {
    P.nodes.push_back(n);
    dep.push_back(d);
    active.push_back(act ? 1 : 0);
    return (int)P.nodes.size() - 1;
  }
  // ---- node factories for the reverse sweeps (region/target set by the caller context) ----
  uint8_t cur_region = R_INV_BWD;
  int cur_target = -1;
  std::vector<int32_t>* cur_list = nullptr;

  int emit(Node n) {
    n.region = cur_region;
    n.target = cur_target;
    int id = add(n, cur_region == R_ROW_BWD ? cur_target : -1, true);
    cur_list->push_back(id);
    return id;
  }
  bool is_const(int id, double v) const { return P.nodes[id].kind == K_CONST && P.nodes[id].value == v; }
  int cst(double v) {
    Node n;
    n.kind = K_CONST;
    n.value = v;
    return emit(n);
  }
  int un(uint8_t op, int a) {
    if (op == U_NEG && P.nodes[a].kind == K_CONST) return cst(-P.nodes[a].value);
    Node n;
    n.kind = K_UNARY;
    n.op = op;
    n.a = a;
    return emit(n);
  }
  int bin(uint8_t op, int a, int b) {
    if (op == RIR_B_MUL) {
      if (is_const(a, 1.0)) return b;
      if (is_const(b, 1.0)) return a;
    }
    if (op == RIR_B_POW) {
      if (is_const(b, 1.0)) return a;
      if (is_const(b, 0.0)) return cst(1.0);
    }
    Node n;
    n.kind = K_BINARY;
    n.op = op;
    n.a = a;
    n.b = b;
    return emit(n);
  }
  int seleq(int idx, int k, int b, int c) {
    Node n;
    n.kind = K_SELEQ;
    n.a = idx;
    n.d = k;
    n.b = b;
    n.c = c;
    return emit(n);
  }
  int accread(int slot) {
    Node n;
    n.kind = K_ACC;
    n.a = slot;
    return emit(n);
  }
  int sum(const std::vector<int>& parts) {
    int s = parts[0];
    for (size_t i = 1; i < parts.size(); i++) s = bin(RIR_B_ADD, s, parts[i]);
    return s;
  }

  // Contributions d(out)/d(operand) for one node, given its adjoint node `adj`.  Mirrors the Diff rules of
  // compute/Gradient.scala:71-152.  `push(operand, contribution)` routes them.
  template <class Push>
  void propagate(int id, int adj, Push push) {
    const Node nd = P.nodes[id];
    switch (nd.kind) {
      case K_UNARY: {
        const int x = nd.a;
        if (!active[x]) return;
        switch (nd.op) {
          case RIR_U_EXP: push(x, bin(RIR_B_MUL, adj, id)); break;                       // g * child
          case RIR_U_LOG: push(x, bin(RIR_B_DIV, adj, x)); break;                        // g * (1/x)
          case RIR_U_ABS: {                                                              // eq(x,0,0, g*x/|x|)
            int t = bin(RIR_B_DIV, bin(RIR_B_MUL, adj, x), id);
            int cmp = bin(RIR_B_COMPARE, x, cst(0.0));
            push(x, seleq(cmp, 0, cst(0.0), t));
            break;
          }
          case RIR_U_NOOP: push(x, adj); break;
          case RIR_U_SIN: push(x, bin(RIR_B_MUL, adj, un(RIR_U_COS, x))); break;
          case RIR_U_COS: push(x, bin(RIR_B_MUL, adj, un(U_NEG, un(RIR_U_SIN, x)))); break;
          case RIR_U_TAN: {
            int c = un(RIR_U_COS, x);
            push(x, bin(RIR_B_DIV, adj, bin(RIR_B_MUL, c, c)));
            break;
          }
          case RIR_U_ASIN:
            push(x, bin(RIR_B_DIV, adj, un(U_SQRT, bin(RIR_B_SUB, cst(1.0), bin(RIR_B_MUL, x, x)))));
            break;
          case RIR_U_ACOS:
            push(x, bin(RIR_B_DIV, un(U_NEG, adj), un(U_SQRT, bin(RIR_B_SUB, cst(1.0), bin(RIR_B_MUL, x, x)))));
            break;
          case RIR_U_ATAN: push(x, bin(RIR_B_DIV, adj, bin(RIR_B_ADD, cst(1.0), bin(RIR_B_MUL, x, x)))); break;
          case U_NEG: push(x, un(U_NEG, adj)); break;
          default: break;
        }
        return;
      }
      case K_BINARY: {
        const int a = nd.a, b = nd.b;
        switch (nd.op) {
          case RIR_B_ADD:
            if (active[a]) push(a, adj);
            if (active[b]) push(b, adj);
            break;
          case RIR_B_SUB:
            if (active[a]) push(a, adj);
            if (active[b]) push(b, un(U_NEG, adj));
            break;
          case RIR_B_MUL:
            if (active[a]) push(a, bin(RIR_B_MUL, adj, b));
            if (active[b]) push(b, bin(RIR_B_MUL, adj, a));
            break;
          case RIR_B_DIV:
            if (active[a]) push(a, bin(RIR_B_DIV, adj, b));
            if (active[b]) push(b, un(U_NEG, bin(RIR_B_DIV, bin(RIR_B_MUL, adj, id), b)));
            break;
          case RIR_B_POW:
            if (active[a]) {  // g * exponent * base.pow(exponent - 1)
              if (P.nodes[b].kind == K_CONST && P.nodes[b].value == -1.0) {
                // y = 1/x: dy/dx = -1/x^2 = -(y*y) -- the node's own value, two multiplications instead of a division per
                // observation (the logistic link 1/(1 + e^z) of every Bernoulli row)
                push(a, bin(RIR_B_MUL, un(U_NEG, adj), bin(RIR_B_MUL, id, id)));
              } else {
                int em1 = P.nodes[b].kind == K_CONST ? cst(P.nodes[b].value - 1.0) : bin(RIR_B_SUB, b, cst(1.0));
                push(a, bin(RIR_B_MUL, bin(RIR_B_MUL, adj, b), bin(RIR_B_POW, a, em1)));
              }
            }
            if (active[b]) {  // g * child * log(eq(base,0,1,base))
              int cmp = bin(RIR_B_COMPARE, a, cst(0.0));
              int safe = seleq(cmp, 0, cst(1.0), a);
              push(b, bin(RIR_B_MUL, bin(RIR_B_MUL, adj, id), un(RIR_U_LOG, safe)));
            }
            break;
          default: break;  // COMPARE: no gradient (compute/Gradient.scala:58-61)
        }
        return;
      }
      case K_LOOKUP: {  // one-hot per entry (compute/Gradient.scala:148-152); large invariant tables are
                        // handled by the caller as a scatter
        for (int j = 0; j < nd.c; j++) {
          int e = P.lookup_refs[nd.b + j];
          if (!active[e]) continue;
          push(e, seleq(nd.a, j + nd.d, adj, cst(0.0)));
        }
        return;
      }
      case K_SELEQ: {
        if (active[nd.b]) push(nd.b, seleq(nd.a, nd.d, adj, cst(0.0)));
        if (active[nd.c]) push(nd.c, seleq(nd.a, nd.d, cst(0.0), adj));
        return;
      }
      default: return;
    }
  }
};

void count_node(const Node& n, double& flops, double& special) {
  switch (n.kind) {
    case K_UNARY:
      if (n.op == RIR_U_NOOP) break;
      if (n.op == RIR_U_ABS || n.op == U_NEG)
        flops += 1;
      else
        special += 1;
      break;
    case K_BINARY:
      if (n.op == RIR_B_ADD || n.op == RIR_B_MUL || n.op == RIR_B_SUB || n.op == RIR_B_COMPARE)
        flops += 1;
      else
        special += 1;
      break;
    default: break;
  }
}

}  // namespace

std::string build_program(const void* rir, size_t len, bool want_adjoint, bool fast_math, Program& P) {
  const uint8_t* p = (const uint8_t*)rir;
  const uint8_t* end = p + len;
  rir_header h;
  if (len < sizeof(h)) return "RIR: truncated header";
  std::memcpy(&h, p, sizeof(h));
  p += sizeof(h);
  if (h.magic != RIR_MAGIC) return "RIR: bad magic";
  if (h.version != RIR_VERSION) return "RIR: unsupported version";
  if (h.n_inputs < h.n_params) return "RIR: n_inputs < n_params";
  if ((size_t)(end - p) < (size_t)h.n_nodes * sizeof(rir_node)) return "RIR: truncated node array";
  const bool has_grad = (h.flags & RIR_FLAG_GRADIENT) != 0;
  if (!has_grad) want_adjoint = true;

  P = Program();
  P.n_params = h.n_params;
  P.n_inputs = h.n_inputs;
  P.symbolic = !want_adjoint;
  Builder B(P, fast_math);

  std::vector<rir_node> raw(h.n_nodes);
  std::memcpy(raw.data(), p, (size_t)h.n_nodes * sizeof(rir_node));
  p += (size_t)h.n_nodes * sizeof(rir_node);
  size_t lrb = ((size_t)h.n_lookup_refs * 4 + 7) & ~(size_t)7;
  if ((size_t)(end - p) < lrb) return "RIR: truncated lookup refs";
  P.lookup_refs.resize(h.n_lookup_refs);
  if (h.n_lookup_refs) std::memcpy(P.lookup_refs.data(), p, (size_t)h.n_lookup_refs * 4);
  p += lrb;
  P.targets.resize(h.n_targets);
  for (uint32_t t = 0; t < h.n_targets; t++) {
    rir_target rt;
    if ((size_t)(end - p) < sizeof(rt)) return "RIR: truncated target";
    std::memcpy(&rt, p, sizeof(rt));
    p += sizeof(rt);
    size_t ob = ((size_t)rt.n_outputs * 4 + 7) & ~(size_t)7;
    if ((size_t)(end - p) < ob) return "RIR: truncated outputs";
    TargetInfo& T = P.targets[t];
    T.n_rows = rt.n_rows;
    T.first_input = rt.first_input;
    T.n_cols = rt.n_cols;
    if (rt.n_outputs != (has_grad ? h.n_params + 1 : 1)) return "RIR: wrong number of outputs for target";
    std::vector<uint32_t> outs(rt.n_outputs);
    std::memcpy(outs.data(), p, (size_t)rt.n_outputs * 4);
    p += ob;
    for (uint32_t o : outs) {
      if (o >= h.n_nodes) return "RIR: output id out of range";
      T.outputs.push_back((int32_t)o);
    }
    if (want_adjoint) T.outputs.resize(1);
    if (T.n_cols > 0 && (T.first_input < h.n_params || T.first_input + T.n_cols > h.n_inputs))
      return "RIR: target column range out of bounds";
  }

  // ---- import nodes, validate, classify ----
  auto target_of_input = [&](int inp) -> int {
    if (inp < (int)h.n_params) return -1;
    for (size_t t = 0; t < P.targets.size(); t++)
      if ((uint32_t)inp >= P.targets[t].first_input && (uint32_t)inp < P.targets[t].first_input + P.targets[t].n_cols)
        return (int)t;
    return -2;
  };
  for (uint32_t i = 0; i < h.n_nodes; i++) {
    const rir_node& r = raw[i];
    Node n;
    n.kind = r.kind;
    n.op = r.op;
    n.a = r.a;
    n.b = r.b;
    n.c = r.c;
    n.d = r.d;
    n.value = r.value;
    auto ok = [&](int32_t x) { return x >= 0 && (uint32_t)x < i; };
    int d = -1;
    bool act = false, good = true;
    auto merge = [&](int x) {
      if (B.active[x]) act = true;
      int dx = B.dep[x];
      if (dx == -1) return;
      if (d == -1 || d == dx)
        d = dx;
      else
        good = false;
    };
    switch (r.kind) {
      case RIR_INPUT:
        if (r.a < 0 || (uint32_t)r.a >= h.n_inputs) return "RIR: input index out of range";
        d = target_of_input(r.a);
        if (d == -2) return "RIR: column input not owned by any target";
        act = (uint32_t)r.a < h.n_params;
        break;
      case RIR_CONST: break;
      case RIR_UNARY:
        if (r.op > RIR_U_ATAN) return "RIR: unknown unary op";
        if (!ok(r.a)) return "RIR: unary operand not defined before use";
        merge(r.a);
        break;
      case RIR_BINARY:
        if (r.op > RIR_B_COMPARE) return "RIR: unknown binary op";
        if (!ok(r.a) || !ok(r.b)) return "RIR: binary operand not defined before use";
        merge(r.a);
        merge(r.b);
        if (r.op == RIR_B_COMPARE) act = false;  // piecewise constant
        break;
      case RIR_LOOKUP:
        if (!ok(r.a) || r.b < 0 || r.c <= 0 || (uint32_t)(r.b + r.c) > h.n_lookup_refs) return "RIR: bad lookup";
        P.has_lookup = true;
        {
          bool idx_act_saved = act;
          merge(r.a);
          act = idx_act_saved;  // the index carries no gradient
          for (int k = 0; k < r.c; k++) {
            if (!ok(P.lookup_refs[r.b + k])) return "RIR: lookup ref not defined before use";
            merge(P.lookup_refs[r.b + k]);
          }
        }
        break;
      default: return "RIR: unknown node kind";
    }
    if (!good) return "RIR: node mixes columns of two targets";
    n.region = d == -1 ? R_INV_FWD : R_ROW_FWD;
    n.target = d;
    B.add(n, d, act);
  }

  // ---- reachability per target ----
  const int N0 = (int)P.nodes.size();
  std::vector<char> inv_needed(N0, 0);
  for (size_t t = 0; t < P.targets.size(); t++) {
    TargetInfo& T = P.targets[t];
    std::vector<char> need(N0, 0);
    for (int o : T.outputs) need[o] = 1;
    for (int i = N0 - 1; i >= 0; i--) {
      if (!need[i]) continue;
      const Node& nd = P.nodes[i];
      switch (nd.kind) {
        case K_UNARY: need[nd.a] = 1; break;
        case K_BINARY: need[nd.a] = need[nd.b] = 1; break;
        case K_LOOKUP:
          need[nd.a] = 1;
          for (int k = 0; k < nd.c; k++) need[P.lookup_refs[nd.b + k]] = 1;
          break;
        default: break;
      }
    }
    for (int i = 0; i < N0; i++) {
      if (!need[i]) continue;
      if (B.dep[i] == -1)
        inv_needed[i] = 1;
      else if (B.dep[i] == (int)t)
        T.row_fwd.push_back(i);
      else
        return "RIR: target reads another target's columns";
    }
    if (!T.row_fwd.empty() && !T.streamed()) return "RIR: target has column-dependent nodes but no rows";
  }
  for (int i = 0; i < N0; i++)
    if (inv_needed[i]) P.inv_fwd.push_back(i);

  const int n = (int)P.n_params;
  if (P.symbolic) {
    // DataFunction: outputs(o) += output(o) for every target in order (ir/DataFunction.scala:32-84)
    P.n_slots = n + 1;
    P.slot_row_accumulated.assign(P.n_slots, 0);
    for (auto& T : P.targets)
      for (int o = 0; o <= n; o++) {
        T.row_acc.push_back({o, T.outputs[o]});
        if (T.streamed()) P.slot_row_accumulated[o] = 1;
      }
  } else {
    // ---- adjoint mode: two-level reverse sweep ----
    P.n_slots = 1;
    std::map<int, std::vector<int>> inv_slots;  // invariant node -> accumulator slots feeding its adjoint
    std::map<int, std::vector<double>> inv_seeds;  // invariant node -> constant seeds
    std::map<int, int> direct_slot;             // invariant node -> its own frontier slot
    std::map<std::vector<int>, int> scatter_base;  // table entries of a large Lookup -> its block of scatter slots
    auto frontier_slot = [&](int node) {
      auto it = direct_slot.find(node);
      if (it != direct_slot.end()) return it->second;
      int s = P.n_slots++;
      direct_slot[node] = s;
      inv_slots[node].push_back(s);
      return s;
    };
    for (size_t t = 0; t < P.targets.size(); t++) {
      TargetInfo& T = P.targets[t];
      const int out = T.outputs[0];
      T.row_acc.push_back({0, out});
      if (!T.streamed()) {
        if (B.active[out]) inv_seeds[out].push_back(1.0);
        continue;
      }
      if (B.dep[out] == -1) {  // constant-in-row output of a streamed target: contributes n_rows times
        if (B.active[out]) inv_seeds[out].push_back((double)T.n_rows);
        continue;
      }
      B.cur_region = R_ROW_BWD;
      B.cur_target = (int)t;
      B.cur_list = &T.row_bwd;
      std::map<int, std::vector<int>> adj;
      adj[out].push_back(B.cst(1.0));
      for (int k = (int)T.row_fwd.size() - 1; k >= 0; k--) {
        const int id = T.row_fwd[k];
        auto it = adj.find(id);
        if (it == adj.end() || !B.active[id]) continue;
        const int a = B.sum(it->second);
        const Node nd = P.nodes[id];
        // large invariant table -> scatter
        if (nd.kind == K_LOOKUP && nd.c > 8) {
          bool all_inv = true;
          for (int j = 0; j < nd.c; j++)
            if (B.dep[P.lookup_refs[nd.b + j]] != -1) all_inv = false;
          if (all_inv) {
            // the 8 unrolled observation splits of Model.observe (core/Model.scala:98-132) each carry their own Lookup
            // over the SAME table entries: they share one block of scatter accumulators
            std::vector<int> refs(P.lookup_refs.begin() + nd.b, P.lookup_refs.begin() + nd.b + nd.c);
            auto sb = scatter_base.find(refs);
            int base;
            if (sb != scatter_base.end()) {
              base = sb->second;
            } else {
              base = P.n_slots;
              P.n_slots += nd.c;
              scatter_base[refs] = base;
              for (int j = 0; j < nd.c; j++) {
                int e = refs[j];
                if (B.active[e]) inv_slots[e].push_back(base + j);
              }
            }
            T.row_scatter.push_back({base, nd.c, nd.d, nd.a, a});
            continue;
          }
        }
        B.propagate(id, a, [&](int x, int contrib) {
          if (B.dep[x] == -1) {
            int s = frontier_slot(x);
            T.row_acc.push_back({s, contrib});
          } else {
            adj[x].push_back(contrib);
          }
        });
      }
    }
    P.slot_row_accumulated.assign(P.n_slots, 1);  // every adjoint slot (and slot 0) may get row contributions
    // ---- invariant reverse sweep ----
    B.cur_region = R_INV_BWD;
    B.cur_target = -1;
    B.cur_list = &P.inv_bwd;
    std::map<int, std::vector<int>> adj;
    std::vector<std::vector<int>> param_adj(n);
    for (int k = (int)P.inv_fwd.size() - 1; k >= 0; k--) {
      const int id = P.inv_fwd[k];
      if (!B.active[id]) continue;
      std::vector<int> parts;
      auto sd = inv_seeds.find(id);
      if (sd != inv_seeds.end()) {
        double tot = 0;
        for (double v : sd->second) tot += v;
        parts.push_back(B.cst(tot));
      }
      auto sl = inv_slots.find(id);
      if (sl != inv_slots.end())
        for (int s : sl->second) parts.push_back(B.accread(s));
      auto it = adj.find(id);
      if (it != adj.end())
        for (int c : it->second) parts.push_back(c);
      if (parts.empty()) continue;
      const int a = B.sum(parts);
      const Node nd = P.nodes[id];
      if (nd.kind == K_INPUT) {
        if (nd.a < n) param_adj[nd.a].push_back(a);
        continue;
      }
      B.propagate(id, a, [&](int x, int contrib) { adj[x].push_back(contrib); });
    }
    P.grad_nodes.resize(n);
    for (int i = 0; i < n; i++) P.grad_nodes[i] = param_adj[i].empty() ? B.cst(0.0) : B.sum(param_adj[i]);
  }

  // ---- dense structure: maximal left-folded sums of parameter x column products in every streamed row body ----
  for (TargetInfo& T : P.targets) {
    if (!T.streamed()) continue;
    auto term = [&](int id, int& param, int& col) {  // MUL(parameter input, column input), either order
      const Node& m = P.nodes[id];
      if (m.kind != K_BINARY || m.op != RIR_B_MUL) return false;
      const Node &x = P.nodes[m.a], &y = P.nodes[m.b];
      if (x.kind != K_INPUT || y.kind != K_INPUT) return false;
      const bool xp = (uint32_t)x.a < P.n_params, yp = (uint32_t)y.a < P.n_params;
      if (xp == yp) return false;
      param = xp ? x.a : y.a;
      col = xp ? y.a : x.a;
      return true;
    };
    std::vector<char> inner(P.nodes.size(), 0);  // ADD nodes that are the left operand of a longer fold
    std::vector<DotInfo> found;
    for (int id : T.row_fwd) {
      const Node& n = P.nodes[id];
      if (n.kind != K_BINARY || n.op != RIR_B_ADD) continue;
      DotInfo d;
      d.node = id;
      int cur = id;
      std::vector<std::pair<int, int>> rev;  // terms from the last to the first
      for (;;) {
        const Node& a = P.nodes[cur];
        int p = 0, c = 0;
        if (a.kind == K_BINARY && a.op == RIR_B_ADD && term(a.b, p, c)) {
          rev.push_back({p, c});
          if (cur != id) inner[cur] = 1;
          cur = a.a;
          continue;
        }
        if (term(cur, p, c))
          rev.push_back({p, c});
        else
          d.base = cur;
        break;
      }
      if (rev.size() < 2) continue;
      for (auto it = rev.rbegin(); it != rev.rend(); ++it) {
        d.params.push_back(it->first);
        d.columns.push_back(it->second);
      }
      found.push_back(std::move(d));
    }
    for (DotInfo& d : found)
      if (!inner[d.node]) T.dots.push_back(std::move(d));
  }

  // ---- op counts ----
  P.counts.flops_row.assign(P.targets.size(), 0.0);
  P.counts.special_row.assign(P.targets.size(), 0.0);
  for (int id : P.inv_fwd) count_node(P.nodes[id], P.counts.flops_inv, P.counts.special_inv);
  for (int id : P.inv_bwd) count_node(P.nodes[id], P.counts.flops_inv, P.counts.special_inv);
  for (size_t t = 0; t < P.targets.size(); t++) {
    TargetInfo& T = P.targets[t];
    double f = 0, s = 0;
    for (int id : T.row_fwd) count_node(P.nodes[id], f, s);
    for (int id : T.row_bwd) count_node(P.nodes[id], f, s);
    f += (double)T.row_acc.size() + (double)T.row_scatter.size();
    if (T.streamed()) {
      P.counts.flops_row[t] = f;
      P.counts.special_row[t] = s;
    } else {
      P.counts.flops_inv += f;
      P.counts.special_inv += s;
    }
  }
  for (auto& T : P.targets)
    if (!T.row_scatter.empty()) P.has_lookup = true;
  return "";
}

std::string build_function(const void* rir, size_t len, Program& P) {
  const uint8_t* p = (const uint8_t*)rir;
  const uint8_t* end = p + len;
  rir_header h;
  if (len < sizeof(h)) return "RIR: truncated header";
  std::memcpy(&h, p, sizeof(h));
  p += sizeof(h);
  if (h.magic != RIR_MAGIC) return "RIR: bad magic";
  if (h.version != RIR_VERSION) return "RIR: unsupported version";
  if (!(h.flags & RIR_FLAG_FUNCTION)) return "RIR: not a function container (RIR_FLAG_FUNCTION clear)";
  if (h.n_inputs != h.n_params) return "RIR: a function container has no column inputs";
  if (h.n_targets != 1) return "RIR: a function container carries exactly one output list";
  if ((size_t)(end - p) < (size_t)h.n_nodes * sizeof(rir_node)) return "RIR: truncated node array";
  P = Program();
  P.n_params = h.n_params;
  P.n_inputs = h.n_inputs;
  P.symbolic = true;
  std::vector<rir_node> raw(h.n_nodes);
  if (h.n_nodes) std::memcpy(raw.data(), p, (size_t)h.n_nodes * sizeof(rir_node));
  p += (size_t)h.n_nodes * sizeof(rir_node);
  const size_t lrb = ((size_t)h.n_lookup_refs * 4 + 7) & ~(size_t)7;
  if ((size_t)(end - p) < lrb) return "RIR: truncated lookup refs";
  P.lookup_refs.resize(h.n_lookup_refs);
  if (h.n_lookup_refs) std::memcpy(P.lookup_refs.data(), p, (size_t)h.n_lookup_refs * 4);
  p += lrb;
  rir_target rt;
  if ((size_t)(end - p) < sizeof(rt)) return "RIR: truncated target";
  std::memcpy(&rt, p, sizeof(rt));
  p += sizeof(rt);
  if (rt.n_rows != 0 || rt.n_cols != 0) return "RIR: a function container streams no rows";
  if (rt.n_outputs == 0) return "RIR: function without outputs";
  if ((size_t)(end - p) < (((size_t)rt.n_outputs * 4 + 7) & ~(size_t)7)) return "RIR: truncated outputs";
  std::vector<uint32_t> outs(rt.n_outputs);
  std::memcpy(outs.data(), p, (size_t)rt.n_outputs * 4);
  for (uint32_t o : outs) {
    if (o >= h.n_nodes) return "RIR: output id out of range";
    P.fn_outputs.push_back((int32_t)o);
  }
  P.nodes.resize(h.n_nodes);
  for (uint32_t i = 0; i < h.n_nodes; i++) {
    const rir_node& r = raw[i];
    auto ok = [&](int32_t x) { return x >= 0 && (uint32_t)x < i; };
    switch (r.kind) {
      case RIR_INPUT:
        if (r.a < 0 || (uint32_t)r.a >= h.n_inputs) return "RIR: input index out of range";
        break;
      case RIR_CONST: break;
      case RIR_UNARY:
        if (r.op > RIR_U_ATAN) return "RIR: unknown unary op";
        if (!ok(r.a)) return "RIR: unary operand not defined before use";
        break;
      case RIR_BINARY:
        if (r.op > RIR_B_COMPARE) return "RIR: unknown binary op";
        if (!ok(r.a) || !ok(r.b)) return "RIR: binary operand not defined before use";
        break;
      case RIR_LOOKUP:
        if (!ok(r.a) || r.b < 0 || r.c <= 0 || (uint32_t)(r.b + r.c) > h.n_lookup_refs) return "RIR: bad lookup";
        for (int k = 0; k < r.c; k++)
          if (!ok(P.lookup_refs[r.b + k])) return "RIR: lookup ref not defined before use";
        P.has_lookup = true;
        break;
      default: return "RIR: unknown node kind";
    }
    Node& n = P.nodes[i];
    n.kind = r.kind;
    n.op = r.op;
    n.region = R_INV_FWD;
    n.target = -1;
    n.a = r.a;
    n.b = r.b;
    n.c = r.c;
    n.d = r.d;
    n.value = r.value;
  }
  // only what some output needs is evaluated (the generated outputN methods evaluate their own expression tree only,
  // ir/OutputMethodGenerator.scala:3-21); shared VarDefs are computed once, like the reference's globals
  std::vector<char> need(h.n_nodes, 0);
  for (int32_t o : P.fn_outputs) need[o] = 1;
  for (int i = (int)h.n_nodes - 1; i >= 0; i--) {
    if (!need[i]) continue;
    const Node& n = P.nodes[i];
    switch (n.kind) {
      case K_UNARY: need[n.a] = 1; break;
      case K_BINARY: need[n.a] = need[n.b] = 1; break;
      case K_LOOKUP:
        need[n.a] = 1;
        for (int k = 0; k < n.c; k++) need[P.lookup_refs[n.b + k]] = 1;
        break;
      default: break;
    }
  }
  for (uint32_t i = 0; i < h.n_nodes; i++)
    if (need[i]) {
      P.inv_fwd.push_back((int32_t)i);
      count_node(P.nodes[i], P.counts.flops_inv, P.counts.special_inv);
    }
  return "";
}

std::string build_generator(const void* rir, size_t len, Program& P, GeneratorPlan& G) {
  if (!rir || len < sizeof(rir_header)) return "RIR: truncated header";
  rir_header h;
  std::memcpy(&h, rir, sizeof(h));
  if (!(h.flags & RIR_FLAG_GENERATOR)) return "RIR: not a generator container (RIR_FLAG_GENERATOR clear)";
  std::string e = build_function(rir, len, P);
  if (!e.empty()) return e;
  // the plan section starts after the (single) target block, whose sizes build_function has checked
  size_t off = sizeof(h) + (size_t)h.n_nodes * sizeof(rir_node) + (((size_t)h.n_lookup_refs * 4 + 7) & ~(size_t)7);
  rir_target rt;
  std::memcpy(&rt, (const uint8_t*)rir + off, sizeof(rt));
  off += sizeof(rt) + (((size_t)rt.n_outputs * 4 + 7) & ~(size_t)7);
  rir_gen_header gh;
  if (len - off < sizeof(gh)) return "RIR: truncated generator header";
  std::memcpy(&gh, (const uint8_t*)rir + off, sizeof(gh));
  off += sizeof(gh);
  if (gh.n_ops == 0) return "RIR: generator without ops";
  if ((len - off) / sizeof(rir_gen_op) < gh.n_ops) return "RIR: truncated generator ops";
  G = GeneratorPlan();
  G.ops.resize(gh.n_ops);
  std::memcpy(G.ops.data(), (const uint8_t*)rir + off, (size_t)gh.n_ops * sizeof(rir_gen_op));
  const int64_t m = (int64_t)P.fn_outputs.size();
  // slots each kind reads; the remaining fields must be -1
  auto arity = [](uint32_t kind) -> int {
    switch (kind) {
      case RIR_G_GAMMA: case RIR_G_SCALE: case RIR_G_TRANSLATE: case RIR_G_BERNOULLI: case RIR_G_GEOMETRIC:
      case RIR_G_POISSON: case RIR_G_VALUE: return 1;
      case RIR_G_BETA: return 2;
      case RIR_G_NEGBINOMIAL: return 5;
      case RIR_G_BINOMIAL: return 6;
      default: return 0;
    }
  };
  // per draw: at most 2^24 values and 2^26 ops executed (an op inside REPEATs counts once per repetition, a repetition
  // itself once), so that no container makes one draw run unboundedly long whatever its RNG budget
  const int64_t kMaxOut = (int64_t)1 << 24;
  const double kMaxExecuted = (double)((int64_t)1 << 26);
  int64_t mult[RIR_G_MAX_DEPTH + 1], emitted[RIR_G_MAX_DEPTH + 1];
  double executed[RIR_G_MAX_DEPTH + 1];
  int depth = 0;
  mult[0] = 1;
  emitted[0] = 0;
  executed[0] = 0;
  for (size_t i = 0; i < G.ops.size(); i++) {
    const rir_gen_op& o = G.ops[i];
    if (o.kind > RIR_G_END) return "RIR: unknown generator op kind at op " + std::to_string(i);
    const int a = arity(o.kind);
    for (int s = 0; s < RIR_G_MAX_SLOTS; s++) {
      if (s < a && (o.slot[s] < 0 || o.slot[s] >= m)) return "RIR: generator slot out of range at op " + std::to_string(i);
      if (s >= a && o.slot[s] != -1) return "RIR: unused generator slot field is not -1 at op " + std::to_string(i);
    }
    if (o.kind != RIR_G_REPEAT && o.k != 0) return "RIR: repeat count on a non-REPEAT op at op " + std::to_string(i);
    if (o.kind == RIR_G_REPEAT) {
      if (o.k < 0 || o.k > 2147483647LL) return "RIR: REPEAT count out of range at op " + std::to_string(i);
      if (depth == RIR_G_MAX_DEPTH) return "RIR: REPEAT nested too deeply at op " + std::to_string(i);
      depth++;
      mult[depth] = o.k;
      emitted[depth] = 0;
      executed[depth] = 1;
    } else if (o.kind == RIR_G_END) {
      if (depth == 0) return "RIR: END without REPEAT at op " + std::to_string(i);
      const int64_t inner = emitted[depth] * mult[depth];
      const double inner_ops = executed[depth] * (double)mult[depth];
      depth--;
      emitted[depth] += inner;
      executed[depth] += inner_ops;
    } else {
      if (o.kind == RIR_G_EMIT) emitted[depth] += 1;
      executed[depth] += 1;
    }
    if (emitted[depth] > kMaxOut) return "RIR: generator emits more than 2^24 values per draw";
    if (executed[depth] > kMaxExecuted) return "RIR: generator executes more than 2^26 ops per draw";
  }
  if (depth != 0) return "RIR: REPEAT without END";
  if (emitted[0] == 0) return "RIR: generator emits nothing";
  if ((int64_t)gh.m_out != emitted[0]) return "RIR: generator m_out does not match its EMIT ops";
  G.m_out = gh.m_out;
  return "";
}

SeparableInfo analyze_separable(const Program& P, int max_degree, int max_atoms) {
  SeparableInfo R;
  const int N = (int)P.nodes.size();
  // parameter / column dependence of every node
  std::vector<char> pdep(N, 0), cdep(N, 0);
  for (int i = 0; i < N; i++) {
    const Node& n = P.nodes[i];
    auto dep = [&](int x) {
      pdep[i] |= pdep[x];
      cdep[i] |= cdep[x];
    };
    switch (n.kind) {
      case K_INPUT: ((uint32_t)n.a < P.n_params ? pdep[i] : cdep[i]) = 1; break;
      case K_UNARY: dep(n.a); break;
      case K_BINARY: dep(n.a); dep(n.b); break;
      case K_LOOKUP:
        dep(n.a);
        for (int k = 0; k < n.c; k++) dep(P.lookup_refs[n.b + k]);
        break;
      case K_SELEQ: dep(n.a); dep(n.b); dep(n.c); break;
      default: break;
    }
  }
  typedef std::vector<int32_t> Mono;  // sorted ids of column-only atoms; empty = parameter-only term
  typedef std::set<Mono> Poly;
  for (const TargetInfo& T : P.targets) {
    if (!T.streamed()) continue;
    R.streamed_targets++;
    std::map<int, Poly> form;
    bool ok = true;
    std::function<const Poly*(int)> get = [&](int id) -> const Poly* {
      auto it = form.find(id);
      if (it != form.end()) return &it->second;
      Poly p;
      if (!cdep[id])
        p.insert(Mono());  // parameter-only or constant: a coefficient
      else if (!pdep[id])
        p.insert(Mono(1, id));  // column-only: an atom, however complicated
      else {
        const Node& n = P.nodes[id];
        auto mul = [&](const Poly& a, const Poly& b, Poly& out) {
          for (const Mono& x : a)
            for (const Mono& y : b) {
              Mono m(x);
              m.insert(m.end(), y.begin(), y.end());
              std::sort(m.begin(), m.end());
              if ((int)m.size() > max_degree) return false;
              out.insert(std::move(m));
              if ((int)out.size() > max_atoms) return false;
            }
          return true;
        };
        bool good = false;
        if (n.kind == K_BINARY && (n.op == RIR_B_ADD || n.op == RIR_B_SUB)) {
          const Poly *a = get(n.a), *b = ok ? get(n.b) : nullptr;
          if (a && b) {
            p = *a;
            p.insert(b->begin(), b->end());
            good = (int)p.size() <= max_atoms;
          }
        } else if (n.kind == K_BINARY && n.op == RIR_B_MUL) {
          const Poly *a = get(n.a), *b = ok ? get(n.b) : nullptr;
          good = a && b && mul(*a, *b, p);
        } else if (n.kind == K_BINARY && n.op == RIR_B_DIV && !pdep[n.b]) {  // division by a column-only value: times an atom
          const Poly* a = get(n.a);
          Poly inv;
          inv.insert(Mono(1, id));  // stands for 1 / val[n.b]; a distinct atom per node is a safe over-count
          good = a && mul(*a, inv, p);
        } else if (n.kind == K_BINARY && n.op == RIR_B_DIV && !cdep[n.b]) {  // division by a parameter-only value: scales
          const Poly* a = get(n.a);
          if (a) {
            p = *a;
            good = true;
          }
        } else if (n.kind == K_BINARY && n.op == RIR_B_POW && P.nodes[n.b].kind == K_CONST && P.nodes[n.b].value == 2.0) {
          const Poly* a = get(n.a);
          good = a && mul(*a, *a, p);
        } else if (n.kind == K_UNARY && (n.op == RIR_U_NOOP || n.op == U_NEG)) {
          const Poly* a = get(n.a);
          if (a) {
            p = *a;
            good = true;
          }
        }
        if (!good) {  // a nonlinear operation on a node that mixes parameters and columns
          ok = false;
          return nullptr;
        }
      }
      return &form.emplace(id, std::move(p)).first->second;
    };
    const Poly* out = T.outputs.empty() ? nullptr : get(T.outputs[0]);
    if (ok && out) {
      R.separable_targets++;
      for (const Mono& m : *out)
        if (!m.empty()) R.atoms++;
      R.rows_removed += (int64_t)T.n_rows;
    }
  }
  return R;
}

}  // namespace rn

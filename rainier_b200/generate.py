"""
rainier_b200.generate -- lowering of a posterior-predictive generator to a RIR_FLAG_GENERATOR container
(include/rainier_rir.h), the input of CudaGenerator / rn_generator_create.

The Python stand-in of the reference's front end (oracle/rainier_py/core.py) builds generators the way the reference does:
as closures (`Generator.require(reqs)(fn)`, `Injection.transform`'s anonymous class, `map` / `zip` / `repeat`).  The lowering
recognises the closures of the built-in pieces by their definition site and reads the values they close over:

    Normal / Cauchy / Laplace / Uniform standard draws, Gamma.standard(shape), Beta(a, b)
    the Scale / Translate / Exp injections these distributions are made of (Injection.transform)
    Bernoulli, Geometric, Poisson, Binomial, NegativeBinomial
    a Real (Generator.real, a Real as ToGenerator), tuples (zip), Seq / Vec (traverse), repeat(k) with a constant k

Anything else -- user map / flatMap / from closures, categorical, Multinomial as a value, constants other than an empty
Seq -- raises Unsupported naming the piece; the caller keeps the host path.  Every Real a draw reads becomes one output
("slot") of the container's function, deduplicated; Binomial's and NegativeBinomial's inner Reals are rebuilt with the
same expressions their generators use (Discrete.scala:87-97, :203-213).
"""
import struct

from oracle.rainier_py import core
from oracle.rainier_py.compute import Constant, Real, compile_function_rir, jd2i, to_real

(NORMAL, CAUCHY, LAPLACE, UNIFORM, GAMMA, BETA, SCALE, TRANSLATE, EXP, EMIT, BERNOULLI, GEOMETRIC, POISSON, BINOMIAL,
 NEGBINOMIAL, VALUE, REPEAT, END) = range(18)
RIR_FLAG_GENERATOR = 4
GEN_HEADER = struct.Struct("<4I")  # rir_gen_header: n_ops, m_out, reserved[2]
GEN_OP = struct.Struct("<I6iIq")   # rir_gen_op: kind, slot[6], reserved, k
MAX_SLOTS = 6


class Unsupported(ValueError):
    """The generator contains a piece the device path does not lower."""


def _closure(f):
    return dict(zip(f.__code__.co_freevars, (c.cell_contents for c in (f.__closure__ or ()))))


class _Lowering:
    def __init__(self):
        self.slots, self.index, self.ops = [], {}, []

    def slot(self, r):
        r = to_real(r)
        if r not in self.index:
            self.index[r] = len(self.slots)
            self.slots.append(r)
        return self.index[r]

    def op(self, kind, slots=(), k=0):
        s = list(slots)
        self.ops.append((kind, s + [-1] * (MAX_SLOTS - len(s)), k))

    # a ToGenerator value (K/Generator.scala:152-248)
    def value(self, t):
        if isinstance(t, core.Generator):
            self.generator(t)
        elif isinstance(t, core.Distribution):
            self.generator(t.generator)
        elif isinstance(t, Real):
            self.op(VALUE, [self.slot(t)])
            self.op(EMIT)
        elif isinstance(t, (tuple, list)):
            for u in t:
                self.value(u)
        else:
            raise Unsupported("no ToGenerator for %r" % (t,))

    def generator(self, g):
        if g.is_const:
            self.const(g.const)
        else:
            self.fn(g.fn)

    def const(self, c):
        if isinstance(c, (list, tuple)) and len(c) == 0:  # the start of traverse
            return
        raise Unsupported("constant generator value %r" % (c,))

    def fn(self, f):
        q, cl = f.__qualname__, _closure(f)
        if q == "Generator.repeat.<locals>.<lambda>":
            k = to_real(cl["k"])
            if not isinstance(k, Constant):
                raise Unsupported("repeat with a non-constant count")
            self.op(REPEAT, k=max(jd2i(k.getDouble()), 0))  # range(n.toInt(k))
            if "fromFn" in cl:
                self.fn(cl["fromFn"])
            else:
                self.const(cl["u"])
            self.op(END)
        elif q == "Generator.zip.<locals>.<lambda>":
            self.fn(cl["lf"]) if "lf" in cl else self.const(cl["t"])
            self.fn(cl["rf"]) if "rf" in cl else self.const(cl["u"])
        elif q == "Generator.map.<locals>.<lambda>" and cl["f"].__qualname__ == "Generator.traverse.<locals>.<lambda>":
            self.fn(cl["fromFn"])  # lr[0] + [lr[1]]: the flattened order is the evaluation order
        elif q in ("Generator.real.<locals>.<lambda>", "to_generator.<locals>.<lambda>"):
            self.op(VALUE, [self.slot(cl["x"] if "x" in cl else cl["t"])])
            self.op(EMIT)
        else:
            self.scalar(f)
            self.op(EMIT)

    def scalar(self, f):
        """one draw of a built-in distribution into v"""
        q, cl = f.__qualname__, _closure(f)
        if q == "Injection.transform.<locals>.<lambda>":
            dist_gen, inj = cl["distGen"], cl["inj"]
            if dist_gen.is_const:
                raise Unsupported("injection of a constant generator")
            self.scalar(dist_gen.fn)
            if isinstance(inj, core.Scale):
                self.op(SCALE, [self.slot(inj.a)])
            elif isinstance(inj, core.Translate):
                self.op(TRANSLATE, [self.slot(inj.b)])
            elif inj is core.Exp:
                self.op(EXP)
            else:
                raise Unsupported("injection %s" % type(inj).__name__)
        elif q == "LocationScaleFamily.__init__.<locals>.<lambda>":
            kinds = {id(core.Normal.generate): NORMAL, id(core.Cauchy.generate): CAUCHY, id(core.Laplace.generate): LAPLACE}
            if id(cl["generate"]) not in kinds:
                raise Unsupported("location-scale family %s" % cl["generate"].__qualname__)
            self.op(kinds[id(cl["generate"])])
        elif q == "Uniform.__new__.<locals>.<lambda>":
            self.op(UNIFORM)
        elif q == "Gamma.standard.<locals>.gen":
            self.op(GAMMA, [self.slot(cl["shape"])])
        elif q == "Generator.map.<locals>.<lambda>" and cl["f"].__qualname__ == "Beta.__init__.<locals>.<lambda>":
            # Gamma(a, 1).generator.zip(Gamma(b, 1).generator): two Scale(1) injections over Gamma.standard
            z = _closure(cl["fromFn"])
            shapes = [_closure(_closure(z[s])["distGen"].fn)["shape"] for s in ("lf", "rf")]
            self.op(BETA, [self.slot(shapes[0]), self.slot(shapes[1])])
        elif q == "Bernoulli.__init__.<locals>.gen":
            self.op(BERNOULLI, [self.slot(cl["p"])])
        elif q == "Geometric.__init__.<locals>.gen":
            self.op(GEOMETRIC, [self.slot(cl["p"])])
        elif q == "Poisson.__init__.<locals>.gen":
            self.op(POISSON, [self.slot(cl["lam"])])
        elif q == "Binomial.__init__.<locals>.gen":
            p, k = cl["p"], cl["k"]
            self.op(BINOMIAL, [self.slot(r) for r in (p, k, p * k, k * p, (k * p * (1 - p)).pow(0.5), to_real(p) + Real.zero)])
        elif q == "NegativeBinomial.__init__.<locals>.gen":
            p, n = cl["p"], cl["nn"]
            self.op(NEGBINOMIAL, [self.slot(r) for r in (p, n, 1 - p, n * p / (1 - p), (n * p).pow(1.0 / 2.0) / (1 - p))])
        elif q == "Generator.map.<locals>.<lambda>":
            raise Unsupported("map closure %s" % cl["f"].__qualname__)
        elif q == "Generator.flatMap.<locals>.inner":
            raise Unsupported("flatMap closure")
        elif q == "Generator.categorical.<locals>.fn":
            raise Unsupported("categorical")
        else:
            raise Unsupported("from / require closure %s" % q)


def m_out(ops):
    mult, emitted = [1], [0]
    for kind, _, k in ops:
        if kind == REPEAT:
            mult.append(k)
            emitted.append(0)
        elif kind == END:
            inner = emitted.pop() * mult.pop()
            emitted[-1] += inner
        elif kind == EMIT:
            emitted[-1] += 1
    return emitted[0]


def pack(function_rir, ops, m):
    """function container + plan -> generator container bytes"""
    rir = bytearray(function_rir)
    flags = struct.unpack_from("<I", rir, 28)[0]
    struct.pack_into("<I", rir, 28, flags | RIR_FLAG_GENERATOR)
    rir += GEN_HEADER.pack(len(ops), m, 0, 0)
    for kind, slots, k in ops:
        rir += GEN_OP.pack(kind, *slots, 0, k)
    return bytes(rir)


def lower_generator(t, parameters):
    """ToGenerator value t over the model's parameters -> RIR_FLAG_GENERATOR container bytes.  Raises Unsupported."""
    L = _Lowering()
    L.value(t)
    if not L.slots:  # a function container has at least one output
        L.slot(Real.zero)
    return pack(compile_function_rir(parameters, L.slots), L.ops, m_out(L.ops))


def slots_of(t):
    """the slot Reals of t's plan, in slot order (for tests and tooling)"""
    L = _Lowering()
    L.value(t)
    return L.slots or [Real.zero]

"""Python mirror of halo2-axiom 0.5.3 `plonk/evaluation.rs` for the quotient polynomial h(X) (SURVEY.md §8(f) rank 1)
and of `arithmetic::{eval_polynomial, kate_division}` (rank 4), on top of the C ABI of include/h2b200.h.

    GraphEvaluator        add_constant / add_rotation / add_calculation / add_expression  -> h2b_graph
    quotient_graph        custom gates:      values[i] = graph(previous = values[i])
    permutation_fold      the permutation argument's terms of `evaluate_h`
    lookup_fold           one lookup argument's five terms
    eval_polynomial, kate_division, poly_lincomb

The upstream file is not vendored under the reference tree; the program encoding is this library's own (see the header).
Expressions are nested tuples:  ("constant", fr) ("fixed", col, rot) ("advice", col, rot) ("instance", col, rot)
("challenge", i) ("negated", e) ("sum", a, b) ("product", a, b) ("scaled", e, fr),  fr = Montgomery [u64;4] limbs.
No field arithmetic happens here: constants are carried as limbs and everything is computed by the kernels."""
from __future__ import annotations
import ctypes as C
import numpy as np
from ._capi import lib, Graph
from .host import Context, _ptr, _u64

# value-source kinds / opcodes of include/h2b200.h
CONSTANT, INTERMEDIATE, FIXED, ADVICE, INSTANCE, CHALLENGE, BETA, GAMMA, THETA, Y, PREVIOUS = range(11)
ADD, SUB, MUL, SQUARE, DOUBLE, NEGATE, HORNER, STORE = range(8)
MAX_CALCULATIONS = 64

FR_ZERO = (0, 0, 0, 0)
FR_ONE = (0xAC96341C4FFFFFFB, 0x36FC76959F60CD29, 0x666EA36F7879462E, 0x0E0A77C19A07DF2F)  # R mod r
FR_TWO = (0x592C68389FFFFFF6, 0x6DF8ED2B3EC19A53, 0xCCDD46DEF0F28C5C, 0x1C14EF83340FBE5E)  # 2R mod r


def src(kind: int, index: int = 0, rot_slot: int = 0) -> tuple:
    return (kind, index, rot_slot)


def _word(s: tuple) -> int:
    kind, index, slot = s
    assert 0 <= index < 65536 and 0 <= slot < 4096
    return kind | (index << 4) | (slot << 20)


def _fr(x) -> tuple:
    return tuple(int(v) for v in np.asarray(x, dtype=np.uint64).reshape(4))


class GraphEvaluator:
    """`GraphEvaluator<C>`: constants start as [0, 1, 2]; calculation t writes intermediate t; identical
    calculations, constants and rotations are shared (as upstream does)."""

    def __init__(self):
        self.constants: list[tuple] = [FR_ZERO, FR_ONE, FR_TWO]
        self.rotations: list[int] = []
        self.calculations: list[tuple] = []  # (opcode, operands...) with HORNER = (HORNER, start, factor, (parts...))

    def add_rotation(self, rotation: int) -> int:
        if rotation not in self.rotations:
            self.rotations.append(rotation)
        return self.rotations.index(rotation)

    def add_constant(self, constant) -> tuple:
        c = _fr(constant)
        if c not in self.constants:
            self.constants.append(c)
        return src(CONSTANT, self.constants.index(c))

    def add_calculation(self, calc: tuple) -> tuple:
        if calc in self.calculations:
            return src(INTERMEDIATE, self.calculations.index(calc))
        assert len(self.calculations) < MAX_CALCULATIONS, "graph: too many calculations for one h2b_graph"
        self.calculations.append(calc)
        return src(INTERMEDIATE, len(self.calculations) - 1)

    def add_expression(self, e: tuple) -> tuple:
        zero, one, two = src(CONSTANT, 0), src(CONSTANT, 1), src(CONSTANT, 2)
        tag = e[0]
        if tag == "constant":
            return self.add_constant(e[1])
        if tag in ("fixed", "advice", "instance"):
            kind = {"fixed": FIXED, "advice": ADVICE, "instance": INSTANCE}[tag]
            return self.add_calculation((STORE, src(kind, e[1], self.add_rotation(e[2]))))
        if tag == "challenge":
            return self.add_calculation((STORE, src(CHALLENGE, e[1])))
        if tag == "negated":
            a = self.add_expression(e[1])
            return a if a == zero else self.add_calculation((NEGATE, a))
        if tag == "sum":
            if e[2][0] == "negated":  # a + (-b) is stored as a subtraction
                a, b = self.add_expression(e[1]), self.add_expression(e[2][1])
                if a == zero:
                    return self.add_calculation((NEGATE, b))
                return a if b == zero else self.add_calculation((SUB, a, b))
            a, b = self.add_expression(e[1]), self.add_expression(e[2])
            if a == zero:
                return b
            if b == zero:
                return a
            return self.add_calculation((ADD,) + tuple(sorted((a, b))))
        if tag == "product":
            a, b = self.add_expression(e[1]), self.add_expression(e[2])
            if a == zero or b == zero:
                return zero
            if a == one:
                return b
            if b == one:
                return a
            if a == two:
                return self.add_calculation((DOUBLE, b))
            if b == two:
                return self.add_calculation((DOUBLE, a))
            if a == b:
                return self.add_calculation((SQUARE, a))
            return self.add_calculation((MUL,) + tuple(sorted((a, b))))
        if tag == "scaled":
            f = _fr(e[2])
            if f == FR_ZERO:
                return zero
            if f == FR_ONE:
                return self.add_expression(e[1])
            cst = self.add_constant(f)
            return self.add_calculation((MUL, self.add_expression(e[1]), cst))
        raise ValueError(f"unknown expression {tag}")

    def add_gates(self, polynomials) -> tuple:
        """evaluate_h's custom-gate program: Horner(PreviousValue, [gate polynomials...], Y)"""
        parts = tuple(self.add_expression(p) for p in polynomials)
        return self.add_calculation((HORNER, src(PREVIOUS), src(Y), parts))

    def add_lookup(self, input_expressions, table_expressions) -> tuple:
        """a lookup argument's program: (theta-compressed inputs + beta) * (theta-compressed table + gamma)"""
        def compress(exprs):
            parts = tuple(self.add_expression(e) for e in exprs)
            return self.add_calculation((HORNER, src(CONSTANT, 0), src(THETA), parts))
        ci, ct = compress(input_expressions), compress(table_expressions)
        right_gamma = self.add_calculation((ADD, ct, src(GAMMA)))
        lc = self.add_calculation((ADD, ci, src(BETA)))
        return self.add_calculation((MUL, lc, right_gamma))

    def program(self) -> np.ndarray:
        words: list[int] = []
        for c in self.calculations:
            words.append(c[0])
            if c[0] == HORNER:
                words += [_word(c[1]), _word(c[2]), len(c[3])] + [_word(p) for p in c[3]]
            else:
                words += [_word(s) for s in c[1:]]
        return np.array(words, dtype=np.uint32)


class BoundGraph:
    """A GraphEvaluator bound to column tables and challenges: owns the arrays the h2b_graph struct points to."""

    def __init__(self, ev: GraphEvaluator, result: tuple, fixed=(), advice=(), instance=(), challenges=(), beta=FR_ZERO,
                 gamma=FR_ZERO, theta=FR_ZERO, y=FR_ZERO):
        self._prog = ev.program()
        self._consts = np.array(ev.constants, dtype=np.uint64).reshape(-1, 4)
        self._rots = np.array(ev.rotations or [0], dtype=np.int32)
        self._chal = np.array([_fr(c) for c in challenges], dtype=np.uint64).reshape(-1, 4)
        # keeps the (contiguous) ndarrays alive; plain ints are device pointers for the `_dev` entry points
        self._cols = [[c if isinstance(c, int) else np.ascontiguousarray(c, dtype=np.uint64) for c in cols]
                      for cols in (fixed, advice, instance)]

        def table(cols):
            ptrs = [c if isinstance(c, int) else c.ctypes.data for c in cols]
            return (C.c_void_p * max(len(ptrs), 1))(*ptrs), len(ptrs)
        self._tables = [table(c) for c in self._cols]
        g = Graph()
        g.program = self._prog.ctypes.data_as(C.POINTER(C.c_uint32))
        g.program_words = len(self._prog)
        g.n_calculations = len(ev.calculations)
        g.result = _word(result)
        g.constants = self._consts.ctypes.data
        g.n_constants = len(self._consts)
        g.rotations = self._rots.ctypes.data_as(C.POINTER(C.c_int32))
        g.n_rotations = len(ev.rotations)
        (g.fixed, g.n_fixed), (g.advice, g.n_advice), (g.instance, g.n_instance) = [
            (C.cast(t, C.POINTER(C.c_void_p)), n) for t, n in self._tables]
        g.challenges = self._chal.ctypes.data if len(self._chal) else None
        g.n_challenges = len(self._chal)
        for name, v in (("beta", beta), ("gamma", gamma), ("theta", theta), ("y", y)):
            setattr(g, name, (C.c_uint64 * 4)(*_fr(v)))
        self.struct = g


def _cols(arrs):
    return [np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4) for a in arrs]


def _table(cols):
    return (C.c_void_p * max(len(cols), 1))(*[c.ctypes.data for c in cols])


def quotient_graph(ctx: Context, graph: BoundGraph, k: int, ext_k: int, values) -> np.ndarray:
    """`*value = custom_gates.evaluate(.., previous_value = *value, idx, ..)` for every extended-domain row"""
    v = _u64(values, 4).copy()
    ctx.check(lib.h2b_quotient_graph(ctx.h, C.byref(graph.struct), k, ext_k, _ptr(v)))
    return v


def lookup_fold(ctx: Context, graph: BoundGraph, z, permuted_input, permuted_table, l0, l_last, l_active, k: int, ext_k: int,
                values) -> np.ndarray:
    a = _cols([z, permuted_input, permuted_table, l0, l_last, l_active])
    v = _u64(values, 4).copy()
    ctx.check(lib.h2b_lookup_fold(ctx.h, C.byref(graph.struct), *[_ptr(x) for x in a], k, ext_k, _ptr(v)))
    return v


def permutation_fold(ctx: Context, z_sets, columns, sigma, chunk_len: int, l0, l_last, l_active, beta, gamma, y,
                     blinding_factors: int, k: int, ext_k: int, values) -> np.ndarray:
    zs, cs, ss = _cols(z_sets), _cols(columns), _cols(sigma)
    ls = _cols([l0, l_last, l_active])
    ch = _cols([beta, gamma, y])  # held in locals: the pointers below must outlive the call
    v = _u64(values, 4).copy()
    ctx.check(lib.h2b_permutation_fold(ctx.h, _table(zs), len(zs), _table(cs), _table(ss), len(cs), chunk_len, *[_ptr(x) for x in ls],
                                       *[_ptr(x) for x in ch], blinding_factors, k, ext_k, _ptr(v)))
    return v


def divide_by_vanishing_poly(ctx: Context, values, k: int, ext_k: int) -> np.ndarray:
    """EvaluationDomain::divide_by_vanishing_poly on the extended coset"""
    v = _u64(values, 4).copy()
    ctx.check(lib.h2b_divide_by_vanishing_poly(ctx.h, _ptr(v), k, ext_k))
    return v


def eval_polynomial(ctx: Context, poly, point) -> np.ndarray:
    """arithmetic::eval_polynomial(poly, point)"""
    a, x = _u64(poly, 4), _u64(point, 4)
    out = np.empty(4, dtype=np.uint64)
    ctx.check(lib.h2b_eval_polynomial(ctx.h, _ptr(a) if len(a) else None, len(a), _ptr(x), _ptr(out)))
    return out


def kate_division(ctx: Context, a, b) -> np.ndarray:
    """arithmetic::kate_division(a, b): quotient of a(X) by (X - b), remainder dropped"""
    a, z = _u64(a, 4), _u64(b, 4)
    q = np.empty((max(len(a), 1) - 1, 4), dtype=np.uint64)
    ctx.check(lib.h2b_kate_division(ctx.h, _ptr(a) if len(a) else None, len(a), _ptr(z), _ptr(q) if len(q) else None))
    return q


def poly_lincomb(ctx: Context, polys, scalars) -> np.ndarray:
    """sum_j scalars[j] * polys[j]"""
    ps = _cols(polys)
    s = _u64(scalars, 4)
    assert len(s) == len(ps)
    out = np.empty_like(ps[0])
    ctx.check(lib.h2b_poly_lincomb(ctx.h, _table(ps), _ptr(s), len(ps), len(ps[0]), _ptr(out) if len(out) else None))
    return out


def permute_expression_pair(ctx: Context, input_expression, table_expression, k: int, blinding_factors: int):
    """plonk/lookup/prover.rs `permute_expression_pair`: returns (permuted_input, permuted_table), 2^k rows each; the
    last blinding_factors + 1 rows are left zero for the caller's blinding scalars.  Raises ConstraintSystemFailure."""
    a, t = _u64(input_expression, 4), _u64(table_expression, 4)
    assert len(a) == len(t) == 1 << k
    pa, pt = np.zeros_like(a), np.zeros_like(t)
    ctx.check(lib.h2b_permute_expression_pair(ctx.h, _ptr(a), _ptr(t), k, blinding_factors, _ptr(pa), _ptr(pt)))
    return pa, pt

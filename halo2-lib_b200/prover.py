"""Resident prover: the device-side data flow of halo2-axiom 0.5.3 `create_proof` for the constraint system halo2-base
builds (one vertical gate per gate-advice column, halo2-base/src/gates/flex_gate/mod.rs:80-91; a range lookup
`q_lookup * a in table`, gates/range/mod.rs:92-94,131-141; equality on the constants column and the gate column,
flex_gate/mod.rs:69,124-129), with every column kept in HBM behind `h2b_poly` handles between the phases.

The proof sequence and the constraint check are implemented once, in C++ (include/h2b200_prover.hpp: ProverCircuit and
ProverSession); `Circuit` and `ProverSession` here bind them through the library's private calls
(halo2-lib_b200/csrc/prover_binding.cu).  Python supplies the inputs (host pointers), the blinding scalars (drawn from
`np.random.default_rng(seed)` in the order the prover asks for them) and, for verification runs, receives the committed
polynomials; the transcript, the challenges and every device call stay in the compiled prover."""
from __future__ import annotations
import ctypes as C
import numpy as np
from ._capi import lib, CHECK_MAX_REPORT, Witness, BuilderView, BLIND_FN, ALLREDUCE_FN, COMMIT_FN
from .host import Context, ParamsKZG

R_MOD = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
MONT_R = (1 << 256) % R_MOD
MONT_RINV = pow(1 << 256, -1, R_MOD)
ROOT_OF_UNITY = pow(7, (R_MOD - 1) >> 28, R_MOD)
DELTA = pow(7, 1 << 28, R_MOD)


def to_limbs(x: int) -> np.ndarray:
    """canonical integer -> Montgomery [u64;4]"""
    v = x % R_MOD * MONT_R % R_MOD
    return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def from_limbs(l) -> int:
    """Montgomery [u64;4] -> canonical integer"""
    return sum(int(v) << (64 * i) for i, v in enumerate(np.asarray(l, dtype=np.uint64).reshape(4))) * MONT_RINV % R_MOD


P_MOD = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
_PR, _PRINV = (1 << 256) % P_MOD, pow(1 << 256, -1, P_MOD)


_PR2, _PR3 = pow(_PR, 2, P_MOD), pow(_PR, 3, P_MOD)
_ONE_BYTES = _PR.to_bytes(32, "little")


def g1_normalize_host(pt) -> np.ndarray:
    """Jacobian (X, Y, Z), Montgomery limbs -> (X / Z^2, Y / Z^3, 1); the identity -> all zero.  The form in which a
    commitment enters the transcript and the proof (the accumulation order inside an MSM is not deterministic, so the
    Jacobian representative is not either; the affine point is), restated on Python integers: the reference the compiled
    prover's batch normalisation is tested against.  (Montgomery domain throughout: with Xm = X R, Zm = Z R the result x R
    is Xm R^2 / Zm^2.)"""
    b = np.ascontiguousarray(pt, dtype=np.uint64).tobytes()
    xm, ym, zm = (int.from_bytes(b[32 * j:32 * j + 32], "little") for j in range(3))
    if zm == 0:
        return np.zeros(12, dtype=np.uint64)
    zi = pow(zm, -1, P_MOD)
    zi2 = zi * zi % P_MOD
    x = xm * zi2 % P_MOD * _PR2 % P_MOD
    y = ym * zi2 % P_MOD * zi % P_MOD * _PR3 % P_MOD
    return np.frombuffer(x.to_bytes(32, "little") + y.to_bytes(32, "little") + _ONE_BYTES, dtype=np.uint64)


class Poly:
    """h2b_poly: a device-resident column / polynomial"""

    def __init__(self, ctx: Context, n: int):
        self.ctx, self.n = ctx, n
        h = C.c_void_p()
        ctx.check(lib.h2b_poly_alloc(ctx.h, n, C.byref(h)))
        self.h = h
        self.ptr = int(lib.h2b_poly_device_ptr(h))

    def upload(self, host: np.ndarray, offset: int = 0):
        a = np.ascontiguousarray(host, dtype=np.uint64).reshape(-1, 4)
        self.ctx.check(lib.h2b_poly_upload(self.ctx.h, self.h, offset, C.c_void_p(a.ctypes.data), len(a)))

    def upload_ptr(self, host_ptr: int, n: int, offset: int = 0):
        self.ctx.check(lib.h2b_poly_upload(self.ctx.h, self.h, offset, C.c_void_p(host_ptr), n))

    def download(self, offset: int = 0, n: int | None = None) -> np.ndarray:
        n = self.n - offset if n is None else n
        out = np.empty((n, 4), dtype=np.uint64)
        self.ctx.check(lib.h2b_poly_download(self.ctx.h, self.h, offset, C.c_void_p(out.ctypes.data), n))
        return out

    def at(self, elem_offset: int) -> int:
        return self.ptr + 32 * elem_offset

    def free(self):
        if self.h:
            lib.h2b_poly_free(self.ctx.h, self.h)
            self.h = None


def _rows(a, n: int, what: str) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4)
    if len(a) != n:
        raise ValueError("Circuit: column %s must hold 2^k rows" % what)
    return a


class Column:
    """A read-only view of rows of a device polynomial the compiled prover owns (valid while its circuit / session lives)"""

    def __init__(self, ctx: Context, poly: C.c_void_p, offset: int, n: int):
        self.ctx, self.poly, self.offset, self.n = ctx, poly, offset, n
        self.ptr = int(lib.h2b_poly_device_ptr(poly)) + 32 * offset

    def download(self, offset: int = 0, n: int | None = None) -> np.ndarray:
        n = self.n - offset if n is None else n
        out = np.empty((n, 4), dtype=np.uint64)
        self.ctx.check(lib.h2b_poly_download(self.ctx.h, self.poly, self.offset + offset, C.c_void_p(out.ctypes.data), n))
        return out

    def at(self, elem_offset: int) -> int:
        return self.ptr + 32 * elem_offset


class _Columns:
    """name -> Column of one table of a circuit or session"""

    def __init__(self, owner, table: str):
        self.owner, self.table = owner, table

    def __getitem__(self, name: str) -> Column:
        return self.owner.column(self.table, name)


def _column(ctx: Context, fn, h, table: str, name: str) -> Column:
    poly, off, rows = C.c_void_p(), C.c_size_t(), C.c_size_t()
    ctx.check(fn(h, table.encode(), name.encode(), C.byref(poly), C.byref(off), C.byref(rows)))
    return Column(ctx, poly, off.value, rows.value)


class Circuit:
    """The fixed side of a synthetic halo2-base circuit (what keygen_pk would hold), resident on the GPU in the three forms
    create_proof needs: Lagrange values, coefficients, extended-coset evaluations (h2b::ProverCircuit).

    Shape (halo2-base `BaseCircuitParams`: num_advice_per_phase, num_lookup_advice_per_phase, num_fixed = F):
      A gate-advice columns a0..a{A-1}, each with its selector q{j} and the vertical gate (flex_gate/mod.rs:80-91);
      L lookup-advice columns l0..l{L-1}, each looked up in `table` as it is (range/mod.rs:131-150); with L = 0 the one
      lookup is `q_lookup * a0 in table` (range/mod.rs:92-94), or none at all with selector_lookup = False;
      F constants columns c, c1..c{F-1} (F = 0: none); I instance columns i0..i{I-1} (BaseConfig::configure,
      gates/circuit/mod.rs:87-93); equality on [c, c1.., a0.., l0.., i0..] in that order (the permutation's column order).
    The shape numbers and column names are read from the compiled circuit.  `lagr`, `coeff`, `ext` (by column name) and
    `sigma_map` (the decoded sigma of the check) look up its device columns.

    compress_selectors: lay the fixed side out as halo2's keygen_vk does (DESIGN.md §4.13).  The columns passed are the same
    (q{j}, [q_lookup], [table], c..; every selector value 0 or 1); the circuit combines the selectors into the columns s0, s1..
    itself.  `fixed_names` lists the fixed columns in column order (the vk's), `fixed_queries` in query order (the evaluations
    and openings), and `selectors` maps each selector to (column, root, combination length); without compression every
    selector is its own column with root 1 and both orders are q0.., [q_lookup], [table], c.."""

    def __init__(self, ctx: Context, k: int, fixed_lagrange: dict, sigma_lagrange: list, A: int = 1, L: int = 0,
                 selector_lookup: bool = True, I: int = 0, F: int = 1, compress_selectors: bool = False):
        n = 1 << k
        fixed = {nm: _rows(a, n, nm) for nm, a in fixed_lagrange.items()}
        sigma = [_rows(a, n, "sigma %d" % i) for i, a in enumerate(sigma_lagrange)]
        names = (C.c_char_p * len(fixed))(*[nm.encode() for nm in fixed])
        ptrs = (C.c_void_p * len(fixed))(*[a.ctypes.data for a in fixed.values()])
        sptrs = (C.c_void_p * len(sigma))(*[a.ctypes.data for a in sigma])
        h = C.c_void_p()
        ctx.check(lib.h2bp_circuit_create(ctx.h, k, A, L, int(selector_lookup), I, F, names, ptrs, len(fixed), sptrs, len(sigma), C.byref(h),
                                          int(compress_selectors)))
        self._bind(ctx, k, A, L, h)

    def _bind(self, ctx: Context, k: int, A: int, L: int, h: C.c_void_p):
        """take ownership of a compiled circuit and read its shape and column names"""
        self.ctx, self.k, self.n, self.A, self.L = ctx, k, 1 << k, A, L
        self._h = h
        shape, text = (C.c_uint64 * 8)(), C.create_string_buffer(1 << 16)
        ctx.check(lib.h2bp_circuit_info(h, shape, text, len(text)))
        self.degree, self.chunk, self.ext_k, self.bf, self.u, self.n_sets, self.n_lookups, sel = (int(v) for v in shape)
        self.selector_lookup = bool(sel)
        lists = {key: v.split(",") if v else [] for key, v in (line.split("=", 1) for line in text.value.decode().split("\n"))}
        self.adv_names, self.perm_cols, self.fixed_names, self.sigma_names, self.const_names = (
            lists[key] for key in ("adv", "perm", "fixed", "sigma", "const"))
        self.fixed_queries = lists["queries"]
        self.selectors = {nm: (col, int(root), int(ln)) for nm, col, root, ln in (e.split(":") for e in lists["selectors"])}
        self.compressed = any(col != nm for nm, (col, _, _) in self.selectors.items())
        self.F = len(self.const_names)
        self.I = len(self.perm_cols) - self.F - A - L
        self.lagr, self.coeff, self.ext = _Columns(self, "lagr"), _Columns(self, "coeff"), _Columns(self, "ext")

    def column(self, table: str, name: str = "") -> Column:
        return _column(self.ctx, lib.h2bp_circuit_column, self._h, table, name)

    @property
    def sigma_map(self) -> Column:
        """map[c][r] = c' << k | r' (u32, perm_cols order), decoded on first use; raises H2BError naming the first (column,
        row) whose sigma entry is not delta^c' omega^r' for a permutation column c'"""
        return self.column("sigma_map")

    def free(self):
        if self._h:
            lib.h2bp_circuit_free(self._h)
            self._h = None


def synthetic_circuit(ctx: Context, k: int, rng: np.random.Generator, lookup_bits: int = 8, A: int = 1, L: int = 0,
                      selector_lookup: bool = True):
    """A SATISFIED instance of the shape above.  Returns a dict:
      cols        the A + L advice columns as the assignment must produce them (n x 4 Montgomery limbs each),
      virtual     the virtual column V of the gate cells (ctx.advice concatenated over the threads) and `break_points`
                  (App. A.2: column j takes V[start_j .. start_j + bp_j], the break cell is copied into the next column),
      lookup      the cells to look up in `assign_raw` order (cell i goes to lookup column i mod L, row i div L),
      fixed, sigma, usable.
    Gates on rows 4i..4i+3 of every gate column (a3 = a0 + a1*a2, computed on the GPU); the small operands a1 are looked
    up — through q_lookup on a0's column when L = 0, through copies into the lookup-advice columns otherwise (with the
    copy constraints halo2-base adds); every bit cell a2 is tied into one cycle with the constant cell of its value."""
    n = 1 << k
    usable = n - 20
    G = usable // 4 if A == 1 else (usable - 4) // 4       # gates per column
    lookup_bits = min(lookup_bits, k - 2)                   # the table's 2^bits rows must fit the usable rows
    mont_small = lambda v: ctx.field_op(1, 5, np.stack([v.astype(np.uint64)] + [np.zeros(len(v), dtype=np.uint64)] * 3, axis=1))
    one = to_limbs(1)
    rows = 4 * np.arange(G)
    cols, a1_all, a2_all = [], [], []
    for j in range(A):
        a0c = rng.integers(0, 1 << 62, size=G, dtype=np.int64).astype(np.uint64)
        a1c = rng.integers(0, 1 << lookup_bits, size=G, dtype=np.int64).astype(np.uint64)  # looked up
        a2c = rng.integers(0, 2, size=G, dtype=np.int64).astype(np.uint64)                # bits: many equal cells
        A0, A1, A2 = mont_small(a0c), mont_small(a1c), mont_small(a2c)
        A3 = ctx.field_op(1, 1, A0, ctx.field_op(1, 0, A1, A2))
        col = np.zeros((n, 4), dtype=np.uint64)
        col[rows], col[rows + 1], col[rows + 2], col[rows + 3] = A0, A1, A2, A3
        cols.append(col)
        a1_all.append(A1)
        a2_all.append(a2c)
    # the virtual column: the gate cells of every column back to back; break point 4G: the cell at row 4G of column j is
    # the copy of column j + 1's first cell that the walk makes
    virtual = np.concatenate([c[: 4 * G] for c in cols]) if A > 1 else cols[0][:usable].copy()
    break_points = np.array([4 * G] * (A - 1), dtype=np.uint64)
    for j in range(A - 1):
        cols[j][4 * G] = cols[j + 1][0]
    fixed = {}
    for j in range(A):
        q = np.zeros((n, 4), dtype=np.uint64); q[rows] = one
        fixed["q%d" % j] = q
    t = np.zeros((n, 4), dtype=np.uint64)
    t[: 1 << lookup_bits] = mont_small(np.arange(1 << lookup_bits, dtype=np.uint64))
    fixed["table"] = t
    c = np.zeros((n, 4), dtype=np.uint64)
    c[0], c[1] = to_limbs(0), one
    fixed["c"] = c
    # ---- lookups
    lookup_cells = np.zeros((0, 4), dtype=np.uint64)
    lk_src = []  # (gate column, row) of the cell copied into lookup cell i
    if L == 0:
        if selector_lookup:
            qlk = np.zeros((n, 4), dtype=np.uint64); qlk[rows + 1] = one
            fixed["q_lookup"] = qlk
    else:
        cap = L * (usable - 7)
        per_col = min(G, cap // A)
        lookup_cells = np.concatenate([a1_all[j][:per_col] for j in range(A)])
        lk_src = [(j, 4 * i + 1) for j in range(A) for i in range(per_col)]
        for tcol in range(L):
            col = np.zeros((n, 4), dtype=np.uint64)
            part = lookup_cells[tcol::L]
            col[: len(part)] = part
            cols.append(col)
    # ---- permutation: identity values delta^c * omega^i per permutation column c, then the cycles
    w = pow(ROOT_OF_UNITY, 1 << (28 - k), R_MOD)
    wp = _geometric(ctx, w, n)                       # omega^i, Montgomery limbs
    ids = [wp]
    for cidx in range(1, 1 + A + L):
        ids.append(ctx.field_op(1, 0, ids[-1], np.tile(to_limbs(DELTA), (n, 1))))
    ids = np.stack(ids)                               # [perm column][row]
    sig = ids.copy()

    def tie(pc, pr):
        """one cycle through the cells (permutation column pc[i], row pr[i])"""
        pc, pr = np.asarray(pc), np.asarray(pr)
        if len(pc) > 1:
            sig[pc, pr] = ids[np.roll(pc, -1), np.roll(pr, -1)]
    for bit in (0, 1):  # c[bit] -> every advice cell that holds `bit`
        pc, pr = [np.array([0])], [np.array([bit])]
        for j in range(A):
            cells = rows[a2_all[j] == bit] + 2
            pc.append(np.full(len(cells), 1 + j)); pr.append(cells)
        tie(np.concatenate(pc), np.concatenate(pr))
    if L:  # the copies into the lookup-advice columns: 2-cycles, all at once
        i = np.arange(len(lk_src))
        src_c = np.array([1 + j for j, _ in lk_src]); src_r = np.array([r for _, r in lk_src])
        dst_c = 1 + A + (i % L); dst_r = i // L
        sig[src_c, src_r] = ids[dst_c, dst_r]
        sig[dst_c, dst_r] = ids[src_c, src_r]
    return {"cols": cols, "virtual": virtual, "break_points": break_points, "lookup": lookup_cells, "fixed": fixed,
            "sigma": [sig[cidx] for cidx in range(1 + A + L)], "usable": usable, "A": A, "L": L}


def _geometric(ctx: Context, w: int, n: int) -> np.ndarray:
    """[w^0, w^1, ..., w^(n-1)] as Montgomery limbs, by doubling with the GPU's element-wise multiplier"""
    out = np.zeros((n, 4), dtype=np.uint64)
    out[0] = to_limbs(1)
    have, step = 1, w
    while have < n:
        m = min(have, n - have)
        out[have:have + m] = ctx.field_op(1, 0, out[:m], np.tile(to_limbs(pow(w, have, R_MOD)), (m, 1)))
        have += m
    return out


def _reports(words: np.ndarray, max_report: int) -> list:
    """report rows of max_report + 1 words (the failure count, then the rows) -> [(count, the first min(count, max_report) rows)]"""
    return [(int(r[0]), [int(x) for x in r[1:1 + min(int(r[0]), max_report)]]) for r in words]


def _instance_columns(who: str, I: int, columns, width: int):
    """(pointer array, length array, the arrays) of I instance columns: `columns` a list of I arrays (uint64 indices, width 1, or
    Montgomery values, width 4); None: every column empty"""
    cols = [()] * I if columns is None else list(columns)
    if len(cols) != I:
        raise ValueError("%s: %d instance columns for a circuit with %d" % (who, len(cols), I))
    arrs = [np.ascontiguousarray(c, dtype=np.uint64).reshape(-1, width) for c in cols]
    ptrs = (C.c_void_p * max(I, 1))(*[a.ctypes.data if a.size else None for a in arrs])
    lens = (C.c_size_t * max(I, 1))(*[len(a) for a in arrs])
    return ptrs, lens, arrs


def _builder_view(who: str, n_cells: int, selectors, advice_equalities, constant_equalities, lookups, cells=None, rational_index=None,
                  rational_den=None, I: int = 0, instances=None, public=None):
    """(BuilderView, the arrays it points to) of a builder in MockProver's form; instances: per instance column the indices of
    its cells, public: per instance column its values (MockProver)"""
    u64 = lambda a: np.ascontiguousarray(a, dtype=np.uint64)
    V = u64(np.zeros((0, 4)) if cells is None else cells).reshape(-1, 4)
    S = np.ascontiguousarray(selectors, dtype=np.uint8).reshape(-1)
    if len(S) != n_cells:
        raise ValueError(who + ": one selector per cell")
    E = u64(advice_equalities).reshape(-1, 2)
    ce, ci = (np.zeros((0, 4)), []) if constant_equalities is None else constant_equalities
    Kc, Ki = u64(ce).reshape(-1, 4), u64(ci).reshape(-1)
    if len(Kc) != len(Ki):
        raise ValueError(who + ": one index per constant")
    LK = u64(lookups).reshape(-1)
    RI = u64([] if rational_index is None else rational_index).reshape(-1)
    RD = u64(np.zeros((0, 4)) if rational_den is None else rational_den).reshape(-1, 4)
    if len(RI) != len(RD):
        raise ValueError(who + ": rational_index and rational_den differ in length")
    p = lambda a: a.ctypes.data if a.size else None
    view = BuilderView(p(V), n_cells, p(RI), p(RD), len(RI), p(S), p(E), len(E), p(Kc), p(Ki), len(Ki), p(LK), len(LK))
    ip, il, ia = _instance_columns(who, I, instances, 1)
    keep = (V, S, E, Kc, Ki, LK, RI, RD, ip, il, ia)
    if I:
        view.instance_index, view.n_instance, view.n_instance_columns = C.cast(ip, C.c_void_p), C.cast(il, C.c_void_p), I
        if public is not None:
            vp, vl, va = _instance_columns(who, I, public, 4)
            if list(vl)[:I] != list(il)[:I]:
                raise ValueError(who + ": one public value per instance cell")
            view.instance_values = C.cast(vp, C.c_void_p)
            keep += (vp, vl, va)
    return view, keep


def keygen(ctx: Context, params: ParamsKZG, k: int, A: int = 1, L: int = 0, selector_lookup: bool = True, lookup_bits: int = 8,
           max_rows: int | None = None, selectors=(), advice_equalities=(), constant_equalities=None, lookups=(), timings: dict | None = None,
           I: int = 0, instances=None, F: int = 1, compress_selectors: bool = False):
    """keygen_vk + keygen_pk of a halo2-base builder in its keygen form, on the device (h2b::keygen, include/h2b200_keygen.hpp).

    The arguments mean what they mean for MockProver.run (selectors: one per cell of the virtual column, which fixes its length;
    no witness values are read).  sigma is the one halo2's permutation Assembly builds from halo2-base's copy calls, bit for bit.
    I instance columns, `instances` the indices of each one's cells (BaseCircuitBuilder::assigned_instances; None: all empty):
    their copies follow the region's.  F constants columns c, c1.. (BaseCircuitParams::num_fixed, 0 when the builder has no
    constant equalities): distinct constant d of the sorted order goes to column d mod F, row d div F.
    Returns (circuit, vk, break_points): `circuit` is a Circuit that ProverSession takes; vk = {"fixed": {name: commitment},
    "permutation": [commitment per permutation column, perm_cols order]}, each commitment affine as 12 Montgomery limbs
    (x, y, 1; the identity all zero), of the column's Lagrange values.  halo2-base's panics raise H2BError with its message.
    `timings`, when a dict, receives the milliseconds of the phases copies / forest / sigma / pk / vk.
    compress_selectors: keygen_vk's selector compression (see Circuit; its time counts in `pk`): vk["fixed"] then holds halo2's
    fixed columns in halo2's column order, [table], c.., s0, s1.."""
    max_rows = (1 << k) - 9 if max_rows is None else max_rows
    n_cells = len(np.asarray(selectors).reshape(-1))
    view, keep = _builder_view("keygen", n_cells, selectors, advice_equalities, constant_equalities, lookups, I=I, instances=instances)
    bps, nbp = np.zeros(max(A, 1), dtype=np.uint64), C.c_uint64()
    n_fixed = A + (1 if selector_lookup and L == 0 else 0) + (1 if L or selector_lookup else 0) + F
    vk = np.zeros((n_fixed + F + A + L + I, 12), dtype=np.uint64)
    times = np.zeros(5, dtype=np.float64)
    h = C.c_void_p()
    ctx.check(lib.h2bp_keygen(ctx.h, params.h, k, params.count, A, L, int(selector_lookup), lookup_bits, max_rows, F, C.byref(view), C.byref(h),
                              C.c_void_p(bps.ctypes.data), C.byref(nbp), C.c_void_p(vk.ctypes.data), C.c_void_p(times.ctypes.data),
                              int(compress_selectors)))
    cs = Circuit.__new__(Circuit)
    cs._bind(ctx, k, A, L, h)
    if timings is not None:
        timings.update(zip(("copies", "forest", "sigma", "pk", "vk"), (float(t) for t in times)))
    nf = len(cs.fixed_names)
    out = {"fixed": {nm: vk[i] for i, nm in enumerate(cs.fixed_names)}, "permutation": list(vk[nf:nf + len(cs.perm_cols)])}
    return cs, out, [int(b) for b in bps[:nbp.value]]


class ProverSession:
    """One proof at a time on one context (h2b::ProverSession): owns the resident working set, allocated once and reused for
    every proof.  `lagr`, `coef`, `ext` (by column name), `h` and `check_report` look up its device columns."""

    def __init__(self, ctx: Context, params: ParamsKZG, circuit: Circuit):
        self.ctx, self.params, self.cs = ctx, params, circuit
        h = C.c_void_p()
        ctx.check(lib.h2bp_session_create(ctx.h, params.h, circuit.k, params.count, circuit._h, C.byref(h)))
        self._h = h
        counts, text = (C.c_uint64 * 2)(), C.create_string_buffer(1 << 16)
        ctx.check(lib.h2bp_session_info(h, counts, text, len(text)))
        self.n_commitments = int(counts[0])
        self.queries = [(nm, int(r)) for nm, r in (q.rsplit(":", 1) for q in text.value.decode().split(","))]
        self.lagr, self.coef, self.ext = _Columns(self, "lagr"), _Columns(self, "coef"), _Columns(self, "ext")
        self.keep = None  # verification runs: dict that receives the committed polynomials (downloaded, untimed)
        self.blind_log = None
        self.blind_source = None  # optional callable rows -> (rows, 4) Montgomery limbs (tests: replay a fixed proof)
        self._rng = self._error = None
        self._blind_cb = BLIND_FN(lambda _, rows, out: self._guard(self._blind, rows, out))
        self._commit_cb = COMMIT_FN(lambda _, basis, rows, n: self._guard(self._committed, basis, rows, n))
        self._allreduce_cb = None

    def shard(self, begin: int, n_loc: int, allreduce):
        """multi-GPU: this rank commits rows [begin, begin + n_loc) of every polynomial and `allreduce(ptr, m)` combines the
        partial commitments of all ranks in place on the device (h2b_g1_allreduce_dev); everything else is replicated"""
        self._allreduce_cb = ALLREDUCE_FN(lambda _, ptr, m: self._guard(allreduce, ptr, m))
        self.ctx.check(lib.h2bp_session_shard(self._h, begin, n_loc, self._allreduce_cb, None))

    def column(self, table: str, name: str = "") -> Column:
        return _column(self.ctx, lib.h2bp_session_column, self._h, table, name)

    @property
    def h(self) -> Column:
        """the quotient: values on the extended coset, then the coefficients of its degree - 1 pieces of n"""
        return self.column("h")

    @property
    def check_report(self) -> Column:
        """the report block of the last check"""
        return self.column("check_report")

    # ---- callbacks of the compiled prover: an exception is kept for the caller and stops the proof
    def _guard(self, fn, *args) -> int:
        try:
            fn(*args)
            return 0
        except BaseException as e:  # noqa: B036 (re-raised by _done)
            self._error = e
            return 1

    def _blind(self, rows: int, out: int):
        if self.blind_source is not None:  # the caller's blinding scalars (Montgomery limbs), in the order of use
            b = np.ascontiguousarray(self.blind_source(rows), dtype=np.uint64).reshape(rows, 4)
        else:
            b = self._rng.integers(0, 1 << 62, size=(rows, 4), dtype=np.int64).astype(np.uint64)
            b[:, 3] &= np.uint64((1 << 60) - 1)
        if self.blind_log is not None:  # the blinding rows in the order of use (a replay feeds them back)
            self.blind_log.append(b)
        C.memmove(out, b.ctypes.data, b.nbytes)

    def _committed(self, basis: int, rows: int, n: int):
        arr = np.empty((n, 4), dtype=np.uint64)
        C.memmove(arr.ctypes.data, rows, 32 * n)
        self.keep.setdefault("committed", []).append((basis, arr))

    def _done(self, rc: int):
        err, self._error = self._error, None
        if err is not None:
            raise err
        self.ctx.check(rc)

    def _witness(self, who, witness_ptr, n_cells, break_points, lookup_ptr, n_lookup, rational_index_ptr, rational_den_ptr, n_rational,
                 lookup_index_ptr, instances=None):
        """(Witness, the arrays it points to)"""
        if lookup_ptr and lookup_index_ptr:
            raise ValueError(who + ": pass the looked-up cells either as values (lookup_ptr) or as indices (lookup_index_ptr)")
        if n_rational and not (rational_index_ptr and rational_den_ptr):
            raise ValueError(who + ": n_rational > 0 needs rational_index_ptr and rational_den_ptr")
        bp = np.ascontiguousarray([] if break_points is None else break_points, dtype=np.uint64).reshape(-1)
        w = Witness(witness_ptr or None, n_cells, bp.ctypes.data if len(bp) else None, len(bp), lookup_ptr or None,
                    lookup_index_ptr or None, n_lookup, rational_index_ptr or None, rational_den_ptr or None, n_rational)
        I = self.cs.I
        inst = _instance_columns(who, I, instances, 4)
        if I:
            w.instance, w.n_instance, w.n_instance_columns = C.cast(inst[0], C.c_void_p), C.cast(inst[1], C.c_void_p), I
        return w, (bp, inst)

    def check(self, witness_ptr: int, n_cells: int, break_points=None, lookup_ptr: int = 0, n_lookup: int = 0, rational_index_ptr: int = 0,
              rational_den_ptr: int = 0, n_rational: int = 0, lookup_index_ptr: int = 0, max_report: int = 16, instances=None) -> dict:
        """MockProver::verify for this circuit: which gates, lookups and copy constraints the witness breaks, and where.
        Takes the witness exactly as `prove` does and runs the same assignment; no blinding, no random polynomial, no transcript.
        The values checked are the ones a proof would commit before blinding, with rows >= u read as 0:
          gates[j]    rows r < u with q{j}(r) (a{j}(r) + a{j}(r+1) a{j}(r+2) - a{j}(r+3)) != 0 (rotations mod n);
          lookups[t]  rows r < u whose input (q_lookup * a0, or l{t}) is not among the table's rows [0, u);
          copies[c]   rows r < n of permutation column c (perm_cols order) whose value differs from the cell sigma_c(r) names;
                      an instance column holds the public values `instances` (as for `prove`) at rows [0, len), zero after.
        Each entry is (failure count, the first min(count, max_report) failing rows ascending).  Every report comes down in one
        copy.  A bad halo2-base index raises H2BError; so does a sigma entry that names no cell (on the circuit's first check)."""
        w, keep = self._witness("check", witness_ptr, n_cells, break_points, lookup_ptr, n_lookup, rational_index_ptr, rational_den_ptr,
                                n_rational, lookup_index_ptr, instances)
        if not 1 <= max_report <= CHECK_MAX_REPORT:
            raise ValueError("check: max_report must be in 1..%d" % CHECK_MAX_REPORT)
        cs = self.cs
        A, nl = cs.A, cs.n_lookups
        words = np.empty((A + nl + len(cs.perm_cols), max_report + 1), dtype=np.uint64)
        self._done(lib.h2bp_check(self._h, C.byref(w), max_report, C.c_void_p(words.ctypes.data)))
        reports = _reports(words, max_report)
        res = {"gates": reports[:A], "lookups": reports[A:A + nl], "copies": reports[A + nl:]}
        res["satisfied"] = not any(c for c, _ in reports)
        return res

    def prove(self, witness_ptr: int, n_cells: int, random_poly_ptr: int, seed: int = 0, break_points=None,
              lookup_ptr: int = 0, n_lookup: int = 0, rational_index_ptr: int = 0, rational_den_ptr: int = 0, n_rational: int = 0,
              lookup_index_ptr: int = 0, instances=None) -> dict:
        """witness_ptr: host pointer (pinned) to the n_cells Montgomery Fr cells of the virtual column, `break_points` as
        keygen pinned them; lookup_ptr / n_lookup: the cells to look up (L > 0); random_poly_ptr: n elements.

        halo2-base's own witness form (`Vec<Assigned<F>>` walked once, nothing inverted): the witness holds n for every
        Rational(n, d) cell, rational_index_ptr / rational_den_ptr the n_rational (uint64 virtual-column index, Montgomery d)
        pairs, indices strictly increasing; lookup_index_ptr (instead of lookup_ptr) the n_lookup uint64 virtual-column
        indices of the looked-up cells in `assign_raw` order.  The device makes of them what batch_invert_assigned and
        assign_raw make (d = 0 -> 0).  A bad index raises H2BError once phase 0's commitments are down; no proof is returned.

        instances: the public values, one (len_m x 4) Montgomery array per instance column of the circuit (None: all empty); they
        enter the transcript before the advice commitments, column by column, and fill rows [0, len_m) of the column.  More than
        u values in a column raise H2BError (InstanceTooLarge)."""
        w, keep = self._witness("prove", witness_ptr, n_cells, break_points, lookup_ptr, n_lookup, rational_index_ptr, rational_den_ptr,
                                n_rational, lookup_index_ptr, instances)
        self._rng = np.random.default_rng(seed)
        cm = np.empty((self.n_commitments, 12), dtype=np.uint64)
        ev = np.empty((len(self.queries), 4), dtype=np.uint64)
        ch = np.empty((5, 4), dtype=np.uint64)
        nbytes = np.empty(2, dtype=np.uint64)
        vp = lambda a: C.c_void_p(a.ctypes.data)
        self._done(lib.h2bp_prove(self._h, C.byref(w), C.c_void_p(random_poly_ptr), self._blind_cb, None,
                                  self._commit_cb if self.keep is not None else COMMIT_FN(), None, vp(cm), vp(ev), vp(ch), vp(nbytes)))
        return {"commitments": list(cm), "evals": {q: ev[i] for i, q in enumerate(self.queries)},
                "challenges": dict(zip(("theta", "beta", "gamma", "y", "x"), (from_limbs(c) for c in ch))),
                "h2d_bytes": int(nbytes[0]), "d2h_bytes": int(nbytes[1])}

    def gen_proof(self, witness_ptr: int, n_cells: int, random_poly_ptr: int, vk_repr: int, instances=None, seed: int = 0, break_points=None,
                  lookup_ptr: int = 0, n_lookup: int = 0, rational_index_ptr: int = 0, rational_den_ptr: int = 0, n_rational: int = 0,
                  lookup_index_ptr: int = 0) -> bytes:
        """The proof bytes halo2-base's gen_proof_with_instances returns (transcript.finalize() of halo2's Blake2bWrite), for the
        witness as `prove` takes it: the same device phases up to the h pieces, then halo2's evaluations and ProverSHPLONK
        (h2b::ProverSession::create_proof_halo2).  vk_repr: the verifying key's transcript_repr as a canonical integer (vk.hash_into
        absorbs it first); instances: the public values as for `prove`.  Blinding scalars as for `prove` (`seed`, `blind_source`)."""
        w, keep = self._witness("gen_proof", witness_ptr, n_cells, break_points, lookup_ptr, n_lookup, rational_index_ptr, rational_den_ptr,
                                n_rational, lookup_index_ptr, instances)
        self._rng = np.random.default_rng(seed)
        repr_limbs = to_limbs(vk_repr)
        cap = 32 * (self.n_commitments + len(self.queries) + 8)  # halo2's proof holds fewer points and scalars than `prove` returns
        out, n = np.zeros(cap, dtype=np.uint8), C.c_size_t()
        self._done(lib.h2bp_prove_halo2(self._h, C.byref(w), C.c_void_p(random_poly_ptr), self._blind_cb, None, C.c_void_p(repr_limbs.ctypes.data),
                                        C.c_void_p(out.ctypes.data), cap, C.byref(n)))
        return out[:n.value].tobytes()

    def free(self):
        if self._h:
            lib.h2bp_session_free(self._h)
            self._h = None


class MockProver:
    """MockProver::run + verify for a halo2-base builder in its keygen form, with no SRS, sigma or proving key
    (h2b::MockProver, include/h2b200_mock.hpp): what BaseTester::run_builder asks of halo2's MockProver.

    Shape as `Circuit`: A gate-advice columns, L lookup-advice columns (or the selector lookup when L = 0, or no lookup), F
    constants columns, the table 0 .. 2^lookup_bits - 1, and max_rows = 2^k - unusable_rows as calculate_params gets it
    (at most 2^k - 7; default 2^k - 9, BaseTester's unusable_rows), and I instance columns.  F changes no value check, only how
    many distinct constants fit (F u).  `lagr[name]` (a{j}, l{t}, q{j}, q_lookup, table) views the columns of the last run."""

    def __init__(self, ctx: Context, k: int, A: int = 1, L: int = 0, selector_lookup: bool = True, lookup_bits: int = 8,
                 max_rows: int | None = None, I: int = 0, F: int = 1):
        self.ctx, self.k, self.A, self.L, self.I, self.F = ctx, k, A, L, I, F
        self.max_rows = (1 << k) - 9 if max_rows is None else max_rows
        h, nl = C.c_void_p(), C.c_uint64()
        ctx.check(lib.h2bp_mock_create(ctx.h, k, A, L, int(selector_lookup), lookup_bits, self.max_rows, I, F, C.byref(h), C.byref(nl)))
        self._h, self.n_lookups = h, int(nl.value)
        self.lagr = _Columns(self, "lagr")

    def column(self, table: str, name: str) -> Column:
        if table != "lagr":
            raise KeyError(table)
        poly, off, rows = C.c_void_p(), C.c_size_t(), C.c_size_t()
        self.ctx.check(lib.h2bp_mock_column(self._h, name.encode(), C.byref(poly), C.byref(off), C.byref(rows)))
        return Column(self.ctx, poly, off.value, rows.value)

    def run(self, cells, selectors, advice_equalities=(), constant_equalities=None, lookups=(), rational_index=None, rational_den=None,
            max_report: int = 16, instances=None, public=None) -> dict:
        """cells: the virtual column (n x 4 Montgomery limbs), in either witness form (rational_index / rational_den: the
        (uint64 index, Montgomery d) pairs of the Rational cells, indices strictly increasing); selectors: one bool per cell;
        advice_equalities: (a, b) index pairs; constant_equalities: (constants (m x 4 Montgomery limbs), indices); lookups:
        indices of the looked-up cells in assign_raw order (L > 0) or of the cells whose raw row gets q_lookup (L = 0).

        Returns gates[j], lookups[t] (failing rows < u), equalities and constants (failing equality indices), each as
        (count, the first min(count, max_report) ascending); equality_cells / constant_cells: the raw cells ((column, row)) of
        every reported equality; break_points; satisfied.  halo2-base's panics raise H2BError with its message.

        instances / public: per instance column, the indices of its cells and its public values (Montgomery), one value per cell
        (None: all empty).  instances[m] reports the rows r whose cell differs from public[m][r], instance_cells[m] their raw
        cells; more than u values raise H2BError (InstanceTooLarge).

        distinct_constants: the number D of distinct constants, from which calculate_params sets num_fixed = ceil(D / 2^k)."""
        if not 1 <= max_report <= CHECK_MAX_REPORT:
            raise ValueError("MockProver: max_report must be in 1..%d" % CHECK_MAX_REPORT)
        V = np.ascontiguousarray(cells, dtype=np.uint64).reshape(-1, 4)
        I = self.I
        view, keep = _builder_view("MockProver", len(V), selectors, advice_equalities, constant_equalities, lookups, V, rational_index,
                                   rational_den, I, instances, [()] * I if public is None else public)
        A, nl = self.A, self.n_lookups
        bps, nbp, distinct = np.zeros(max(A, 1), dtype=np.uint64), C.c_uint64(), C.c_uint64()
        words = np.empty((A + nl + 2 + I, max_report + 1), dtype=np.uint64)
        cells_out = np.empty((6 + 2 * I) * max_report, dtype=np.uint64)
        self.ctx.check(lib.h2bp_mock_run(self._h, C.byref(view), max_report, C.c_void_p(bps.ctypes.data), C.byref(nbp),
                                         C.c_void_p(words.ctypes.data), C.c_void_p(cells_out.ctypes.data), C.byref(distinct)))
        reports = _reports(words, max_report)
        eq, co = reports[A + nl], reports[A + nl + 1]
        ec = cells_out[:4 * max_report].reshape(-1, 4)
        cc = cells_out[4 * max_report:6 * max_report].reshape(-1, 2)
        inst = reports[A + nl + 2:]
        ic = [cells_out[(6 + 2 * m) * max_report:(8 + 2 * m) * max_report].reshape(-1, 2)[:len(inst[m][1])] for m in range(I)]
        return {"gates": reports[:A], "lookups": reports[A:A + nl], "equalities": eq, "constants": co,
                "equality_cells": [((int(c[0]), int(c[1])), (int(c[2]), int(c[3]))) for c in ec[:len(eq[1])]],
                "constant_cells": [(int(c[0]), int(c[1])) for c in cc[:len(co[1])]],
                "break_points": [int(b) for b in bps[:nbp.value]], "satisfied": not any(c for c, _ in reports),
                "instances": inst, "instance_cells": [[(int(c[0]), int(c[1])) for c in x] for x in ic],
                "distinct_constants": int(distinct.value)}

    def free(self):
        if self._h:
            lib.h2bp_mock_free(self._h)
            self._h = None

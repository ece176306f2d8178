"""Resident prover core: the device-side data flow of halo2-axiom 0.5.3 `create_proof` for the constraint system
halo2-base builds (one vertical gate per gate-advice column, halo2-base/src/gates/flex_gate/mod.rs:80-91; a range lookup
`q_lookup * a in table`, gates/range/mod.rs:92-94,131-141; equality on the constants column and the gate column,
flex_gate/mod.rs:69,124-129), with every column kept in HBM behind `h2b_poly` handles between the phases:

    witness (host) --H2D--> assign_witnesses --> commit advice                                   (SURVEY.md §3.3 step 2)
    theta:  q_lookup * a, permute_expression_pair --> commit A', S'                              (step 3)
    beta, gamma:  permutation product, lookup product, random polynomial (host) --> commit       (steps 4, 5)
    y:  lagrange_to_coeff + coeff_to_extended of every column, gate / permutation / lookup terms folded on the
        extended coset, divide_by_vanishing_poly, extended_to_coeff, h pieces --> commit         (step 6)
    x:  evaluations                                                                              (step 7)
    SHPLONK-shaped opening: per rotation set a linear combination and kate divisions, two commitments   (step 8)

Only the witness cells, the random polynomial and the blinding scalars go up; only commitments and evaluations come
down.  The transcript stays on the host (as it stays in Rust): challenges are squeezed from Blake2b over the commitment
bytes.  The prover crate is not vendored (SURVEY.md §0), so phase order and term order are restated; what the tests and
bench.py check is protocol-level: every commitment equals the closed form of the polynomial it commits, and the quotient
identity  sum of folded terms (x) == h(x) * (x^n - 1)  holds at the challenge point.

No field arithmetic happens here on the hot path: everything is computed by the kernels behind include/h2b200.h."""
from __future__ import annotations
import ctypes as C
import hashlib
import numpy as np
from ._capi import lib, BASIS_MONOMIAL, BASIS_LAGRANGE, H2B_ERR_ARG, CHECK_MAX_REPORT
from .host import Context, ParamsKZG, H2BError
from . import evaluation as ev

R_MOD = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
MONT_R = (1 << 256) % R_MOD
MONT_RINV = pow(1 << 256, -1, R_MOD)
ROOT_OF_UNITY = pow(7, (R_MOD - 1) >> 28, R_MOD)
DELTA = pow(7, 1 << 28, R_MOD)
BLINDING_FACTORS = 6  # max(3, queries of the gate column = 4) + 2  (SURVEY.md App. B)
GATES_PER_PROGRAM = 5  # vertical gates per GraphEvaluator program (10 calculations each, 64 per program)


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
    commitment enters the transcript and the proof: the accumulation order inside an MSM is not deterministic (atomics in the
    counting sort), so the Jacobian representative is not either; the affine point is.  One modular inversion per
    commitment on the host, as the Rust prover's `to_affine`.  (Montgomery domain throughout: with Xm = X R, Zm = Z R the
    result x R is Xm R^2 / Zm^2.)"""
    b = np.ascontiguousarray(pt, dtype=np.uint64).tobytes()
    xm, ym, zm = (int.from_bytes(b[32 * j:32 * j + 32], "little") for j in range(3))
    if zm == 0:
        return np.zeros(12, dtype=np.uint64)
    zi = pow(zm, -1, P_MOD)
    zi2 = zi * zi % P_MOD
    x = xm * zi2 % P_MOD * _PR2 % P_MOD
    y = ym * zi2 % P_MOD * zi % P_MOD * _PR3 % P_MOD
    return np.frombuffer(x.to_bytes(32, "little") + y.to_bytes(32, "little") + _ONE_BYTES, dtype=np.uint64)


def g1_normalize_host_batch(pts: np.ndarray) -> np.ndarray:
    """g1_normalize_host over the m commitments of a phase with ONE modular inversion (Montgomery's trick)"""
    pts = np.ascontiguousarray(pts, dtype=np.uint64).reshape(-1, 12)
    b = pts.tobytes()
    val = [int.from_bytes(b[32 * j:32 * j + 32], "little") for j in range(3 * len(pts))]
    zs = [val[3 * i + 2] for i in range(len(pts))]
    pref, acc = [], 1
    for z in zs:  # prefix products over the non-zero z
        pref.append(acc)
        if z:
            acc = acc * z % P_MOD
    inv = pow(acc, -1, P_MOD)
    out = bytearray(96 * len(pts))
    for i in range(len(pts) - 1, -1, -1):
        z = zs[i]
        if not z:
            continue
        zi = inv * pref[i] % P_MOD
        inv = inv * z % P_MOD
        zi2 = zi * zi % P_MOD
        x = val[3 * i] * zi2 % P_MOD * _PR2 % P_MOD
        y = val[3 * i + 1] * zi2 % P_MOD * zi % P_MOD * _PR3 % P_MOD
        out[96 * i:96 * i + 96] = x.to_bytes(32, "little") + y.to_bytes(32, "little") + _ONE_BYTES
    return np.frombuffer(bytes(out), dtype=np.uint64).reshape(-1, 12)


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


class Transcript:
    """Blake2b over what the prover writes; `squeeze` yields an Fr challenge (host side, as the Rust transcript)"""

    def __init__(self):
        self.h = hashlib.blake2b(digest_size=64)

    def absorb(self, arr):
        self.h.update(np.ascontiguousarray(arr).tobytes())

    def squeeze(self) -> int:
        d = self.h.digest()
        self.h.update(b"\x00")
        return int.from_bytes(d, "little") % R_MOD


class Circuit:
    """The fixed side of a synthetic halo2-base circuit (what keygen_pk would hold), resident on the GPU in the three forms
    create_proof needs: Lagrange values, coefficients, extended-coset evaluations.

    Shape (halo2-base `BaseCircuitParams`: num_advice_per_phase, num_lookup_advice_per_phase, num_fixed = 1):
      A gate-advice columns a0..a{A-1}, each with its selector q{j} and the vertical gate (flex_gate/mod.rs:80-91);
      L lookup-advice columns l0..l{L-1}, each looked up in `table` as it is (range/mod.rs:131-150); with L = 0 the one
      lookup is `q_lookup * a0 in table` (range/mod.rs:92-94);
      one constants column c; equality on [c, a0.., l0..] in that order (the permutation's column order).
    Degree 5 with the selector lookup, 4 with lookup-advice columns, 3 without any lookup: permutation sets of degree - 2
    columns, degree - 1 pieces of h."""

    def __init__(self, ctx: Context, k: int, fixed_lagrange: dict, sigma_lagrange: list, A: int = 1, L: int = 0,
                 selector_lookup: bool = True):
        self.ctx, self.k, self.n, self.A, self.L = ctx, k, 1 << k, A, L
        self.selector_lookup = selector_lookup and L == 0  # False with L = 0: a circuit without any lookup (inner_product bench)
        self.degree = 4 if L else (5 if self.selector_lookup else 3)
        self.chunk = self.degree - 2
        self.ext_k = k + (1 if self.degree == 3 else 2)  # EvaluationDomain::new(j = degree, k): 2^ext_k >= (degree - 1) n
        self.bf = BLINDING_FACTORS
        self.u = self.n - (self.bf + 1)
        self.adv_names = ["a%d" % j for j in range(A)] + ["l%d" % t for t in range(L)]
        self.perm_cols = ["c"] + self.adv_names
        self.n_sets = (len(self.perm_cols) + self.chunk - 1) // self.chunk
        self.n_lookups = L if L else (1 if self.selector_lookup else 0)
        self.fixed_names = ["q%d" % j for j in range(A)] + (["q_lookup"] if self.selector_lookup else []) + (["table"] if self.n_lookups else []) + ["c"]
        assert len(sigma_lagrange) == len(self.perm_cols) and all(nm in fixed_lagrange for nm in self.fixed_names)
        n, ne = self.n, 1 << self.ext_k
        vp = C.c_void_p
        l0 = np.zeros((n, 4), dtype=np.uint64); l0[0] = to_limbs(1)
        ll = np.zeros((n, 4), dtype=np.uint64); ll[self.u] = to_limbs(1)
        la = np.zeros((n, 4), dtype=np.uint64); la[: self.u] = to_limbs(1)
        cols = {nm: fixed_lagrange[nm] for nm in self.fixed_names}
        cols.update({"sigma_" + nm: sg for nm, sg in zip(self.perm_cols, sigma_lagrange)})
        cols.update({"l0": l0, "l_last": ll, "l_active": la})
        self.sigma_names = ["sigma_" + nm for nm in self.perm_cols]
        self.lagr, self.coeff, self.ext = {}, {}, {}
        for name, arr in cols.items():
            lg, cf, ex = Poly(ctx, n), Poly(ctx, n), Poly(ctx, ne)
            lg.upload(arr)
            cf.upload(arr)
            ctx.check(lib.h2b_lagrange_to_coeff_dev(ctx.h, vp(cf.ptr), k))
            ctx.check(lib.h2b_coeff_to_extended_dev(ctx.h, vp(cf.ptr), n, self.ext_k, vp(ex.ptr)))
            self.lagr[name], self.coeff[name], self.ext[name] = lg, cf, ex
        ctx.synchronize()
        # the gate programs: one vertical gate per gate-advice column, GATES_PER_PROGRAM columns per h2b_graph (a program holds
        # at most 64 calculations; every program continues the Horner fold in y from the previous value, so a chain of
        # programs is the one fold evaluate_h does); inside a program fixed slot i = q{j0 + i}, advice slot i = a{j0 + i}
        self.gate_programs = []
        for j0 in range(0, A, GATES_PER_PROGRAM):
            g = ev.GraphEvaluator()
            js = list(range(j0, min(A, j0 + GATES_PER_PROGRAM)))
            gates = []
            for i in range(len(js)):
                a = lambda r, i=i: ("advice", i, r)
                gates.append(("product", ("fixed", i, 0), ("sum", ("sum", a(0), ("product", a(1), a(2))), ("negated", a(3)))))
            self.gate_programs.append((g, g.add_gates(gates), js))
        # the lookups' programs: (compressed input + beta)(compressed table + gamma)
        g2 = ev.GraphEvaluator()
        if L == 0:   # fixed slots [q_lookup, table], advice slot [a0]
            self.lk_graph, self.lk_res = g2, g2.add_lookup([("product", ("fixed", 0, 0), ("advice", 0, 0))], [("fixed", 1, 0)])
        else:        # fixed slot [table], advice slot [l{t}]
            self.lk_graph, self.lk_res = g2, g2.add_lookup([("advice", 0, 0)], [("fixed", 0, 0)])
        self._check = None  # what ProverSession.check needs beyond a proof, built by its first call (check_state)

    def check_state(self):
        """(gate program, its result, sigma map) for the constraint check, built on the first call: the vertical gate
        q * (a + b c - d) as one program on fixed slot 0 / advice slot 0 (bound to q{j}, a{j} for every gate column), and the
        sigma columns decoded into map[c][r] = c' << k | r' (u32, perm_cols order).  Raises H2BError naming the first
        (column, row) whose sigma entry is not delta^c' omega^r' for a permutation column c'."""
        if self._check is None:
            ctx, npc = self.ctx, len(self.perm_cols)
            g = ev.GraphEvaluator()
            a = lambda r: ("advice", 0, r)
            res = g.add_expression(("product", ("fixed", 0, 0), ("sum", ("sum", a(0), ("product", a(1), a(2))), ("negated", a(3)))))
            smap = Poly(ctx, (npc * self.n + 7) // 8)
            rep = Poly(ctx, (2 * npc + 3) // 4)  # max_report = 1: count and first row per column
            sig = (C.c_void_p * npc)(*[self.lagr[nm].ptr for nm in self.sigma_names])
            try:
                ctx.check(lib.h2b_permutation_decode_dev(ctx.h, sig, npc, self.k, C.c_void_p(smap.ptr), 1, C.c_void_p(rep.ptr)))
                words = rep.download().reshape(-1)
            finally:
                rep.free()
            bad = [c for c in range(npc) if words[2 * c]]
            if bad:
                smap.free()
                c = bad[0]
                raise H2BError(H2B_ERR_ARG, "Circuit: the sigma entry of permutation column %d (%s) at row %d is not delta^c omega^r "
                                            "for any of the %d permutation columns" % (c, self.perm_cols[c], int(words[2 * c + 1]), npc))
            self._check = (g, res, smap)
        return self._check

    def free(self):
        for d in (self.lagr, self.coeff, self.ext):
            for p in d.values():
                p.free()
        if self._check is not None:
            self._check[2].free()
            self._check = None


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


class ProverSession:
    """One proof at a time on one context; owns the resident working set (allocated once, reused for every proof)."""

    def __init__(self, ctx: Context, params: ParamsKZG, circuit: Circuit):
        self.ctx, self.params, self.cs = ctx, params, circuit
        cs = circuit
        n, ne = cs.n, 1 << cs.ext_k
        self.polys = []

        def P(m):
            p = Poly(ctx, m)
            self.polys.append(p)
            return p
        self.v = P(n * cs.A)                            # virtual column (gate cells)
        self.lkv = P(n * cs.L) if cs.L else None        # cells to look up
        self.adv_block = P(n * (cs.A + cs.L))           # the advice columns, one n-row slice each (assignment output)
        self.lagr, self.coef, self.ext = {}, {}, {}     # by column name: Lagrange / coefficient / extended-coset form
        for j, nm in enumerate(cs.adv_names):
            self.lagr[nm] = _View(self.adv_block, j * n, n)
        names = list(cs.adv_names)
        for t in range(cs.n_lookups):
            names += ["pa%d" % t, "ps%d" % t, "zl%d" % t]
        names += ["zp%d" % s for s in range(cs.n_sets)]
        for nm in names:
            if nm not in self.lagr:
                self.lagr[nm] = P(n)
            self.coef[nm] = P(n)
            self.ext[nm] = P(ne)
        self.inp = P(n) if cs.selector_lookup else None  # compressed lookup input q_lookup * a0
        self.rnd = P(n)                                 # random polynomial of the vanishing argument
        self.h = P(ne)                                  # quotient values, then its coefficients (degree - 1 pieces of n)
        self.tmp = [P(n) for _ in range(4)]
        self.tmp_side = [P(n) for _ in range(3)]
        # commitments of a phase: up to 16 x 12 limbs (3 elements each); element 48 holds the verdict words of the halo2-base
        # witness form (u32 at byte 0: the Rational list, at byte 4: the lookup indices), downloaded with phase 0's commitments
        self.d_out = P(49)
        self.d_status = P(max(1, cs.n_lookups))         # verdict word of every lookup permutation
        self.grown = {}                                 # halo2-base witness form: buffers grown to the largest R / n_lookup seen
        self.zero = P(1)                                # one zero element (never written)
        self.h2d_bytes = self.d2h_bytes = 0
        self.begin, self.n_loc, self.allreduce = 0, n, None
        self.keep = None  # verification runs: dict that receives the committed polynomials (downloaded, untimed)
        self.blind_log = None
        self.blind_source = None  # optional callable rows -> (rows, 4) Montgomery limbs (tests: replay a fixed proof)

    def shard(self, begin: int, n_loc: int, allreduce):
        """multi-GPU: this rank commits rows [begin, begin + n_loc) of every polynomial and `allreduce(ptr, m)` combines the
        partial commitments of all ranks in place on the device (h2b_g1_allreduce_dev); everything else is replicated"""
        self.begin, self.n_loc, self.allreduce = begin, n_loc, allreduce

    # ---- helpers
    def _commit(self, items, verdict: bool = False) -> np.ndarray:
        """items: list of (basis, device pointer); batched launches of up to 16, the commitments come down in one copy each.
        verdict: the first copy also brings element 48 (the witness-form verdict words) down, into self.verdict"""
        ctx = self.ctx
        outs = []
        for lo in range(0, len(items), 16):
            part = items[lo:lo + 16]
            m = len(part)
            ptrs = (C.c_void_p * m)(*[p + 32 * self.begin for _, p in part])
            bs = (C.c_int * m)(*[b for b, _ in part])
            ctx.check(lib.h2b_msm_g1_batch_dev(ctx.h, self.params.h, bs, ptrs, m, self.n_loc, C.c_void_p(self.d_out.ptr)))
            if self.allreduce is not None:
                self.allreduce(self.d_out.ptr, m)
            if self.keep is not None:  # untimed verification run: remember what was committed
                for b, p in part:
                    arr = np.empty((self.cs.n, 4), dtype=np.uint64)
                    ctx.synchronize()
                    self._raw_download(p, arr)
                    self.keep.setdefault("committed", []).append((b, arr))
            cnt = 49 if verdict and lo == 0 else m * 3
            out = np.empty((cnt, 4), dtype=np.uint64)
            ctx.check(lib.h2b_poly_download(ctx.h, self.d_out.h, 0, C.c_void_p(out.ctypes.data), cnt))
            self.d2h_bytes += cnt * 32
            if cnt == 49:
                self.verdict = (int(out[48, 0]) & 0xFFFFFFFF, int(out[48, 0]) >> 32)
            outs.append(g1_normalize_host_batch(out[: m * 3]))
        return np.concatenate(outs)

    def _raw_download(self, dev_ptr: int, arr: np.ndarray):
        """device pointer inside one of the session's polynomials -> host (verification only)"""
        for p in self.polys:
            if p.ptr <= dev_ptr < p.ptr + 32 * p.n:
                self.ctx.check(lib.h2b_poly_download(self.ctx.h, p.h, (dev_ptr - p.ptr) // 32, C.c_void_p(arr.ctypes.data), len(arr)))
                return
        raise ValueError("pointer outside the session's polynomials")

    def _grown(self, name: str, n: int) -> Poly:
        """a session buffer of at least n elements; reallocated only when a proof needs more than any proof before it"""
        p = self.grown.get(name)
        if p is None or p.n < n:
            if p is not None:
                self.polys.remove(p)
                p.free()
            p = Poly(self.ctx, max(n, 1))
            self.polys.append(p)
            self.grown[name] = p
        return p

    def _upload_u64(self, name: str, host_ptr: int, count: int) -> Poly:
        """count uint64 words from host_ptr into the session buffer `name`: whole 32-byte elements straight from the caller's
        array, the last 1..3 words through a zero-padded element (nothing past the end of the caller's array is read)"""
        p = self._grown(name, (count + 3) // 4)
        full = count // 4
        if full:
            p.upload_ptr(host_ptr, full)
        if count % 4:
            tail = np.zeros(4, dtype=np.uint64)
            C.memmove(tail.ctypes.data, host_ptr + 32 * full, 8 * (count % 4))
            p.upload(tail, full)
        self.h2d_bytes += 8 * count
        return p

    def _blind(self, col, first_row: int, rng: np.random.Generator):
        cnt = self.cs.n - first_row
        if self.blind_source is not None:  # the caller's blinding scalars (Montgomery limbs), in the order of use
            b = np.ascontiguousarray(self.blind_source(cnt), dtype=np.uint64).reshape(cnt, 4)
        else:
            b = rng.integers(0, 1 << 62, size=(cnt, 4), dtype=np.int64).astype(np.uint64)
            b[:, 3] &= np.uint64((1 << 60) - 1)
        if self.blind_log is not None:  # the blinding rows in the order of use (the C++ twin replays them)
            self.blind_log.append(b)
        col.upload(b, first_row)
        self.h2d_bytes += cnt * 32

    def _lincomb(self, ptrs, scalars, out: Poly):
        """out = sum_i scalars[i] * ptrs[i] over n coefficients (h2b_poly_lincomb takes at most 32 polynomials a call)"""
        ctx, n, vp = self.ctx, self.cs.n, C.c_void_p
        first = True
        for lo in range(0, len(ptrs), 31):
            pp, sc = list(ptrs[lo:lo + 31]), list(scalars[lo:lo + 31])
            if not first:
                pp, sc = [out.ptr] + pp, [1] + sc
            arr = (C.c_void_p * len(pp))(*pp)
            lim = np.stack([to_limbs(x) for x in sc])
            ctx.check(lib.h2b_poly_lincomb_dev(ctx.h, arr, vp(lim.ctypes.data), len(pp), n, vp(out.ptr)))
            first = False

    @staticmethod
    def _check_witness_args(lookup_ptr, lookup_index_ptr, n_rational, rational_index_ptr, rational_den_ptr, who):
        if lookup_ptr and lookup_index_ptr:
            raise ValueError(who + ": pass the looked-up cells either as values (lookup_ptr) or as indices (lookup_index_ptr)")
        if n_rational and not (rational_index_ptr and rational_den_ptr):
            raise ValueError(who + ": n_rational > 0 needs rational_index_ptr and rational_den_ptr")

    @staticmethod
    def _witness_error(rat: int, lk: int, who: str):
        """the verdict words of the halo2-base witness form (rat: h2b_apply_rational_dev, lk: the indexed gather) -> H2BError"""
        why = (["a Rational index is >= the witness length"] if rat & 1 else []) + \
              (["the Rational indices do not strictly increase"] if rat & 2 else []) + \
              (["a lookup index is >= the witness length"] if lk & 1 else [])
        raise H2BError(H2B_ERR_ARG, who + ": " + "; ".join(why))

    def _assign_witness(self, witness_ptr, n_cells, break_points, lookup_ptr, n_lookup, rational_index_ptr, rational_den_ptr, n_rational,
                        lookup_index_ptr, random_poly_ptr=0):
        """phase 0 up to the advice columns in self.adv_block (what `prove` and `check` share): the witness, the halo2-base
        form's Rational pairs and lookup indices or the looked-up values go up, the Rational cells become n * d^-1 and the
        assignment lays out the gate and lookup-advice columns (all 2^k rows written).  With the halo2-base form the two
        verdict words land in element 48 of d_out.  random_poly_ptr != 0: the random polynomial goes up on the side queue,
        beside the assignment."""
        ctx, cs, vp = self.ctx, self.cs, C.c_void_p
        k, n, A, L = cs.k, cs.n, cs.A, cs.L
        hb_form = bool(n_rational or lookup_index_ptr)
        self.v.upload_ptr(witness_ptr, n_cells)
        self.h2d_bytes += n_cells * 32
        if n_rational:
            den = self._grown("rational_den", n_rational)
            den.upload_ptr(rational_den_ptr, n_rational)
            self.h2d_bytes += n_rational * 32
            rat_idx = self._upload_u64("rational_index", rational_index_ptr, n_rational)
        if L and lookup_index_ptr:
            lk_idx = self._upload_u64("lookup_index", lookup_index_ptr, n_lookup)
        elif L:
            self.lkv.upload_ptr(lookup_ptr, n_lookup)
            self.h2d_bytes += n_lookup * 32
        if random_poly_ptr:
            ctx.check(lib.h2b_ctx_side_begin(ctx.h))
            ctx.check(lib.h2b_poly_upload_async(ctx.h, self.rnd.h, 0, vp(random_poly_ptr), n))
            ctx.check(lib.h2b_ctx_side_end(ctx.h))
            self.h2d_bytes += n * 32
        verdict = self.d_out.at(48)
        if hb_form:  # zeroes both verdict words, then the Rational cells become n * d^-1 before anything reads the witness
            ctx.check(lib.h2b_apply_rational_dev(ctx.h, vp(self.v.ptr), n_cells, vp(rat_idx.ptr if n_rational else 0),
                                                 vp(den.ptr if n_rational else 0), n_rational, vp(verdict)))
        nbp = 0 if break_points is None else len(break_points)
        bp_arr = (C.c_uint64 * max(1, nbp))(*[int(b) for b in (break_points if nbp else [])])
        ctx.check(lib.h2b_assign_columns_dev(ctx.h, vp(self.v.ptr), n_cells, bp_arr if nbp else None, nbp, k, A, vp(self.adv_block.ptr)))
        if L and lookup_index_ptr:
            ctx.check(lib.h2b_assign_lookups_indexed_dev(ctx.h, vp(self.v.ptr), n_cells, vp(lk_idx.ptr), n_lookup, k, L,
                                                         vp(self.adv_block.at(A * n)), vp(verdict + 4)))
        elif L:
            ctx.check(lib.h2b_assign_lookups_dev(ctx.h, vp(self.lkv.ptr), n_lookup, k, L, vp(self.adv_block.at(A * n))))

    def check(self, witness_ptr: int, n_cells: int, break_points=None, lookup_ptr: int = 0, n_lookup: int = 0, rational_index_ptr: int = 0,
              rational_den_ptr: int = 0, n_rational: int = 0, lookup_index_ptr: int = 0, max_report: int = 16) -> dict:
        """MockProver::verify for this circuit: which gates, lookups and copy constraints the witness breaks, and where.
        Takes the witness exactly as `prove` does and runs the same assignment; no blinding, no random polynomial, no transcript.
        The values checked are the ones a proof would commit before blinding, with rows >= u read as 0:
          gates[j]    rows r < u with q{j}(r) (a{j}(r) + a{j}(r+1) a{j}(r+2) - a{j}(r+3)) != 0 (rotations mod n);
          lookups[t]  rows r < u whose input (q_lookup * a0, or l{t}) is not among the table's rows [0, u);
          copies[c]   rows r < n of permutation column c (perm_cols order) whose value differs from the cell sigma_c(r) names.
        Each entry is (failure count, the first min(count, max_report) failing rows ascending).  Every report comes down in one
        copy.  A bad halo2-base index raises H2BError; so does a sigma entry that names no cell (on the circuit's first check)."""
        ctx, cs, vp = self.ctx, self.cs, C.c_void_p
        k, n, u, A, L = cs.k, cs.n, cs.u, cs.A, cs.L
        self._check_witness_args(lookup_ptr, lookup_index_ptr, n_rational, rational_index_ptr, rational_den_ptr, "check")
        if not 1 <= max_report <= CHECK_MAX_REPORT:
            raise ValueError("check: max_report must be in 1..%d" % CHECK_MAX_REPORT)
        gate, gate_res, smap = cs.check_state()
        hb_form = bool(n_rational or lookup_index_ptr)
        self.h2d_bytes = self.d2h_bytes = 0
        self._assign_witness(witness_ptr, n_cells, break_points, lookup_ptr, n_lookup, rational_index_ptr, rational_den_ptr, n_rational,
                             lookup_index_ptr)
        zero_rows = self._grown("zero_rows", n - u)  # zero-filled, never written
        for nm in cs.adv_names:
            ctx.check(lib.h2b_poly_copy_dev(ctx.h, vp(self.lagr[nm].at(u)), vp(zero_rows.ptr), n - u))
        # report block: element 0 = the witness-form verdict words, then max_report + 1 words per gate, lookup, permutation column
        W, npc = max_report + 1, len(cs.perm_cols)
        n_items = A + cs.n_lookups + npc
        rep = self._grown("check_report", 1 + (n_items * W + 3) // 4)
        at = lambda i: vp(rep.ptr + 32 + 8 * W * i)
        if hb_form:
            ctx.check(lib.h2b_poly_copy_dev(ctx.h, vp(rep.ptr), vp(self.d_out.at(48)), 1))
        for j in range(A):
            bg = ev.BoundGraph(gate, gate_res, fixed=[cs.lagr["q%d" % j].ptr], advice=[self.lagr["a%d" % j].ptr])
            ctx.check(lib.h2b_check_graph_dev(ctx.h, C.byref(bg.struct), k, u, max_report, at(j)))
        for t in range(cs.n_lookups):
            if L == 0:
                ctx.check(lib.h2b_fr_mul_elementwise_dev(ctx.h, vp(cs.lagr["q_lookup"].ptr), vp(self.lagr["a0"].ptr), n, vp(self.inp.ptr)))
                inp = self.inp.ptr
            else:
                inp = self.lagr["l%d" % t].ptr
            ctx.check(lib.h2b_check_lookup_dev(ctx.h, vp(inp), vp(cs.lagr["table"].ptr), k, u, max_report, at(A + t)))
        cols = [cs.lagr["c"].ptr] + [self.lagr[nm].ptr for nm in cs.adv_names]
        ctx.check(lib.h2b_check_copies_dev(ctx.h, (C.c_void_p * npc)(*cols), vp(smap.ptr), npc, k, max_report, at(A + cs.n_lookups)))
        words = rep.download(0, 1 + (n_items * W + 3) // 4).reshape(-1)
        self.d2h_bytes = 8 * len(words)
        if hb_form:
            rat, lk = int(words[0]) & 0xFFFFFFFF, int(words[0]) >> 32
            lk = lk if L and lookup_index_ptr else 0  # the lookup word is only written by the indexed gather
            if rat or lk:
                self._witness_error(rat, lk, "check")
        reports = []
        for i in range(n_items):
            w = words[4 + W * i: 4 + W * (i + 1)]
            cnt = int(w[0])
            reports.append((cnt, [int(r) for r in w[1:1 + min(cnt, max_report)]]))
        res = {"gates": reports[:A], "lookups": reports[A:A + cs.n_lookups], "copies": reports[A + cs.n_lookups:]}
        res["satisfied"] = not any(c for c, _ in reports)
        return res

    def prove(self, witness_ptr: int, n_cells: int, random_poly_ptr: int, seed: int = 0, break_points=None,
              lookup_ptr: int = 0, n_lookup: int = 0, rational_index_ptr: int = 0, rational_den_ptr: int = 0, n_rational: int = 0,
              lookup_index_ptr: int = 0) -> dict:
        """witness_ptr: host pointer (pinned) to the n_cells Montgomery Fr cells of the virtual column, `break_points` as
        keygen pinned them; lookup_ptr / n_lookup: the cells to look up (L > 0); random_poly_ptr: n elements.

        halo2-base's own witness form (`Vec<Assigned<F>>` walked once, nothing inverted): the witness holds n for every
        Rational(n, d) cell, rational_index_ptr / rational_den_ptr the n_rational (uint64 virtual-column index, Montgomery d)
        pairs, indices strictly increasing; lookup_index_ptr (instead of lookup_ptr) the n_lookup uint64 virtual-column
        indices of the looked-up cells in `assign_raw` order.  The device makes of them what batch_invert_assigned and
        assign_raw make (d = 0 -> 0).  A bad index raises H2BError once phase 0's commitments are down; no proof is returned."""
        ctx, cs, vp = self.ctx, self.cs, C.c_void_p
        k, n, ext_k, bf, u, A, L = cs.k, cs.n, cs.ext_k, cs.bf, cs.u, cs.A, cs.L
        self._check_witness_args(lookup_ptr, lookup_index_ptr, n_rational, rational_index_ptr, rational_den_ptr, "prove")
        hb_form = bool(n_rational or lookup_index_ptr)
        rng = np.random.default_rng(seed)
        tr = Transcript()
        self.h2d_bytes = self.d2h_bytes = 0
        res = {"commitments": []}
        import os, time
        trace = [] if os.environ.get("H2B_PROVER_TRACE") else None

        def mark(label):  # diagnostic: wall clock per phase with a full synchronisation (changes the overlap: not for timing runs)
            if trace is not None:
                ctx.synchronize()
                trace.append((label, time.perf_counter()))
        mark("start")

        def side_transforms(names):
            """beside the main queue: Lagrange -> coefficient buffer, lagrange_to_coeff, coeff_to_extended"""
            ctx.check(lib.h2b_ctx_side_begin(ctx.h))
            try:
                for nm in names:
                    ctx.check(lib.h2b_poly_copy_dev(ctx.h, vp(self.coef[nm].ptr), vp(self.lagr[nm].ptr), n))
                    ctx.check(lib.h2b_lagrange_to_coeff_dev(ctx.h, vp(self.coef[nm].ptr), k))
                    ctx.check(lib.h2b_coeff_to_extended_dev(ctx.h, vp(self.coef[nm].ptr), n, ext_k, vp(self.ext[nm].ptr)))
            finally:
                ctx.check(lib.h2b_ctx_side_end(ctx.h))

        def commit(items, verdict=False):
            cm = self._commit(items, verdict)
            res["commitments"] += list(cm)
            tr.absorb(cm)

        # ---- phase 0: witness up, assignment, advice commitments (the random polynomial goes up beside it)
        self._assign_witness(witness_ptr, n_cells, break_points, lookup_ptr, n_lookup, rational_index_ptr, rational_den_ptr, n_rational,
                             lookup_index_ptr, random_poly_ptr)
        for nm in cs.adv_names:
            self._blind(self.lagr[nm], u, rng)
        commit([(BASIS_LAGRANGE, self.lagr[nm].ptr) for nm in cs.adv_names], verdict=hb_form)
        rat, lk = self.verdict if hb_form else (0, 0)
        if rat or (L and lookup_index_ptr and lk):
            ctx.check(lib.h2b_ctx_side_join(ctx.h))  # nothing of this proof stays in flight behind the error
            ctx.synchronize()
            self._witness_error(rat, lk if L and lookup_index_ptr else 0, "prove")
        theta = tr.squeeze()
        mark("phase0 advice")
        ctx.check(lib.h2b_ctx_side_join(ctx.h))  # the random polynomial arrived while phase 0 ran
        side_transforms(cs.adv_names)
        # ---- lookups: compressed input, permuted pair (enqueue only: the verdict words land in d_status and are read
        # right after the commitments of this phase, whose download synchronises anyway)
        lk_in = []
        for t in range(cs.n_lookups):
            if L == 0:
                ctx.check(lib.h2b_fr_mul_elementwise_dev(ctx.h, vp(cs.lagr["q_lookup"].ptr), vp(self.lagr["a0"].ptr), n, vp(self.inp.ptr)))
                lk_in.append(self.inp.ptr)
            else:
                lk_in.append(self.lagr["l%d" % t].ptr)
            pa, ps = self.lagr["pa%d" % t], self.lagr["ps%d" % t]
            ctx.check(lib.h2b_permute_expression_pair_async_dev(ctx.h, vp(lk_in[t]), vp(cs.lagr["table"].ptr), k, bf, vp(pa.ptr), vp(ps.ptr),
                                                                vp(self.d_status.at(t))))
            self._blind(pa, u, rng)
            self._blind(ps, u, rng)
        if cs.n_lookups:
            commit([(BASIS_LAGRANGE, self.lagr[nm % t].ptr) for t in range(cs.n_lookups) for nm in ("pa%d", "ps%d")])
            if self.d_status.download()[:, 0].any():
                raise H2BError(-5, "permute_expression_pair: an input value is not in the table (ConstraintSystemFailure)")
            self.d2h_bytes += 32 * cs.n_lookups
        beta, gamma = tr.squeeze(), tr.squeeze()
        bl, gl = to_limbs(beta), to_limbs(gamma)
        mark("phase1 lookup permuted")
        perm_names = [nm % t for t in range(cs.n_lookups) for nm in ("pa%d", "ps%d")]
        side_transforms(perm_names)
        # ---- product columns + the vanishing argument's random polynomial
        col_ptr = {"c": cs.lagr["c"].ptr}
        col_ptr.update({nm: self.lagr[nm].ptr for nm in cs.adv_names})
        for s in range(cs.n_sets):
            part = cs.perm_cols[s * cs.chunk:(s + 1) * cs.chunk]
            cols = (C.c_void_p * len(part))(*[col_ptr[nm] for nm in part])
            sig = (C.c_void_p * len(part))(*[cs.lagr["sigma_" + nm].ptr for nm in part])
            start = None if s == 0 else vp(self.lagr["zp%d" % (s - 1)].at(u))  # chained through the previous set's closing value
            ctx.check(lib.h2b_permutation_product_dev(ctx.h, cols, sig, len(part), s * cs.chunk, vp(bl.ctypes.data), vp(gl.ctypes.data), k, bf,
                                                      start, vp(self.lagr["zp%d" % s].ptr)))
        for t in range(cs.n_lookups):
            ctx.check(lib.h2b_lookup_product_dev(ctx.h, vp(lk_in[t]), vp(cs.lagr["table"].ptr), vp(self.lagr["pa%d" % t].ptr),
                                                 vp(self.lagr["ps%d" % t].ptr), vp(bl.ctypes.data), vp(gl.ctypes.data), k, bf,
                                                 vp(self.lagr["zl%d" % t].ptr)))
        prod_names = ["zp%d" % s for s in range(cs.n_sets)] + ["zl%d" % t for t in range(cs.n_lookups)]
        for nm in prod_names:
            self._blind(self.lagr[nm], u + 1, rng)
        side_transforms(prod_names)  # beside the commitments below
        commit([(BASIS_LAGRANGE, self.lagr[nm].ptr) for nm in prod_names] + [(BASIS_MONOMIAL, self.rnd.ptr)])
        y = tr.squeeze()
        yl = to_limbs(y)
        mark("phase2 products+random")
        ctx.check(lib.h2b_ctx_side_join(ctx.h))  # every column is now in coefficient and extended form
        mark("transforms")
        # ---- quotient: gate, permutation and lookup terms folded with y on the extended coset
        kw = dict(beta=bl, gamma=gl, theta=to_limbs(theta), y=yl)
        ctx.check(lib.h2b_poly_zero(ctx.h, self.h.h))
        for g, g_res, js in cs.gate_programs:
            bg = ev.BoundGraph(g, g_res, fixed=[cs.ext["q%d" % j].ptr for j in js], advice=[self.ext["a%d" % j].ptr for j in js], **kw)
            ctx.check(lib.h2b_quotient_graph_dev(ctx.h, C.byref(bg.struct), k, ext_k, vp(self.h.ptr)))
        ext_ptr = {"c": cs.ext["c"].ptr}
        ext_ptr.update({nm: self.ext[nm].ptr for nm in cs.adv_names})
        npc = len(cs.perm_cols)
        tz = (C.c_void_p * cs.n_sets)(*[self.ext["zp%d" % s].ptr for s in range(cs.n_sets)])
        tc = (C.c_void_p * npc)(*[ext_ptr[nm] for nm in cs.perm_cols])
        ts = (C.c_void_p * npc)(*[cs.ext["sigma_" + nm].ptr for nm in cs.perm_cols])
        ctx.check(lib.h2b_permutation_fold_dev(ctx.h, tz, cs.n_sets, tc, ts, npc, cs.chunk, vp(cs.ext["l0"].ptr), vp(cs.ext["l_last"].ptr),
                                               vp(cs.ext["l_active"].ptr), vp(bl.ctypes.data), vp(gl.ctypes.data), vp(yl.ctypes.data), bf, k, ext_k,
                                               vp(self.h.ptr)))
        for t in range(cs.n_lookups):
            if L == 0:
                blk = ev.BoundGraph(cs.lk_graph, cs.lk_res, fixed=[cs.ext["q_lookup"].ptr, cs.ext["table"].ptr], advice=[self.ext["a0"].ptr], **kw)
            else:
                blk = ev.BoundGraph(cs.lk_graph, cs.lk_res, fixed=[cs.ext["table"].ptr], advice=[self.ext["l%d" % t].ptr], **kw)
            ctx.check(lib.h2b_lookup_fold_dev(ctx.h, C.byref(blk.struct), vp(self.ext["zl%d" % t].ptr), vp(self.ext["pa%d" % t].ptr),
                                              vp(self.ext["ps%d" % t].ptr), vp(cs.ext["l0"].ptr), vp(cs.ext["l_last"].ptr),
                                              vp(cs.ext["l_active"].ptr), k, ext_k, vp(self.h.ptr)))
        ctx.check(lib.h2b_divide_by_vanishing_poly_dev(ctx.h, vp(self.h.ptr), k, ext_k))
        ctx.check(lib.h2b_extended_to_coeff_dev(ctx.h, vp(self.h.ptr), ext_k))
        mark("quotient")
        pieces = cs.degree - 1
        commit([(BASIS_MONOMIAL, self.h.at(j * n)) for j in range(pieces)])
        x = tr.squeeze()
        mark("phase3 h pieces")
        # ---- evaluations at x and its rotations
        w = pow(ROOT_OF_UNITY, 1 << (28 - k), R_MOD)
        rot = lambda r: x * pow(w, r % n, R_MOD) % R_MOD
        last = -(bf + 1)
        queries = [("a%d" % j, self.coef["a%d" % j].ptr, r) for j in range(A) for r in (0, 1, 2, 3)]
        queries += [("l%d" % t, self.coef["l%d" % t].ptr, 0) for t in range(L)]
        queries += [(nm, cs.coeff[nm].ptr, 0) for nm in cs.fixed_names + cs.sigma_names]
        for s in range(cs.n_sets):  # every set at x and omega x; all but the last one also at omega^last x
            queries += [("zp%d" % s, self.coef["zp%d" % s].ptr, r) for r in ((0, 1, last) if s < cs.n_sets - 1 else (0, 1))]
        for t in range(cs.n_lookups):
            queries += [("pa%d" % t, self.coef["pa%d" % t].ptr, 0), ("pa%d" % t, self.coef["pa%d" % t].ptr, -1),
                        ("ps%d" % t, self.coef["ps%d" % t].ptr, 0), ("zl%d" % t, self.coef["zl%d" % t].ptr, 0),
                        ("zl%d" % t, self.coef["zl%d" % t].ptr, 1)]
        queries += [("h%d" % j, self.h.at(j * n), 0) for j in range(pieces)] + [("rnd", self.rnd.ptr, 0)]
        m = len(queries)
        polys = (C.c_void_p * m)(*[p for _, p, _ in queries])
        xs = np.stack([to_limbs(rot(r)) for _, _, r in queries])
        ev_out = np.empty((m, 4), dtype=np.uint64)
        ctx.check(lib.h2b_eval_polynomial_batch_dev(ctx.h, polys, vp(xs.ctypes.data), m, n, vp(ev_out.ctypes.data)))
        self.d2h_bytes += m * 32
        tr.absorb(ev_out)
        res["evals"] = {(nm, r): ev_out[i] for i, (nm, _, r) in enumerate(queries)}
        res["challenges"] = dict(theta=theta, beta=beta, gamma=gamma, y=y, x=x)
        mark("evaluations")
        # ---- SHPLONK-shaped opening: per rotation set sum_i v^i p_i, divided by (X - point) for every point of the set
        v_ch, mu = tr.squeeze(), tr.squeeze()
        by_rot = {}
        for nm, ptr, r in queries:
            by_rot.setdefault(ptr, (nm, []))[1].append(r)
        groups = {}
        for ptr, (nm, rots) in by_rot.items():
            groups.setdefault(tuple(rots), []).append(ptr)
        sets = sorted(groups.items(), key=lambda kv: (len(kv[0]), kv[0]))  # deterministic order: by rotation set

        def run_sets(which, bufs):
            """sum over the given rotation sets of mu^s * (sum_i v^i p_i) / prod (X - point); result in bufs[2]"""
            f, qd, acc = bufs
            first = True
            for si in which:
                rots, plist = sets[si]
                self._lincomb(plist, [pow(v_ch, i, R_MOD) for i in range(len(plist))], f)
                src, dst = f, qd
                for r in rots:  # successive divisions by (X - point): the quotient by the set's vanishing polynomial
                    z = to_limbs(rot(r))
                    ctx.check(lib.h2b_kate_division_dev(ctx.h, vp(src.ptr), n, vp(z.ctypes.data), vp(dst.ptr)))
                    # kate_division writes the n - 1 quotient coefficients; the buffer is reused as an n-coefficient
                    # polynomial (next division, linear combination), so its top coefficient is cleared
                    ctx.check(lib.h2b_poly_copy_dev(ctx.h, vp(dst.at(n - 1)), vp(self.zero.ptr), 1))
                    src, dst = dst, src
                mu_s = pow(mu, si, R_MOD)
                if first:
                    self._lincomb([src.ptr], [mu_s], acc)
                    first = False
                else:
                    self._lincomb([acc.ptr, src.ptr], [1, mu_s], acc)
            return not first

        # the rotation sets are independent: every other one on the side queue (own scratch), the rest on the main queue
        side_sets = list(range(0, len(sets), 2))
        main_sets = list(range(1, len(sets), 2))
        ctx.check(lib.h2b_ctx_side_begin(ctx.h))
        try:
            run_sets(side_sets, self.tmp_side)
        finally:
            ctx.check(lib.h2b_ctx_side_end(ctx.h))
        have_main = run_sets(main_sets, self.tmp[:3])
        ctx.check(lib.h2b_ctx_side_join(ctx.h))
        if have_main:
            self._lincomb([self.tmp[2].ptr, self.tmp_side[2].ptr], [1, 1], self.tmp[2])
        else:
            ctx.check(lib.h2b_poly_copy_dev(ctx.h, vp(self.tmp[2].ptr), vp(self.tmp_side[2].ptr), n))
        mark("shplonk arithmetic")
        commit([(BASIS_MONOMIAL, self.tmp[2].ptr)])
        u_ch = tr.squeeze()
        # final quotient: L(X) = h_spl-weighted combination, W' = L / (X - u) (the remainder is dropped by kate_division)
        ul = to_limbs(u_ch)
        ctx.check(lib.h2b_kate_division_dev(ctx.h, vp(self.tmp[2].ptr), n, vp(ul.ctypes.data), vp(self.tmp[3].ptr)))
        ctx.check(lib.h2b_poly_copy_dev(ctx.h, vp(self.tmp[3].at(n - 1)), vp(self.zero.ptr), 1))
        cm = self._commit([(BASIS_MONOMIAL, self.tmp[3].ptr)])
        res["commitments"] += list(cm)
        res["h2d_bytes"], res["d2h_bytes"] = self.h2d_bytes, self.d2h_bytes
        mark("phase4-5 openings")
        if trace is not None:
            import sys
            print("prover trace (ms): " + ", ".join("%s=%.2f" % (l, 1e3 * (t - trace[i][1])) for i, (l, t) in enumerate(trace[1:])), file=sys.stderr)
        return res

    def free(self):
        for p in self.polys:
            p.free()


class _View:
    """n rows of a larger device polynomial, with the upload / pointer surface of Poly (an advice column inside the block the
    assignment kernels write)"""

    def __init__(self, parent: Poly, offset: int, n: int):
        self.parent, self.offset, self.n = parent, offset, n
        self.ptr = parent.at(offset)

    def upload(self, host: np.ndarray, offset: int = 0):
        self.parent.upload(host, self.offset + offset)

    def download(self, offset: int = 0, n: int | None = None) -> np.ndarray:
        return self.parent.download(self.offset + offset, self.n - offset if n is None else n)

    def at(self, elem_offset: int) -> int:
        return self.ptr + 32 * elem_offset

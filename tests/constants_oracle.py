"""Several constants columns (BaseCircuitParams::num_fixed = F, F >= 0) of a halo2-base builder, restated on top of the existing
oracles for tests/test_oracle_constants.py and tests/test_gpu_constants.py.  Permutation columns [c, c1.., c{F-1}, a0.., l0..,
i0..]: constants column f is permutation column f, a_j is F + j, l_t is F + A + t, i_m is F + A + L + m.

  assign_constants    CopyConstraintManager::assign_raw's placement (virtual_region/copy_constraints.rs:135-152) literally: the
                      constant equalities sorted by (constant, cell), each new constant at (fixed_col, fixed_offset), fixed_col
                      stepping left to right and wrapping to the next row ("left to right, then top to bottom"); config[0] of an
                      empty column list (F = 0) and a row >= u (halo2's assign_fixed) panic as they do there;
  copy_sequence       the copy calls of BaseCircuitBuilder::synthesize with F constants columns: break copies, lookup copies,
                      advice equalities sorted by (a, b), constant equalities as (the constant's cell) ~ raw(cell), then
                      assign_instances' copies (instance_oracle.copy_sequence's order);
  const_columns       the F constants columns keygen fills (canonical values, zero elsewhere);
  mock_run            builder_oracle.run's keygen pass and checks in its order, with the capacity panic of F columns in place of
                      its one-column one, instance_oracle.mock_run's instance reports, and distinct_constants;
  check               ProverSession.check's copy reports over [c.., a0.., l0.., i0..];
  quotient_identity   instance_oracle.quotient_identity with the F constants columns first in the permutation terms;
  create_proof        instance_oracle.create_proof (oracle/prover_ref's flow with public inputs) with F constants columns.
With F = 1 each gives the existing oracle's result (tests/test_oracle_constants.py checks it)."""
from __future__ import annotations
import numpy as np
import builder_oracle as bo
import instance_oracle as io
import keygen_oracle as ko
import mock_oracle as mo
import prover_check as pc
from oracle import pyref
from oracle.prover_ref import Transcript, fr_bytes, g1_bytes

R = pyref.R
BLINDING_FACTORS = 6


def const_names(F: int) -> list:
    return ["c%d" % f if f else "c" for f in range(F)]


def assign_constants(constant_equalities, F: int, u: int, k: int) -> dict:
    """{canonical constant: (constants column, row)}"""
    config = list(range(F))
    cells = {}
    fixed_col = fixed_offset = 0
    for c, _ in sorted((int(c) % R, int(i)) for c, i in constant_equalities):
        if c not in cells:
            if fixed_col >= len(config):
                raise bo.Panic("index out of bounds: the len is %d but the index is %d" % (len(config), fixed_col))
            if fixed_offset >= u:
                raise bo.Panic("NotEnoughRowsAvailable { current_k: %d }" % k)
            cells[c] = (config[fixed_col], fixed_offset)
            fixed_col += 1
            if fixed_col >= len(config):
                fixed_col = 0
                fixed_offset += 1
    return cells


def _raw_ids(bps, n: int, F: int, p) -> np.ndarray:
    """keygen_oracle._raw_ids with the advice columns after F constants columns"""
    return ko._raw_ids(bps, n, p) + (F - 1) * n


def copy_sequence(k: int, A: int, L: int, max_rows: int, b: dict, F: int = 1, instances=None):
    """(pairs: the copy calls as (E, 2) cell ids in call order, const_cells: {canonical constant: cell id f 2^k + row},
    break points).  With F = 1 it is keygen_oracle.copy_sequence (and instance_oracle.copy_sequence with instances)."""
    n = 1 << k
    u = n - (BLINDING_FACTORS + 1)
    bps = bo.assign_with_constraints(b["contexts"], A, max_rows, record=False)[0]
    consts = np.asarray(b["constants"], dtype=np.uint64)
    idx = np.asarray(b["constant_index"], dtype=np.int64)
    placed = assign_constants(zip(consts.tolist(), idx.tolist()), F, u, k)
    parts = [np.array([[(F + 1 + j) * n, (F + j) * n + bp] for j, bp in enumerate(bps)], dtype=np.int64).reshape(-1, 2)]
    if L:
        i = np.arange(len(b["lookups"]), dtype=np.int64)
        parts.append(np.stack([_raw_ids(bps, n, F, b["lookups"]), (F + A + i % L) * n + i // L], axis=1))
    E = np.asarray(b["advice_equalities"], dtype=np.int64).reshape(-1, 2)
    E = E[np.lexsort((E[:, 1], E[:, 0]))]
    parts.append(np.stack([_raw_ids(bps, n, F, E[:, 0]), _raw_ids(bps, n, F, E[:, 1])], axis=1).reshape(-1, 2))
    order = np.lexsort((idx, consts))
    const_cells = {c: col * n + row for c, (col, row) in placed.items()}
    cell = np.array([const_cells[int(c)] for c in consts[order].tolist()], dtype=np.int64)
    parts.append(np.stack([cell, _raw_ids(bps, n, F, idx[order])], axis=1).reshape(-1, 2))
    N = len(b["selectors"])
    for m, ix in enumerate(instances or []):
        ix = np.asarray(ix, dtype=np.int64).reshape(-1)
        for r, p in enumerate(ix.tolist()):
            if p >= N:
                raise bo.Panic("instance not assigned")
            if r >= u:
                raise bo.Panic("NotEnoughRowsAvailable { current_k: %d }" % k)
        parts.append(np.stack([_raw_ids(bps, n, F, ix), (F + A + L + m) * n + np.arange(len(ix))], axis=1).reshape(-1, 2))
    return np.concatenate(parts).astype(np.int64), const_cells, [int(x) for x in bps]


def const_columns(k: int, F: int, const_cells: dict) -> list:
    """the F constants columns as lists of canonical values"""
    n = 1 << k
    cols = [[0] * n for _ in range(F)]
    for c, cell in const_cells.items():
        cols[cell // n][cell % n] = c
    return cols


def mock_run(k: int, A: int, L: int, sel: bool, bits: int, max_rows: int, b: dict, values, F: int = 1, instances=(), public=(),
             max_report: int = 16) -> dict:
    """MockProver.run's result with F constants columns, as builder_oracle.run (instance_oracle.mock_run with instance columns)
    gives it for one column: F changes only the capacity panic.  Panics in builder_oracle.run's order: the walk and the lookups,
    then the constants (assign_constants with F columns), then the cells of the equalities; plus distinct_constants = D"""
    u = (1 << k) - (BLINDING_FACTORS + 1)
    if any(len(p) > u for p in public):
        raise bo.Panic("InstanceTooLarge")
    N = len(values)
    bps, raw, _ = bo.assign_with_constraints(b["contexts"], A, max_rows)
    bo.assign_lookups_in_phase(b["lookups"], lambda p: raw[p], N, A, L, sel, max_rows)
    consts, idx = [int(c) % R for c in b["constants"]], [int(i) for i in b["constant_index"]]
    assign_constants(zip(consts, idx), F, u, k)
    no_consts = dict(b, constants=np.zeros(0, dtype=np.uint64), constant_index=np.zeros(0, dtype=np.uint64))
    res = bo.run(k, A, L, sel, bits, max_rows, no_consts, values, max_report)  # gates, lookups, advice equalities
    if any(i >= N for i in idx):
        raise bo.Panic("virtual cell not assigned")
    res["constants"] = bo._report([i for i, (c, x) in enumerate(zip(consts, idx)) if int(values[x]) % R != c], max_report)
    res["constant_cells"] = [raw[idx[i]] for i in res["constants"][1]]
    res["satisfied"] = res["satisfied"] and res["constants"][0] == 0
    if instances:  # the instance reports do not depend on the constants
        got = io.mock_run(k, A, L, sel, bits, max_rows, no_consts, values, instances, public, max_report)
        res.update({key: got[key] for key in ("instances", "instance_cells")})
        res["satisfied"] = res["satisfied"] and not any(c for c, _ in res["instances"])
    res["distinct_constants"] = len({int(c) % R for c in b["constants"]})
    return res


def check(k: int, F: int, c_cols, sigma, cols, public=(), max_report: int = 16) -> list:
    """the copy reports of ProverSession.check, one per permutation column [c.., a0.., l0.., i0..]: cells whose value differs from
    the one sigma names.  c_cols: the F constants columns, cols: the A + L advice columns (rows >= u read as 0), public: the values
    of each instance column (rows [0, len), zero after); all canonical"""
    n = 1 << k
    u = n - (BLINDING_FACTORS + 1)
    body = [list(c) for c in cols] + [list(p) + [0] * (n - len(p)) for p in public]
    value = lambda c, r: int(c_cols[c][r]) % R if c < F else (int(body[c - F][r]) % R if r < u else 0)
    targets, bad = mo.decode_sigma(k, sigma)
    assert not bad, bad[:1]
    return [mo._report([r for r in range(n) if value(c, r) != value(*targets[(c, r)])], max_report) for c in range(len(sigma))]


def quotient_identity(res: dict, k: int, A: int, L: int, selector_lookup: bool, F: int, public=()) -> tuple[int, int]:
    """(left, right) of fold(terms)(x) == h(x) (x^n - 1) with F constants columns first in the permutation and instance columns
    last; public: per instance column canonical values"""
    bf = BLINDING_FACTORS
    n = 1 << k
    u = n - (bf + 1)
    n_lookups = L if L else (1 if selector_lookup else 0)
    degree = 4 if L else (5 if n_lookups else 3)
    chunk = degree - 2
    ch = res["challenges"]
    beta, gamma, y, x = ch["beta"], ch["gamma"], ch["y"], ch["x"]
    inst = {"i%d" % m: sum(int(v) * pc.lagrange_at(k, r, x) for r, v in enumerate(col)) % R for m, col in enumerate(public)}
    e = lambda name, r=0: inst[name] if name in inst else pc.fr(res["evals"][(name, r)])
    last = -(bf + 1)
    l0, l_last = pc.lagrange_at(k, 0, x), pc.lagrange_at(k, u, x)
    l_blind = sum(pc.lagrange_at(k, i, x) for i in range(u + 1, n)) % R
    l_active = (1 - l_last - l_blind) % R
    v = 0
    for j in range(A):
        a = "a%d" % j
        v = (v * y + e("q%d" % j) * (e(a, 0) + e(a, 1) * e(a, 2) - e(a, 3))) % R
    perm = const_names(F) + ["a%d" % j for j in range(A)] + ["l%d" % t for t in range(L)] + list(inst)
    n_sets = (len(perm) + chunk - 1) // chunk
    v = (v * y + (1 - e("zp0")) * l0) % R
    zl_ = e("zp%d" % (n_sets - 1))
    v = (v * y + (zl_ * zl_ - zl_) * l_last) % R
    for s in range(1, n_sets):
        v = (v * y + (e("zp%d" % s) - e("zp%d" % (s - 1), last)) * l0) % R
    for s in range(n_sets):
        left, right = e("zp%d" % s, 1), e("zp%d" % s, 0)
        for cidx in range(s * chunk, min(len(perm), (s + 1) * chunk)):
            val = e(perm[cidx])
            left = left * (val + beta * e("sigma_" + perm[cidx]) + gamma) % R
            right = right * (val + beta * pow(pc.DELTA, cidx, R) % R * x + gamma) % R
        v = (v * y + (left - right) * l_active) % R
    for t in range(n_lookups):
        pa, pa_p, ps = e("pa%d" % t, 0), e("pa%d" % t, -1), e("ps%d" % t, 0)
        zl, zl_n = e("zl%d" % t, 0), e("zl%d" % t, 1)
        inp = e("q_lookup") * e("a0") % R if L == 0 else e("l%d" % t)
        v = (v * y + (1 - zl) * l0) % R
        v = (v * y + (zl * zl - zl) * l_last) % R
        v = (v * y + (zl_n * (pa + beta) % R * (ps + gamma) - zl * (inp + beta) % R * (e("table") + gamma)) * l_active) % R
        v = (v * y + (pa - ps) * l0) % R
        v = (v * y + (pa - ps) * (pa - pa_p) % R * l_active) % R
    xn = pow(x, n, R)
    h = sum(e("h%d" % j) * pow(xn, j, R) for j in range(degree - 1)) % R
    return v % R, h * (xn - 1) % R


# ------------------------------------------------------------------------------------------------ the prover with constants columns
# instance_oracle.create_proof (oracle/prover_ref's flow with public inputs) with F constants columns: the constants columns are
# fixed columns, listed after the table, transformed with the fixed side, queried at x and placed first in the permutation.
def create_proof(k: int, A: int, L: int, selector_lookup: bool, F: int, fixed: dict, sigma: list, virtual: list, break_points: list,
                 lookup_cells: list, random_poly: list, blind, bases_m: list, bases_l: list, instances=None) -> dict:
    """instance_oracle.create_proof with F constants columns c, c1.. (fixed columns, after the table; the first F permutation
    columns): `fixed` holds them by name, `sigma` has one column per permutation column [c, c1.., a0.., l0.., i0..].  With F = 1 it
    is instance_oracle.create_proof.  Returns
    {"commitments": [96-byte strings], "evals": [(name, rotation, value)], "challenges": {...}}."""
    n = 1 << k
    selector_lookup = selector_lookup and L == 0
    n_lookups = L if L else (1 if selector_lookup else 0)
    degree = 4 if L else (5 if selector_lookup else 3)
    chunk = degree - 2
    ext_k = k + (1 if degree == 3 else 2)
    ne = 1 << ext_k
    bf = BLINDING_FACTORS
    u = n - (bf + 1)
    adv_names = ["a%d" % j for j in range(A)] + ["l%d" % t for t in range(L)]
    instances = [] if instances is None else [[int(v) % R for v in col] for col in instances]
    inst_names = ["i%d" % m for m in range(len(instances))]
    consts = const_names(F)
    perm_cols = consts + adv_names + inst_names
    n_sets = (len(perm_cols) + chunk - 1) // chunk
    fixed_names = ["q%d" % j for j in range(A)] + (["q_lookup"] if selector_lookup else []) + (["table"] if n_lookups else []) + consts
    w = pyref.omega_for(k)
    tr = Transcript()
    commitments, lagr, coef, ext = [], {}, {}, {}

    def commit(items):
        """items: (basis, values); basis 0 = monomial (coefficients), 1 = lagrange"""
        out = []
        for basis, vals in items:
            cm = g1_bytes(pyref.msm_naive(vals, bases_l if basis else bases_m))
            commitments.append(cm)
            out.append(cm)
        return b"".join(out)

    def transforms(names):
        for nm in names:
            coef[nm] = pyref.lagrange_to_coeff(lagr[nm], k)
            ext[nm] = pyref.coeff_to_extended(coef[nm], k, ext_k)

    def blind_rows(col, first_row):
        col[first_row:] = blind(n - first_row)

    # the fixed side in its three forms
    fx = {nm: list(fixed[nm]) for nm in fixed_names}
    fx.update({"sigma_" + nm: list(sg) for nm, sg in zip(perm_cols, sigma)})
    fx["l0"] = [1] + [0] * (n - 1)
    fx["l_last"] = [1 if i == u else 0 for i in range(n)]
    fx["l_active"] = [1 if i < u else 0 for i in range(n)]
    fx_coef = {nm: pyref.lagrange_to_coeff(v, k) for nm, v in fx.items()}
    fx_ext = {nm: pyref.coeff_to_extended(c, k, ext_k) for nm, c in fx_coef.items()}

    # ---- the public values: into the transcript (common_scalar, column by column), rows [0, len) of their columns
    for nm, col in zip(inst_names, instances):
        if len(col) > u:
            raise ValueError("InstanceTooLarge")
        tr.absorb(b"".join(fr_bytes(v) for v in col))
        lagr[nm] = col + [0] * (n - len(col))
    # ---- phase 0: assignment (single_phase.rs:273-312, lookups.rs:130-155), blinding rows, advice commitments
    cols = pyref.assign_witnesses([list(virtual)], [int(b) for b in break_points], A, n)
    if L:
        cols += pyref.assign_lookups(list(lookup_cells), L, n)
    for nm, col in zip(adv_names, cols):
        lagr[nm] = col
        blind_rows(col, u)
    tr.absorb(commit([(1, lagr[nm]) for nm in adv_names]))
    theta = tr.squeeze()
    transforms(adv_names + inst_names)
    # ---- lookups: compressed input, permuted pair
    lk_in = []
    for t in range(n_lookups):
        inp = [q * a % R for q, a in zip(fx["q_lookup"], lagr["a0"])] if L == 0 else lagr["l%d" % t]
        lk_in.append(inp)
        pair = pyref.permute_expression_pair(inp[:u], fx["table"][:u])
        if pair is None:
            raise ValueError("ConstraintSystemFailure: a lookup input is not in the table")
        for nm, vals in zip(("pa%d" % t, "ps%d" % t), pair):
            lagr[nm] = list(vals) + [0] * (n - u)
            blind_rows(lagr[nm], u)
    perm_names = [nm % t for t in range(n_lookups) for nm in ("pa%d", "ps%d")]
    if n_lookups:
        tr.absorb(commit([(1, lagr[nm]) for nm in perm_names]))
    beta, gamma = tr.squeeze(), tr.squeeze()
    transforms(perm_names)
    # ---- product columns
    col_of = lambda nm: fx[nm] if nm in consts else lagr[nm]
    start = 1
    for s in range(n_sets):
        z = [start]
        for i in range(u):
            num = den = 1
            for cidx in range(s * chunk, min(len(perm_cols), (s + 1) * chunk)):
                v = col_of(perm_cols[cidx])[i]
                num = num * (v + beta * pow(pyref.DELTA, cidx, R) % R * pow(w, i, R) + gamma) % R
                den = den * (v + beta * fx["sigma_" + perm_cols[cidx]][i] + gamma) % R
            z.append(z[-1] * num % R * pow(den, -1, R) % R)
        start = z[u]
        lagr["zp%d" % s] = z + [0] * (n - u - 1)
    for t in range(n_lookups):
        z = [1]
        pa, ps = lagr["pa%d" % t], lagr["ps%d" % t]
        for i in range(u):
            z.append(z[-1] * (lk_in[t][i] + beta) % R * (fx["table"][i] + gamma) % R * pow((pa[i] + beta) * (ps[i] + gamma) % R, -1, R) % R)
        lagr["zl%d" % t] = z + [0] * (n - u - 1)
    prod_names = ["zp%d" % s for s in range(n_sets)] + ["zl%d" % t for t in range(n_lookups)]
    for nm in prod_names:
        blind_rows(lagr[nm], u + 1)
    transforms(prod_names)
    rnd = [c % R for c in random_poly]
    tr.absorb(commit([(1, lagr[nm]) for nm in prod_names] + [(0, rnd)]))
    y = tr.squeeze()
    # ---- quotient on the extended coset: gates (Horner in y), permutation terms, lookup terms, division by X^n - 1
    rot = lambda col, idx, r: pyref.rotate(col, idx, r, k, ext_k)
    values = []
    for idx in range(ne):
        v = 0
        for j in range(A):
            a = ext["a%d" % j]
            v = (v * y + fx_ext["q%d" % j][idx] * (a[idx] + rot(a, idx, 1) * rot(a, idx, 2) - rot(a, idx, 3))) % R
        values.append(v)
    ext_of = lambda nm: fx_ext[nm] if nm in consts else ext[nm]
    values = pyref.permutation_terms([ext["zp%d" % s] for s in range(n_sets)], [ext_of(nm) for nm in perm_cols],
                                     [fx_ext["sigma_" + nm] for nm in perm_cols], chunk, fx_ext["l0"], fx_ext["l_last"], fx_ext["l_active"],
                                     beta, gamma, y, bf, k, ext_k, values)
    for t in range(n_lookups):
        if L == 0:
            inp_e = [q * a % R for q, a in zip(fx_ext["q_lookup"], ext["a0"])]
        else:
            inp_e = ext["l%d" % t]
        tv = [(i_ + beta) * (t_ + gamma) % R for i_, t_ in zip(inp_e, fx_ext["table"])]
        values = pyref.lookup_terms(tv, ext["zl%d" % t], ext["pa%d" % t], ext["ps%d" % t], fx_ext["l0"], fx_ext["l_last"], fx_ext["l_active"],
                                    beta, gamma, y, k, ext_k, values)
    we = pyref.omega_for(ext_k)
    for idx in range(ne):
        x_row = pyref.ZETA * pow(we, idx, R) % R
        values[idx] = values[idx] * pow(pow(x_row, n, R) - 1, -1, R) % R
    h = pyref.extended_to_coeff(values, k, ext_k)
    pieces = degree - 1
    assert not any(h[pieces * n:]), "the quotient has degree (degree - 1) n at most"
    tr.absorb(commit([(0, h[j * n:(j + 1) * n]) for j in range(pieces)]))
    x = tr.squeeze()
    # ---- evaluations
    point = lambda r: x * pow(w, r % n, R) % R
    last = -(bf + 1)
    queries = [("a%d" % j, coef["a%d" % j], r) for j in range(A) for r in (0, 1, 2, 3)]
    queries += [("l%d" % t, coef["l%d" % t], 0) for t in range(L)]
    queries += [(nm, fx_coef[nm], 0) for nm in fixed_names + ["sigma_" + nm for nm in perm_cols]]
    for s in range(n_sets):
        queries += [("zp%d" % s, coef["zp%d" % s], r) for r in ((0, 1, last) if s < n_sets - 1 else (0, 1))]
    for t in range(n_lookups):
        queries += [("pa%d" % t, coef["pa%d" % t], 0), ("pa%d" % t, coef["pa%d" % t], -1), ("ps%d" % t, coef["ps%d" % t], 0),
                    ("zl%d" % t, coef["zl%d" % t], 0), ("zl%d" % t, coef["zl%d" % t], 1)]
    queries += [("h%d" % j, h[j * n:(j + 1) * n], 0) for j in range(pieces)] + [("rnd", rnd, 0)]
    evals = [(nm, r, pyref.eval_polynomial(poly, point(r))) for nm, poly, r in queries]
    tr.absorb(b"".join(fr_bytes(v) for _, _, v in evals))
    # ---- SHPLONK-shaped opening: per rotation set sum_i v^i p_i divided by every (X - point) of the set
    v_ch, mu = tr.squeeze(), tr.squeeze()
    by_poly = {}
    for nm, poly, r in queries:
        by_poly.setdefault(id(poly), (poly, []))[1].append(r)
    groups = {}
    for poly, rots in by_poly.values():
        groups.setdefault(tuple(rots), []).append(poly)
    sets = sorted(groups.items(), key=lambda kv: (len(kv[0]), kv[0]))
    total = [0] * n
    for si, (rots, plist) in enumerate(sets):
        f = [sum(pow(v_ch, i, R) * p[c] for i, p in enumerate(plist)) % R for c in range(n)]
        for r in rots:
            f = pyref.kate_division(f, point(r)) + [0]  # n - 1 quotient coefficients, kept as an n-coefficient polynomial
        ms = pow(mu, si, R)
        total = [(a + ms * b) % R for a, b in zip(total, f)]
    tr.absorb(commit([(0, total)]))
    u_ch = tr.squeeze()
    commit([(0, pyref.kate_division(total, u_ch) + [0])])
    return {"commitments": commitments, "evals": evals, "challenges": dict(theta=theta, beta=beta, gamma=gamma, y=y, x=x)}

"""Public inputs (instance columns) of a halo2-base builder, restated on top of the existing oracles for
tests/test_oracle_instance.py and tests/test_gpu_instance.py.  Instance column m is permutation column 1 + A + L + m.

  copy_sequence       keygen_oracle.copy_sequence plus the copies of BaseCircuitBuilder::assign_instances, which run after the
                      region (gates/circuit/builder.rs:289-309): raw(index_m[r]) ~ (i_m, r), column by column, row by row;
  mock_run            builder_oracle.run plus the instance check: value(raw(index_m[r])) == public_m[r];
  check               ProverSession.check's reports with instance columns: mock_oracle's copy check over [c, a0.., l0.., i0..];
  theta               the first challenge: Blake2b over the public values (32 Montgomery bytes each, column by column), then the
                      advice commitments;
  quotient_identity   prover_check.quotient_identity with the instance columns in the permutation terms and their evaluation at x
                      computed as the verifier does, sum_r public_m[r] L_r(x) (instance columns are not opened);
  create_proof        oracle/prover_ref.create_proof with instance columns, on plain Python integers."""
from __future__ import annotations
import hashlib
import numpy as np
import builder_oracle as bo
import keygen_oracle as ko
import mock_oracle as mo
import prover_check as pc
from oracle import pyref
from oracle.prover_ref import Transcript, fr_bytes, g1_bytes

R = pc.R
BLINDING_FACTORS = 6


def copy_sequence(k: int, A: int, L: int, max_rows: int, b: dict, instances=None):
    """(pairs, c_rows, break points) as keygen_oracle.copy_sequence, the instance copies appended; halo2-base's and halo2's
    panics at the first failing instance cell"""
    pairs, c_rows, bps = ko.copy_sequence(k, A, L, max_rows, b)
    if instances is None:
        return pairs, c_rows, bps
    n = 1 << k
    u = n - (BLINDING_FACTORS + 1)
    N = len(b["selectors"])
    parts = [pairs]
    for m, idx in enumerate(instances):
        idx = np.asarray(idx, dtype=np.int64).reshape(-1)
        for r, p in enumerate(idx.tolist()):
            if p >= N:
                raise bo.Panic("instance not assigned")
            if r >= u:
                raise bo.Panic("NotEnoughRowsAvailable { current_k: %d }" % k)
        parts.append(np.stack([ko._raw_ids(bps, n, idx), (1 + A + L + m) * n + np.arange(len(idx))], axis=1).reshape(-1, 2))
    return np.concatenate(parts).astype(np.int64), c_rows, bps


def mock_run(k: int, A: int, L: int, sel: bool, bits: int, max_rows: int, b: dict, values, instances, public, max_report: int = 16) -> dict:
    """builder_oracle.run with "instances" (per column: count and failing rows) and "instance_cells" (their raw cells)"""
    u = (1 << k) - (BLINDING_FACTORS + 1)
    if any(len(p) > u for p in public):
        raise bo.Panic("InstanceTooLarge")
    res = bo.run(k, A, L, sel, bits, max_rows, b, values, max_report)
    N = len(values)
    if any(int(p) >= N for idx in instances for p in idx):
        raise bo.Panic("instance not assigned")
    res["instances"], res["instance_cells"] = [], []
    for idx, pub in zip(instances, public):
        rep = bo._report([r for r, (p, v) in enumerate(zip(idx, pub)) if int(values[int(p)]) % R != int(v) % R], max_report)
        res["instances"].append(rep)
        res["instance_cells"].append([bo.raw_cell(res["break_points"], int(idx[r])) for r in rep[1]])
    res["satisfied"] = res["satisfied"] and not any(c for c, _ in res["instances"])
    return res


def check(k: int, c_col, sigma, cols, public, max_report: int = 16) -> list:
    """the copy reports of ProverSession.check, one per permutation column: cells whose value differs from the one sigma names.
    c_col: the constants column, cols: the A + L advice columns (rows >= u read as 0), public: the values of each instance
    column (rows [0, len), zero after); all canonical"""
    n = 1 << k
    u = n - (BLINDING_FACTORS + 1)
    body = [list(c) for c in cols] + [list(p) + [0] * (n - len(p)) for p in public]
    value = lambda c, r: int(c_col[r]) % R if c == 0 else (int(body[c - 1][r]) % R if r < u else 0)
    targets, bad = mo.decode_sigma(k, sigma)
    assert not bad, bad[:1]
    return [mo._report([r for r in range(n) if value(c, r) != value(*targets[(c, r)])], max_report) for c in range(len(sigma))]


def theta(public, advice_commitments) -> int:
    """public: per column (len x 4) Montgomery limbs; advice_commitments: 12 limbs each (affine, Montgomery)"""
    h = hashlib.blake2b(digest_size=64)
    for col in public:
        h.update(np.ascontiguousarray(col, dtype=np.uint64).tobytes())
    for cm in advice_commitments:
        h.update(np.ascontiguousarray(cm, dtype=np.uint64).tobytes())
    return int.from_bytes(h.digest(), "little") % R


def quotient_identity(res: dict, k: int, A: int, L: int, selector_lookup: bool, public) -> tuple[int, int]:
    """(left, right) of fold(terms)(x) == h(x) (x^n - 1) with instance columns; public: per column canonical values"""
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
    perm = ["c"] + ["a%d" % j for j in range(A)] + ["l%d" % t for t in range(L)] + list(inst)
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


# ------------------------------------------------------------------------------------------------ the prover with public inputs
# oracle/prover_ref.create_proof restated with instance columns (recalled halo2-axiom 0.5.3, KZG: QUERY_INSTANCE = false): the
# public values are absorbed as scalars, column by column, before the phase-0 advice commitments (padding zeros are not); a
# column of more than u values is InstanceTooLarge; instance columns are transformed like advice columns and enter the
# permutation product and terms, and are neither committed, blinded nor opened.  With no instance columns it is prover_ref's
# flow line for line (tests/test_oracle_instance.py checks the two give the same bytes).
def create_proof(k: int, A: int, L: int, selector_lookup: bool, fixed: dict, sigma: list, virtual: list, break_points: list,
                 lookup_cells: list, random_poly: list, blind, bases_m: list, bases_l: list, instances=None) -> dict:
    """oracle/prover_ref.create_proof with public inputs: `instances` holds the public values of each instance column (None:
    none, and then the result is prover_ref's); `sigma` has one column per permutation column [c, a0.., l0.., i0..].  Returns
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
    perm_cols = ["c"] + adv_names + inst_names
    n_sets = (len(perm_cols) + chunk - 1) // chunk
    fixed_names = ["q%d" % j for j in range(A)] + (["q_lookup"] if selector_lookup else []) + (["table"] if n_lookups else []) + ["c"]
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
    col_of = lambda nm: fx["c"] if nm == "c" else lagr[nm]
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
    ext_of = lambda nm: fx_ext["c"] if nm == "c" else ext[nm]
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

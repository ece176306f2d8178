"""halo2's selector compression (keygen_vk = keygen_vk_custom(.., compress_selectors = true), recalled from halo2-axiom 0.5.3;
DESIGN.md §2 conventions 11-14, §4.13) restated on plain Python integers for tests/test_oracle_selectors.py and
tests/test_gpu_selectors.py, on top of tests/halo2_proof_oracle.py and tests/constants_oracle.py (unchanged):

  process          convention 12 literally: degree-0 selectors alone first, in selector order; then greedy combinations of the
                   simple selectors within max_degree, never two active on one row;
  compress         the combination columns s0, s1.. of halo2-base's selectors q0.., [q_lookup] (root m + 1 where member m is
                   active) and the layout: fixed columns in column order [table], c.., s.. and in query order c.., [table], s..;
  selector_value   a member's substituted expression S prod_{t != root} (t - S), not normalised;
  create_proof     halo2_proof_oracle.create_proof with the compressed layout (the gate terms through the substitution);
  verify_proof     halo2_proof_oracle.verify_proof with the compressed layout."""
from __future__ import annotations
import numpy as np
import constants_oracle as co
import halo2_proof_oracle as hpo
from oracle import pyref
from oracle.prover_ref import fr_bytes

R = pyref.R
BLINDING_FACTORS = hpo.BLINDING_FACTORS


def process(degrees: list, max_degree: int, conflicts) -> list:
    """the combinations in column allocation order, each the selector indices in join order; conflicts[i][j]: i and j are
    active on a common row"""
    S = len(degrees)
    out = [[i] for i in range(S) if degrees[i] == 0]
    added = [False] * S
    for i in range(S):
        if degrees[i] == 0 or added[i]:
            continue
        assert degrees[i] <= max_degree
        added[i] = True
        d = degrees[i] - 1
        comb = [i]
        for j in range(i + 1, S):
            if d + len(comb) == max_degree:
                break
            if degrees[j] == 0 or added[j]:
                continue
            if any(conflicts[j][m] for m in comb):
                continue
            nd = max(d, degrees[j] - 1)
            if nd + len(comb) + 1 > max_degree:
                continue
            d = nd
            comb.append(j)
            added[j] = True
        out.append(comb)
    return out


def conflicts_of(columns: list) -> list:
    """conflicts[i][j] = some row has columns i and j both 1 (0/1 integer columns)"""
    act = [{r for r, v in enumerate(c) if v} for c in columns]
    return [[bool(a & b) for b in act] for a in act]


def substitute(s: int, root: int, ln: int) -> int:
    v = s % R
    for t in range(1, ln + 1):
        if t != root:
            v = v * (t - s) % R
    return v


def selector_value(lay: dict, sel: str, value_of) -> int:
    """selector `sel` as the gates read it: its column's value (value_of(column)) through the substitution"""
    col, root, ln = lay["selectors"][sel]
    return substitute(value_of(col), root, ln)


def selector_names(A: int, sel: bool) -> list:
    return ["q%d" % j for j in range(A)] + (["q_lookup"] if sel else [])


def max_degree(L: int, sel: bool) -> int:
    return 4 if L else (5 if sel else 3)


def compress(k: int, A: int, L: int, selector_lookup: bool, F: int, fixed: dict):
    """(the compressed fixed columns by name, the layout {"columns", "queries", "selectors": {name: (column, root, len)},
    "combinations": [[selector names in join order]]}) of halo2-base's columns q0.., [q_lookup], [table], c.. (0/1 selectors)"""
    sel = selector_lookup and L == 0
    names = selector_names(A, sel)
    for nm in names:
        if any(v not in (0, 1) for v in fixed[nm]):
            raise ValueError("selector %s holds a value other than 0 or 1" % nm)
    degrees = [0 if nm == "q_lookup" else 3 for nm in names]
    combos = process(degrees, max_degree(L, sel), conflicts_of([fixed[nm] for nm in names]))
    consts = ["c"] + ["c%d" % f for f in range(1, F)] if F else []
    lookup = ["table"] if (L or sel) else []
    out = {nm: list(fixed[nm]) for nm in lookup + consts}
    lay = {"columns": lookup + consts, "queries": consts + lookup, "selectors": {}, "combinations": []}
    n = 1 << k
    for c, comb in enumerate(combos):
        nm = "s%d" % c
        col = [0] * n
        for m, si in enumerate(comb):
            for r, v in enumerate(fixed[names[si]]):
                if v:
                    col[r] = m + 1
            lay["selectors"][names[si]] = (nm, m + 1, len(comb))
        out[nm] = col
        lay["columns"].append(nm)
        lay["queries"].append(nm)
        lay["combinations"].append([names[si] for si in comb])
    return out, lay


def shape(k: int, A: int, L: int, selector_lookup: bool, F: int, I: int, lay: dict) -> dict:
    """halo2_proof_oracle.shape with the fixed columns in the compressed query order"""
    return dict(hpo.shape(k, A, L, selector_lookup, F, I), fixed=list(lay["queries"]))


def phases(s: dict, lay: dict, fixed: dict, sigma: list, virtual: list, break_points: list, lookup_cells: list, random_poly: list, blind, bases_m: list,
           bases_l: list, instances: list, tr) -> dict:
    """halo2_proof_oracle.phases on the compressed layout `lay` (compress()): s["fixed"] lists the fixed columns in query order,
    each gate's selector is its substituted expression of its combination column, the selector lookup reads q_lookup's column."""
    k, n, A, L, ext_k, u = s["k"], s["n"], s["A"], s["L"], s["ext_k"], s["u"]
    bf, chunk, n_sets, n_lookups, consts, perm_cols = BLINDING_FACTORS, s["chunk"], s["n_sets"], s["n_lookups"], s["consts"], s["perm"]
    ne = 1 << ext_k
    adv_names = s["adv"]
    inst_names = ["i%d" % m for m in range(len(instances))]
    w = pyref.omega_for(k)
    lagr, coef, ext, commitments = {}, {}, {}, []

    def commit(items):
        for basis, vals in items:
            pt = pyref.msm_naive(vals, bases_l if basis else bases_m)
            commitments.append(pt)
            tr.write_point(pt)

    def transforms(names):
        for nm in names:
            coef[nm] = pyref.lagrange_to_coeff(lagr[nm], k)
            ext[nm] = pyref.coeff_to_extended(coef[nm], k, ext_k)

    def blind_rows(col, first_row):
        col[first_row:] = blind(n - first_row)

    fx = {nm: list(fixed[nm]) for nm in s["fixed"]}
    fx.update({"sigma_" + nm: list(sg) for nm, sg in zip(perm_cols, sigma)})
    fx["l0"] = [1] + [0] * (n - 1)
    fx["l_last"] = [1 if i == u else 0 for i in range(n)]
    fx["l_active"] = [1 if i < u else 0 for i in range(n)]
    fx_coef = {nm: pyref.lagrange_to_coeff(v, k) for nm, v in fx.items()}
    fx_ext = {nm: pyref.coeff_to_extended(c, k, ext_k) for nm, c in fx_coef.items()}
    for nm, col in zip(inst_names, instances):
        if len(col) > u:
            raise ValueError("InstanceTooLarge")
        for v in col:
            tr.common_scalar(v)
        lagr[nm] = list(col) + [0] * (n - len(col))
    cols = pyref.assign_witnesses([list(virtual)], [int(b) for b in break_points], A, n)
    if L:
        cols += pyref.assign_lookups(list(lookup_cells), L, n)
    for nm, col in zip(adv_names, cols):
        lagr[nm] = col
        blind_rows(col, u)
    commit([(1, lagr[nm]) for nm in adv_names])
    theta = tr.squeeze()
    transforms(adv_names + inst_names)
    lk_in = []
    for t in range(n_lookups):
        inp = [q * a % R for q, a in zip(fx[lay["selectors"]["q_lookup"][0]], lagr["a0"])] if L == 0 else lagr["l%d" % t]
        lk_in.append(inp)
        pair = pyref.permute_expression_pair(inp[:u], fx["table"][:u])
        if pair is None:
            raise ValueError("ConstraintSystemFailure: a lookup input is not in the table")
        for nm, vals in zip(("pa%d" % t, "ps%d" % t), pair):
            lagr[nm] = list(vals) + [0] * (n - u)
            blind_rows(lagr[nm], u)
    perm_names = [nm % t for t in range(n_lookups) for nm in ("pa%d", "ps%d")]
    commit([(1, lagr[nm]) for nm in perm_names])
    beta, gamma = tr.squeeze(), tr.squeeze()
    transforms(perm_names)
    col_of = lambda nm: fx[nm] if nm in consts else lagr[nm]
    start = 1
    for si in range(n_sets):
        z = [start]
        for i in range(u):
            num = den = 1
            for cidx in range(si * chunk, min(len(perm_cols), (si + 1) * chunk)):
                v = col_of(perm_cols[cidx])[i]
                num = num * (v + beta * pow(pyref.DELTA, cidx, R) % R * pow(w, i, R) + gamma) % R
                den = den * (v + beta * fx["sigma_" + perm_cols[cidx]][i] + gamma) % R
            z.append(z[-1] * num % R * pow(den, -1, R) % R)
        start = z[u]
        lagr["zp%d" % si] = z + [0] * (n - u - 1)
    for t in range(n_lookups):
        z = [1]
        pa, ps = lagr["pa%d" % t], lagr["ps%d" % t]
        for i in range(u):
            z.append(z[-1] * (lk_in[t][i] + beta) % R * (fx["table"][i] + gamma) % R * pow((pa[i] + beta) * (ps[i] + gamma) % R, -1, R) % R)
        lagr["zl%d" % t] = z + [0] * (n - u - 1)
    prod_names = ["zp%d" % si for si in range(n_sets)] + ["zl%d" % t for t in range(n_lookups)]
    for nm in prod_names:
        blind_rows(lagr[nm], u + 1)
    transforms(prod_names)
    rnd = [c % R for c in random_poly]
    commit([(1, lagr[nm]) for nm in prod_names] + [(0, rnd)])
    y = tr.squeeze()
    rot = lambda col, idx, r: pyref.rotate(col, idx, r, k, ext_k)
    values = []
    for idx in range(ne):
        v = 0
        for j in range(A):
            a = ext["a%d" % j]
            v = (v * y + selector_value(lay, "q%d" % j, lambda col: fx_ext[col][idx]) * (a[idx] + rot(a, idx, 1) * rot(a, idx, 2) - rot(a, idx, 3))) % R
        values.append(v)
    ext_of = lambda nm: fx_ext[nm] if nm in consts else ext[nm]
    values = pyref.permutation_terms([ext["zp%d" % si] for si in range(n_sets)], [ext_of(nm) for nm in perm_cols],
                                     [fx_ext["sigma_" + nm] for nm in perm_cols], chunk, fx_ext["l0"], fx_ext["l_last"], fx_ext["l_active"],
                                     beta, gamma, y, bf, k, ext_k, values)
    for t in range(n_lookups):
        inp_e = [q * a % R for q, a in zip(fx_ext[lay["selectors"]["q_lookup"][0]], ext["a0"])] if L == 0 else ext["l%d" % t]
        tv = [(i_ + beta) * (t_ + gamma) % R for i_, t_ in zip(inp_e, fx_ext["table"])]
        values = pyref.lookup_terms(tv, ext["zl%d" % t], ext["pa%d" % t], ext["ps%d" % t], fx_ext["l0"], fx_ext["l_last"], fx_ext["l_active"],
                                    beta, gamma, y, k, ext_k, values)
    we = pyref.omega_for(ext_k)
    for idx in range(ne):
        x_row = pyref.ZETA * pow(we, idx, R) % R
        values[idx] = values[idx] * pow(pow(x_row, n, R) - 1, -1, R) % R
    h = pyref.extended_to_coeff(values, k, ext_k)
    pieces = s["degree"] - 1
    assert not any(h[pieces * n:]), "the quotient has degree (degree - 1) n at most"
    commit([(0, h[j * n:(j + 1) * n]) for j in range(pieces)])
    x = tr.squeeze()
    coef.update({nm: fx_coef[nm] for nm in s["fixed"] + s["sigma"]})
    coef["rnd"] = rnd
    return dict(coef=coef, h=[h[j * n:(j + 1) * n] for j in range(pieces)], commitments=commitments,
                challenges=dict(theta=theta, beta=beta, gamma=gamma, y=y, x=x))


def create_proof(k: int, A: int, L: int, selector_lookup: bool, F: int, fixed: dict, sigma: list, virtual: list, break_points: list,
                 lookup_cells: list, random_poly: list, blind, bases_m: list, bases_l: list, instances=None, vk_repr: int = 0) -> bytes:
    """halo2_proof_oracle.create_proof on the compressed layout: `fixed` holds the uncompressed columns (q{j}, [q_lookup],
    [table], c..), compressed here as keygen_vk does"""
    instances = [[int(v) % R for v in col] for col in (instances or [])]
    cfixed, lay = compress(k, A, L, selector_lookup, F, fixed)
    s = shape(k, A, L, selector_lookup, F, len(instances), lay)
    n = s["n"]
    tr = hpo.Blake2bWrite()
    tr.common_scalar(vk_repr)
    ph = phases(s, lay, cfixed, sigma, virtual, break_points, lookup_cells, random_poly, blind, bases_m, bases_l, instances, tr)
    coef, x = ph["coef"], ph["challenges"]["x"]
    w = pyref.omega_for(k)
    point = lambda r: x * pow(w, r % n, R) % R
    for nm, r in hpo.evaluation_order(s):
        tr.write_scalar(pyref.eval_polynomial(coef[nm], point(r)))
    xn = pow(x, n, R)
    coef["h"] = [sum(pow(xn, j, R) * hp[c] for j, hp in enumerate(ph["h"])) % R for c in range(n)]
    sets = hpo.rotation_sets(hpo.opening_order(s))
    y, v = tr.squeeze(), tr.squeeze()
    qs, quotients = [], []
    for rots, names in sets:
        q = [sum(pow(y, j, R) * coef[nm][c] for j, nm in enumerate(names)) % R for c in range(n)]
        d = q
        for r in rots:  # successive divisions: the quotient by Z_{T_s}, remainder dropped
            d = pyref.kate_division(d, point(r))
        qs.append(q)
        quotients.append(d + [0] * (n - len(d)))
    hx = [0] * n
    for d in quotients:
        hx = [(a * v + b) % R for a, b in zip(hx, d)]
    tr.write_point(pyref.msm_naive(hx, bases_m))
    u = tr.squeeze()
    T = sorted({point(r) for rots, _ in sets for r in rots})
    S = len(sets)
    lin = [(-hpo.vanishing_at(T, u) * c) % R for c in hx]
    const = 0
    for si, ((rots, names), q) in enumerate(zip(sets, qs)):
        pts = [point(r) for r in rots]
        coef_s = pow(v, S - 1 - si, R) * hpo.vanishing_at([p for p in T if p not in pts], u) % R
        r_u = hpo.interpolate_at(pts, [pyref.eval_polynomial(q, p) for p in pts], u)
        lin = [(a + coef_s * b) % R for a, b in zip(lin, q)]
        const = (const + coef_s * r_u) % R
    lin[0] = (lin[0] - const) % R
    assert pyref.eval_polynomial(lin, u) == 0, "L(u) = 0"
    tr.write_point(pyref.msm_naive(pyref.kate_division(lin, u) + [0], bases_m))
    return tr.finalize()


def verify_proof(proof: bytes, k: int, A: int, L: int, selector_lookup: bool, F: int, lay: dict, vk: dict, instances, vk_repr: int, g0,
                 tau: int) -> bool:
    """halo2_proof_oracle.verify_proof on the compressed layout `lay` (compress()'s; vk["fixed"] by column name): every gate term
    is recomputed at x from the combination columns' evaluations through each selector's substituted expression"""
    instances = [[int(v) % R for v in col] for col in (instances or [])]
    s = shape(k, A, L, selector_lookup, F, len(instances), lay)
    n = s["n"]
    try:
        tr = hpo.Blake2bRead(proof)
        tr.common_scalar(vk_repr)
        for col in instances:
            for v in col:
                tr.common_scalar(v)
        cm = {nm: tr.read_point() for nm in s["adv"]}
        theta = tr.squeeze()  # noqa: F841  (the lookups here compress one expression each: theta does not enter the terms)
        for t in range(s["n_lookups"]):
            cm["pa%d" % t], cm["ps%d" % t] = tr.read_point(), tr.read_point()
        beta, gamma = tr.squeeze(), tr.squeeze()
        for nm in ["zp%d" % si for si in range(s["n_sets"])] + ["zl%d" % t for t in range(s["n_lookups"])] + ["rnd"]:
            cm[nm] = tr.read_point()
        y = tr.squeeze()
        h_pieces = [tr.read_point() for _ in range(s["degree"] - 1)]
        x = tr.squeeze()
        evals = {q: tr.read_scalar() for q in hpo.evaluation_order(s)}
        y_sh, v = tr.squeeze(), tr.squeeze()
        h1 = tr.read_point()
        u = tr.squeeze()
        h2 = tr.read_point()
        if tr.at != len(tr.proof):
            return False
    except ValueError:
        return False
    cm.update(vk["fixed"])
    cm.update(zip(s["sigma"], vk["permutation"]))
    # the vanishing argument: the expected h(x) from the terms, the h commitment from its pieces
    limbs = {q: np.frombuffer(fr_bytes(e), dtype=np.uint64) for q, e in evals.items()}
    limbs.update({("h%d" % j, 0): np.zeros(4, dtype=np.uint64) for j in range(s["degree"] - 1)})
    for sel in lay["selectors"]:  # the quotient identity reads q{j}(x), q_lookup(x): their substituted values
        limbs[(sel, 0)] = np.frombuffer(fr_bytes(selector_value(lay, sel, lambda col: evals[(col, 0)])), dtype=np.uint64)
    left, _ = co.quotient_identity({"evals": limbs, "challenges": dict(beta=beta, gamma=gamma, y=y, x=x)}, k, A, L, selector_lookup, F,
                                   instances)
    xn = pow(x, n, R)
    evals[("h", 0)] = left * pow(xn - 1, -1, R) % R
    cm["h"] = None
    for j, hp in enumerate(h_pieces):
        cm["h"] = pyref.g1_add(cm["h"], pyref.g1_mul(pow(xn, j, R), hp))
    # SHPLONK: F = sum_s v^(S-1-s) Z_{T\T_s}(u) (sum_j y^j C_sj - r_s(u) [1]) - Z_T(u) H
    w = pyref.omega_for(k)
    point = lambda r: x * pow(w, r % n, R) % R
    sets = hpo.rotation_sets(hpo.opening_order(s))
    T = sorted({point(r) for rots, _ in sets for r in rots})
    S = len(sets)
    scalars = {}
    const = 0
    for si, (rots, names) in enumerate(sets):
        pts = [point(r) for r in rots]
        coef_s = pow(v, S - 1 - si, R) * hpo.vanishing_at([p for p in T if p not in pts], u) % R
        for j, nm in enumerate(names):
            yj = pow(y_sh, j, R)
            scalars[nm] = (scalars.get(nm, 0) + coef_s * yj) % R
            const = (const + coef_s * yj % R * hpo.interpolate_at(pts, [evals[(nm, r)] for r in rots], u)) % R
    acc = pyref.g1_mul(-const % R, g0)
    for nm, sc in scalars.items():
        acc = pyref.g1_add(acc, pyref.g1_mul(sc, cm[nm]))
    acc = pyref.g1_add(acc, pyref.g1_mul(-hpo.vanishing_at(T, u) % R, h1))
    return acc == pyref.g1_mul((tau - u) % R, h2)

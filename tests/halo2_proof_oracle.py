"""halo2's proof bytes, restated on plain Python integers for tests/test_oracle_halo2_proof.py and tests/test_gpu_halo2_proof.py:
what ProverSession.gen_proof (include/h2b200_prover.hpp, create_proof_halo2) must write, and a verifier that checks them.

  Blake2bWrite / Blake2bRead  halo2's transcript (recalled from halo2-axiom 0.5.3, DESIGN §2): Blake2b-512 personalized
                              "Halo2-Transcript"; a point enters as 1 || x || y (canonical little-endian), a scalar as 2 || its
                              canonical bytes; a challenge absorbs 0 and is the digest of the state mod r; points are written
                              compressed (oracle/pyref.g1_compress), scalars as their 32 canonical bytes;
  phases                      constants_oracle.create_proof's flow (oracle/prover_ref -> instance_oracle -> constants_oracle) from
                              phase 0 up to the h pieces and x, through any transcript with common_scalar / write_point / squeeze;
  create_proof                vk.hash_into, the phases, halo2's evaluation order, h(X) = sum_i x^(n i) h_i, ProverSHPLONK with the
                              assertion L(u) = 0;
  verify_proof                reads the bytes back, recomputes every challenge, h(x) from the gate, permutation and lookup terms
                              (constants_oracle.quotient_identity), the h commitment and SHPLONK's F, and accepts iff
                              F = (tau - u) W' — the pairing equation e(F + u W', [1]_2) = e(W', [tau]_2) for params of a known tau."""
from __future__ import annotations
import hashlib
import numpy as np
import constants_oracle as co
from oracle import pyref
from oracle.prover_ref import fr_bytes

R, P = pyref.R, pyref.P
BLINDING_FACTORS = 6
PERSONAL = b"Halo2-Transcript"


class Blake2bWrite:
    def __init__(self):
        self.h = hashlib.blake2b(digest_size=64, person=PERSONAL)
        self.out = bytearray()

    def common_point(self, pt):
        if pt is None:
            raise ValueError("the identity cannot enter the transcript")
        self.h.update(b"\x01" + pt[0].to_bytes(32, "little") + pt[1].to_bytes(32, "little"))

    def common_scalar(self, v: int):
        self.h.update(b"\x02" + (v % R).to_bytes(32, "little"))

    def write_point(self, pt):
        self.common_point(pt)
        self.out += pyref.g1_compress(pt)

    def write_scalar(self, v: int):
        self.common_scalar(v)
        self.out += (v % R).to_bytes(32, "little")

    def squeeze(self) -> int:
        self.h.update(b"\x00")
        return int.from_bytes(self.h.digest(), "little") % R

    def finalize(self) -> bytes:
        return bytes(self.out)


class Blake2bRead(Blake2bWrite):
    def __init__(self, proof: bytes):
        super().__init__()
        self.proof, self.at = bytes(proof), 0

    def _take(self) -> bytes:
        if self.at + 32 > len(self.proof):
            raise ValueError("the proof ends early")
        b = self.proof[self.at:self.at + 32]
        self.at += 32
        return b

    def read_point(self):
        pt, ok = pyref.g1_decompress(self._take())
        if not ok:
            raise ValueError("not a point")
        self.common_point(pt)
        return pt

    def read_scalar(self) -> int:
        v = int.from_bytes(self._take(), "little")
        if v >= R:
            raise ValueError("not a canonical scalar")
        self.common_scalar(v)
        return v


def shape(k: int, A: int, L: int, selector_lookup: bool, F: int, I: int) -> dict:
    sel = selector_lookup and L == 0
    n_lookups = L if L else (1 if sel else 0)
    degree = 4 if L else (5 if sel else 3)
    consts = co.const_names(F)
    adv = ["a%d" % j for j in range(A)] + ["l%d" % t for t in range(L)]
    perm = consts + adv + ["i%d" % m for m in range(I)]
    chunk = degree - 2
    fixed = ["q%d" % j for j in range(A)] + (["q_lookup"] if sel else []) + (["table"] if n_lookups else []) + consts
    return dict(k=k, n=1 << k, A=A, L=L, sel=sel, F=F, I=I, n_lookups=n_lookups, degree=degree, chunk=chunk, consts=consts, adv=adv,
                perm=perm, n_sets=-(-len(perm) // chunk), fixed=fixed, sigma=["sigma_" + nm for nm in perm],
                ext_k=k + (1 if degree == 3 else 2), u=(1 << k) - (BLINDING_FACTORS + 1))


def phases(s: dict, fixed: dict, sigma: list, virtual: list, break_points: list, lookup_cells: list, random_poly: list, blind, bases_m: list,
           bases_l: list, instances: list, tr) -> dict:
    """constants_oracle.create_proof from phase 0 to the challenge x: the public values as common_scalars, every commitment
    through write_point.  Returns the coefficient forms of every column (coef, fx_coef), the h pieces, rnd and the challenges."""
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
        inp = [q * a % R for q, a in zip(fx["q_lookup"], lagr["a0"])] if L == 0 else lagr["l%d" % t]
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
            v = (v * y + fx_ext["q%d" % j][idx] * (a[idx] + rot(a, idx, 1) * rot(a, idx, 2) - rot(a, idx, 3))) % R
        values.append(v)
    ext_of = lambda nm: fx_ext[nm] if nm in consts else ext[nm]
    values = pyref.permutation_terms([ext["zp%d" % si] for si in range(n_sets)], [ext_of(nm) for nm in perm_cols],
                                     [fx_ext["sigma_" + nm] for nm in perm_cols], chunk, fx_ext["l0"], fx_ext["l_last"], fx_ext["l_active"],
                                     beta, gamma, y, bf, k, ext_k, values)
    for t in range(n_lookups):
        inp_e = [q * a % R for q, a in zip(fx_ext["q_lookup"], ext["a0"])] if L == 0 else ext["l%d" % t]
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


def evaluation_order(s: dict) -> list:
    """(column, rotation) of the written evaluations, in halo2's order"""
    last = -(BLINDING_FACTORS + 1)
    q = [("a%d" % j, r) for j in range(s["A"]) for r in (0, 1, 2, 3)] + [("l%d" % t, 0) for t in range(s["L"])]
    q += [(nm, 0) for nm in s["fixed"]] + [("rnd", 0)] + [(nm, 0) for nm in s["sigma"]]
    for si in range(s["n_sets"]):
        q += [("zp%d" % si, r) for r in ((0, 1, last) if si + 1 < s["n_sets"] else (0, 1))]
    for t in range(s["n_lookups"]):
        q += [("zl%d" % t, 0), ("zl%d" % t, 1), ("pa%d" % t, 0), ("pa%d" % t, -1), ("ps%d" % t, 0)]
    return q


def opening_order(s: dict) -> list:
    """(column, rotation) of the opening queries, in halo2's order; "h" is h(X) = sum_i x^(n i) h_i"""
    last = -(BLINDING_FACTORS + 1)
    q = [("a%d" % j, r) for j in range(s["A"]) for r in (0, 1, 2, 3)] + [("l%d" % t, 0) for t in range(s["L"])]
    q += [("zp%d" % si, r) for si in range(s["n_sets"]) for r in (0, 1)]
    q += [("zp%d" % si, last) for si in reversed(range(s["n_sets"] - 1))]
    for t in range(s["n_lookups"]):
        q += [("zl%d" % t, 0), ("pa%d" % t, 0), ("ps%d" % t, 0), ("pa%d" % t, -1), ("zl%d" % t, 1)]
    return q + [(nm, 0) for nm in s["fixed"] + s["sigma"]] + [("h", 0), ("rnd", 0)]


def rotation_sets(queries: list) -> list:
    """ProverSHPLONK's intermediate sets: commitments grouped by identity in first-appearance order, then by equal point sets.
    queries: (commitment id, rotation); returns [(sorted rotations, [commitment ids])]"""
    by_id = {}
    for cid, r in queries:
        rots = by_id.setdefault(cid, [])
        if r not in rots:
            rots.append(r)
    sets = {}
    for cid, rots in by_id.items():
        sets.setdefault(tuple(sorted(rots)), []).append(cid)
    return list(sets.items())


def vanishing_at(points, u: int) -> int:
    z = 1
    for p in points:
        z = z * (u - p) % R
    return z


def interpolate_at(points, values, u: int) -> int:
    """r(u) for the polynomial of degree < len(points) through (points[j], values[j])"""
    acc = 0
    for j, (zj, vj) in enumerate(zip(points, values)):
        num = den = 1
        for t, zt in enumerate(points):
            if t != j:
                num, den = num * (u - zt) % R, den * (zj - zt) % R
        acc = (acc + vj * num * pow(den, -1, R)) % R
    return acc


def create_proof(k: int, A: int, L: int, selector_lookup: bool, F: int, fixed: dict, sigma: list, virtual: list, break_points: list,
                 lookup_cells: list, random_poly: list, blind, bases_m: list, bases_l: list, instances=None, vk_repr: int = 0) -> bytes:
    """the bytes of create_proof_halo2 (arguments as constants_oracle.create_proof, canonical integers; vk_repr canonical)"""
    instances = [[int(v) % R for v in col] for col in (instances or [])]
    s = shape(k, A, L, selector_lookup, F, len(instances))
    n = s["n"]
    tr = Blake2bWrite()
    tr.common_scalar(vk_repr)
    ph = phases(s, fixed, sigma, virtual, break_points, lookup_cells, random_poly, blind, bases_m, bases_l, instances, tr)
    coef, x = ph["coef"], ph["challenges"]["x"]
    w = pyref.omega_for(k)
    point = lambda r: x * pow(w, r % n, R) % R
    for nm, r in evaluation_order(s):
        tr.write_scalar(pyref.eval_polynomial(coef[nm], point(r)))
    xn = pow(x, n, R)
    coef["h"] = [sum(pow(xn, j, R) * hp[c] for j, hp in enumerate(ph["h"])) % R for c in range(n)]
    sets = rotation_sets(opening_order(s))
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
    lin = [(-vanishing_at(T, u) * c) % R for c in hx]
    const = 0
    for si, ((rots, names), q) in enumerate(zip(sets, qs)):
        pts = [point(r) for r in rots]
        coef_s = pow(v, S - 1 - si, R) * vanishing_at([p for p in T if p not in pts], u) % R
        r_u = interpolate_at(pts, [pyref.eval_polynomial(q, p) for p in pts], u)
        lin = [(a + coef_s * b) % R for a, b in zip(lin, q)]
        const = (const + coef_s * r_u) % R
    lin[0] = (lin[0] - const) % R
    assert pyref.eval_polynomial(lin, u) == 0, "L(u) = 0"
    tr.write_point(pyref.msm_naive(pyref.kate_division(lin, u) + [0], bases_m))
    return tr.finalize()


def verify_proof(proof: bytes, k: int, A: int, L: int, selector_lookup: bool, F: int, vk: dict, instances, vk_repr: int, g0, tau: int) -> bool:
    """halo2's verify_proof for params of a known tau (g0 = [1]_1 = params.g[0]); vk = {"fixed": {name: point}, "permutation":
    [point per permutation column]} (affine, canonical); instances: the public values per instance column (canonical)"""
    instances = [[int(v) % R for v in col] for col in (instances or [])]
    s = shape(k, A, L, selector_lookup, F, len(instances))
    n = s["n"]
    try:
        tr = Blake2bRead(proof)
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
        evals = {q: tr.read_scalar() for q in evaluation_order(s)}
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
    sets = rotation_sets(opening_order(s))
    T = sorted({point(r) for rots, _ in sets for r in rots})
    S = len(sets)
    scalars = {}
    const = 0
    for si, (rots, names) in enumerate(sets):
        pts = [point(r) for r in rots]
        coef_s = pow(v, S - 1 - si, R) * vanishing_at([p for p in T if p not in pts], u) % R
        for j, nm in enumerate(names):
            yj = pow(y_sh, j, R)
            scalars[nm] = (scalars.get(nm, 0) + coef_s * yj) % R
            const = (const + coef_s * yj % R * interpolate_at(pts, [evals[(nm, r)] for r in rots], u)) % R
    acc = pyref.g1_mul(-const % R, g0)
    for nm, sc in scalars.items():
        acc = pyref.g1_add(acc, pyref.g1_mul(sc, cm[nm]))
    acc = pyref.g1_add(acc, pyref.g1_mul(-vanishing_at(T, u) % R, h1))
    return acc == pyref.g1_mul((tau - u) % R, h2)

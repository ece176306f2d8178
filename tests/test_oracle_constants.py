"""CPU tests of the constants-column oracles (tests/constants_oracle.py): with F constants columns, halo2's permutation Assembly on
halo2-base's copy calls agrees with the closed form and the C Assembly, its cycles are the classes of the copy graph with every
constant's cell in the class of the cells tied to it, F = 1 gives the existing oracles' results, the capacity panics come at
D = F u + 1 (and at the first constant when F = 0), and the oracle prover with F constants columns satisfies the quotient
identity and breaks it when a value or a sigma entry of column c1 is wrong."""
import random
import numpy as np
import pytest
from oracle import pyref, prover_ref
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
import builder_oracle as bo
import keygen_oracle as ko
import instance_oracle as io
import constants_oracle as co
import test_oracle_prover as top

R = pyref.R
SHAPES = [(1, 0, True), (3, 2, False), (2, 0, False), (2, 1, True)]
FS = [0, 1, 2, 3, 7]


def _cycles(mapping) -> np.ndarray:
    """the cycle id (its smallest cell) of every cell of a permutation"""
    out = np.full(len(mapping), -1, dtype=np.int64)
    for x in range(len(mapping)):
        if out[x] >= 0:
            continue
        cyc, y = [x], int(mapping[x])
        while y != x:
            cyc.append(y)
            y = int(mapping[y])
        out[cyc] = min(cyc)
    return out


def builder(rng, k, A, L, sel, bits, max_rows, F, contexts=2, fill=1.0):
    """builder_oracle.make_builder with more constant equalities: duplicates of existing ones and cells tied to a second
    constant; F = 0: no constants at all"""
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, fill=fill, contexts=contexts)
    if F == 0:
        return dict(b, constants=np.zeros(0, dtype=np.uint64), constant_index=np.zeros(0, dtype=np.uint64))
    N = len(b["selectors"])
    m = len(b["constants"])
    dup = rng.choice(m, size=min(m, 6), replace=False)
    cells = rng.choice(N, size=6, replace=False).astype(np.uint64)
    extra_c = np.concatenate([b["constants"][dup], rng.integers(2, 1 << 40, size=6, dtype=np.int64).astype(np.uint64)])
    extra_i = np.concatenate([b["constant_index"][dup], cells])
    return dict(b, constants=np.concatenate([b["constants"], extra_c]), constant_index=np.concatenate([b["constant_index"], extra_i]))


def _instances(rng, b, I, count):
    return [rng.choice(len(b["selectors"]), size=count).astype(np.uint64) for _ in range(I)]


@pytest.mark.parametrize("I", [0, 1])
@pytest.mark.parametrize("F", FS)
@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_assembly_closed_form_and_c_agree_with_constants_columns(A, L, sel, F, I):
    k = 7
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(70 + 10 * A + L + 3 * F + I)
    b = builder(rng, k, A, L, sel, 4, max_rows, F)
    inst = _instances(rng, b, I, 12)
    pairs, const_cells, bps = co.copy_sequence(k, A, L, max_rows, b, F, inst)
    n, V = 1 << k, (F + A + L + I) << k
    lit = ko.assembly(V, pairs)
    assert np.array_equal(lit, ko.closed_form(V, pairs))
    assert np.array_equal(lit, ko.assembly_c(V, pairs))
    g = coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(V, V))
    _, comp = connected_components(g, directed=False)
    cyc = _cycles(lit)
    assert len(set(zip(cyc.tolist(), comp.tolist()))) == len(set(cyc.tolist())) == len(set(comp.tolist()))
    # left to right, then top to bottom; every tied cell in its constant's cycle
    ranks = sorted(const_cells)
    assert [const_cells[c] for c in ranks] == [(d % F) * n + d // F for d in range(len(ranks))]
    for c, p in zip(b["constants"].tolist(), b["constant_index"].tolist()):
        j, row = bo.raw_cell(bps, p)
        assert cyc[const_cells[int(c)]] == cyc[(F + j) * n + row]


def test_one_constants_column_is_the_existing_sequence():
    k, A, L = 7, 2, 1
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(2)
    b = builder(rng, k, A, L, False, 4, max_rows, 1)
    got, want = co.copy_sequence(k, A, L, max_rows, b, 1), ko.copy_sequence(k, A, L, max_rows, b)
    assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
    inst = _instances(rng, b, 2, 9)
    got, want = co.copy_sequence(k, A, L, max_rows, b, 1, inst), io.copy_sequence(k, A, L, max_rows, b, inst)
    assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
    res = co.mock_run(k, A, L, False, 4, max_rows, b, b["values"], 1)
    base = bo.run(k, A, L, False, 4, max_rows, b, b["values"])
    assert {key: res[key] for key in base if key != "q"} == {key: v for key, v in base.items() if key != "q"}
    assert res["distinct_constants"] == len(set(b["constants"].tolist()))
    public = [[int(b["values"][int(p)]) for p in idx] for idx in inst]
    public[1][3] += 1
    res = co.mock_run(k, A, L, False, 4, max_rows, b, b["values"], 1, inst, public)
    base = io.mock_run(k, A, L, False, 4, max_rows, b, b["values"], inst, public)
    assert {key: res[key] for key in base if key != "q"} == {key: v for key, v in base.items() if key != "q"} and not res["satisfied"]


@pytest.mark.parametrize("F", [1, 2, 3, 7])
def test_capacity(F):
    """D = F u distinct constants fit, D = F u + 1 is halo2's NotEnoughRowsAvailable, in every oracle that places them"""
    k, A, L, sel, bits = 6, 1, 0, False, 2
    u, max_rows = (1 << k) - 7, (1 << k) - 9
    b = bo.make_builder(np.random.default_rng(5), k, A, L, sel, bits, max_rows)
    N = len(b["selectors"])
    for D, ok in ((F * u, True), (F * u + 1, False)):
        eqs = [(c + 10, c % N) for c in range(D)]
        bb = dict(b, constants=np.array([c for c, _ in eqs], dtype=np.uint64), constant_index=np.array([i for _, i in eqs], dtype=np.uint64))
        calls = (lambda: co.assign_constants(eqs, F, u, k), lambda: co.copy_sequence(k, A, L, max_rows, bb, F),
                 lambda: co.mock_run(k, A, L, sel, bits, max_rows, bb, b["values"], F))
        for call in calls:
            if ok:
                call()
            else:
                with pytest.raises(bo.Panic, match=r"NotEnoughRowsAvailable \{ current_k: 6 \}"):
                    call()
    # halo2-base sizes F by 2^k, not u: a builder with F u < D <= F 2^k is under-provisioned there too
    assert F * u + 1 <= F * (1 << k)
    placed = co.assign_constants([(c, 0) for c in range(F * u)], F, u, k)
    assert placed == {c: (c % F, c // F) for c in range(F * u)}
    # one column: builder_oracle's placement, rows 0, 1, ..
    if F == 1:
        assert {c: row for c, (_, row) in placed.items()} == bo.assign_constants([(c, 0) for c in range(u)], u, k)


def test_no_constants_column():
    k, A, L, sel, bits = 6, 1, 0, True, 3
    u, max_rows = (1 << k) - 7, (1 << k) - 9
    b = bo.make_builder(np.random.default_rng(6), k, A, L, sel, bits, max_rows)
    msg = "index out of bounds: the len is 0 but the index is 0"
    for call in (lambda: co.assign_constants([(5, 0)], 0, u, k), lambda: co.copy_sequence(k, A, L, max_rows, b, 0),
                 lambda: co.mock_run(k, A, L, sel, bits, max_rows, b, b["values"], 0)):
        with pytest.raises(bo.Panic, match=msg):
            call()
    none = dict(b, constants=np.zeros(0, dtype=np.uint64), constant_index=np.zeros(0, dtype=np.uint64))
    pairs, cells, _ = co.copy_sequence(k, A, L, max_rows, none, 0)
    assert cells == {} and pairs.max() < (A + L) << k
    res = co.mock_run(k, A, L, sel, bits, max_rows, none, b["values"], 0)
    assert res["satisfied"] and res["distinct_constants"] == 0


def test_mock_and_check_report_a_broken_constant_in_c1():
    """a cell tied to a constant of column c1 holds another value: MockProver reports the constant equality, the check two cells
    of its cycle"""
    k, A, L, sel, bits, F = 7, 2, 1, False, 4, 2
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(8)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
    pairs, cells, bps = co.copy_sequence(k, A, L, max_rows, b, F)
    n = 1 << k
    in_c1 = [i for i, c in enumerate(b["constants"].tolist()) if cells[int(c)] // n == 1]
    i = in_c1[0]
    values = b["values"].copy()
    values[int(b["constant_index"][i])] += 1
    res = co.mock_run(k, A, L, sel, bits, max_rows, b, values, F)
    assert not res["satisfied"] and i in res["constants"][1]
    cols = _advice_columns(k, A, L, bps, b, values)
    rep = co.check(k, F, co.const_columns(k, F, cells), _sigma(k, F + A + L, pairs), cols)
    assert co.check(k, F, co.const_columns(k, F, cells), _sigma(k, F + A + L, pairs), _advice_columns(k, A, L, bps, b, b["values"])) == \
        [(0, [])] * (F + A + L)
    # one wrong cell in the cycle of a constant of c1: the cell and the one whose sigma names it
    assert sum(c for c, _ in rep) == 2


def _sigma(k, npc, pairs):
    """sigma's canonical values, column by column, of the Assembly of `pairs`"""
    n, w = 1 << k, pyref.omega_for(k)
    mp = ko.assembly(npc << k, pairs)
    return [[pow(pyref.DELTA, int(x) >> k, R) * pow(w, int(x) & (n - 1), R) % R for x in mp[c * n:(c + 1) * n]] for c in range(npc)]


def _advice_columns(k, A, L, bps, b, values):
    """the A gate columns and the L lookup columns the keygen pass assigns, canonical"""
    n = 1 << k
    cols = [[0] * n for _ in range(A + L)]
    for j, (s, cnt) in enumerate(bo.spans(bps, len(values))):
        for r in range(cnt):
            cols[j][r] = int(values[s + r]) % R
    for i, p in enumerate(b["lookups"].tolist() if L else []):
        cols[A + i % L][i // L] = int(values[p]) % R
    return cols


# ------------------------------------------------------------------------------------------------ the oracle prover
def _keygen_instance(k, A, L, sel, bits, F, seed):
    """a satisfied keygen-form builder with its fixed columns and sigma from the oracles (canonical integers)"""
    n = 1 << k
    max_rows = n - 9
    rng = np.random.default_rng(seed)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, fill=0.6)
    if F == 0:
        b = dict(b, constants=np.zeros(0, dtype=np.uint64), constant_index=np.zeros(0, dtype=np.uint64))
    pairs, cells, bps = co.copy_sequence(k, A, L, max_rows, b, F)
    sigma = _sigma(k, F + A + L, pairs)
    run = co.mock_run(k, A, L, sel, bits, max_rows, b, b["values"], F)
    fixed = {"q%d" % j: [1 if r in run["q"][j] else 0 for r in range(n)] for j in range(A)}
    fixed["table"] = list(range(1 << bits)) + [0] * (n - (1 << bits))
    if sel and L == 0:
        fixed["q_lookup"] = [1 if r in run["q_lookup"] else 0 for r in range(n)]
    for nm, col in zip(co.const_names(F), co.const_columns(k, F, cells)):
        fixed[nm] = col
    lookup = [int(b["values"][p]) for p in b["lookups"].tolist()] if L else []
    return dict(fixed=fixed, sigma=sigma, virtual=[int(v) for v in b["values"]], break_points=bps, lookup=lookup, cells=cells)


def _prove(k, A, L, sel, F, seed, inst, prover=None):
    rng = random.Random(seed + 1)
    n = 1 << k
    blind = lambda rows: [rng.randrange(R) for _ in range(rows)]
    args = (k, A, L, sel, inst["fixed"], inst["sigma"], inst["virtual"], inst["break_points"], inst["lookup"],
            [rng.randrange(R) for _ in range(n)], blind, top.small_bases(n, 3, 5), top.small_bases(n, 7, 11))
    res = prover(*args) if prover else co.create_proof(*args[:4], F, *args[4:])
    as_limbs = lambda v: np.frombuffer(prover_ref.fr_bytes(v), dtype=np.uint64)
    return {"evals": {(nm, r): as_limbs(v) for nm, r, v in res["evals"]}, "challenges": res["challenges"], "commitments": res["commitments"]}


def _identity_fails(k, A, L, sel, F, seed, inst):
    try:
        bad = _prove(k, A, L, sel, F, seed, inst)
    except AssertionError:  # not divisible by X^n - 1
        return True
    left, right = co.quotient_identity(bad, k, A, L, sel, F)
    return left != right


def test_oracle_prover_with_one_constants_column_is_the_existing_one():
    k, A, L, sel, seed = 5, 2, 1, True, 31
    inst = top.int_instance(k, A, L, sel, seed)
    got, want = _prove(k, A, L, sel, 1, seed, inst), _prove(k, A, L, sel, 1, seed, inst, io.create_proof)
    assert got["commitments"] == want["commitments"] and got["challenges"] == want["challenges"]
    assert list(got["evals"]) == list(want["evals"]) and all(np.array_equal(got["evals"][q], want["evals"][q]) for q in want["evals"])
    assert co.quotient_identity(got, k, A, L, sel, 1) == io.quotient_identity(got, k, A, L, sel, [])


@pytest.mark.parametrize("F", [0, 2, 3])
@pytest.mark.parametrize("A,L,sel", [(1, 0, True), (2, 1, False)])
def test_oracle_prover_with_constants_columns(A, L, sel, F):
    """the quotient identity holds with F constants columns; a value or a sigma entry of c1 changed breaks it"""
    k, bits, seed = 6, 3, 900 + 10 * A + F
    inst = _keygen_instance(k, A, L, sel, bits, F, seed)
    res = _prove(k, A, L, sel, F, seed, inst)
    assert [nm for nm, r in res["evals"] if nm.startswith("sigma_")] == ["sigma_" + c for c in co.const_names(F)] + \
        ["sigma_a%d" % j for j in range(A)] + ["sigma_l%d" % t for t in range(L)]
    left, right = co.quotient_identity(res, k, A, L, sel, F)
    assert left == right
    if F < 2:
        return
    n = 1 << k
    row = next(cell % n for cell in inst["cells"].values() if cell // n == 1)
    c1 = list(inst["fixed"]["c1"])
    c1[row] = (c1[row] + 1) % R
    assert _identity_fails(k, A, L, sel, F, seed, dict(inst, fixed=dict(inst["fixed"], c1=c1)))
    sig = [list(s) for s in inst["sigma"]]
    sig[1][row], sig[1][row + 1] = sig[1][row + 1], sig[1][row]
    assert _identity_fails(k, A, L, sel, F, seed, dict(inst, sigma=sig))

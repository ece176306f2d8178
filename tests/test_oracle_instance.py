"""CPU tests of the instance-column oracles (tests/instance_oracle.py): halo2's permutation Assembly on halo2-base's copy calls
with assign_instances' copies appended agrees with the closed form and the C Assembly, its cycles are the classes of the copy
graph with every instance cell in the class of the advice cell it copies, the panics come at the first failing instance cell,
and calls without instance columns give the existing oracles' results.  The oracle prover with public inputs
(instance_oracle.create_proof) gives oracle/prover_ref's bytes without them, satisfies the extended quotient identity with them,
and breaks it when a public value or an instance column's sigma entry is wrong."""
import json
import os
import random
import numpy as np
import pytest
from oracle import pyref, prover_ref
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
import builder_oracle as bo
import keygen_oracle as ko
import instance_oracle as io
import prover_check as pc
import test_oracle_prover as top

R = pyref.R

SHAPES = [(1, 0, True), (3, 2, False), (2, 0, False), (2, 1, True)]


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


def _instances(rng, b, I, count):
    N = len(b["selectors"])
    return [rng.choice(N, size=count, replace=True).astype(np.uint64) for _ in range(I)]


@pytest.mark.parametrize("I", [1, 2])
@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_assembly_closed_form_and_c_agree_with_instance_copies(A, L, sel, I):
    k = 7
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(40 + 10 * A + L + I)
    b = bo.make_builder(rng, k, A, L, sel, 4, max_rows, contexts=2)
    inst = _instances(rng, b, I, 16)
    pairs, _, bps = io.copy_sequence(k, A, L, max_rows, b, inst)
    n, V = 1 << k, (1 + A + L + I) << k
    lit = ko.assembly(V, pairs)
    assert np.array_equal(lit, ko.closed_form(V, pairs))
    assert np.array_equal(lit, ko.assembly_c(V, pairs))
    g = coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(V, V))
    _, comp = connected_components(g, directed=False)
    cyc = _cycles(lit)
    # one cycle per class: the partitions agree
    assert len(set(zip(cyc.tolist(), comp.tolist()))) == len(set(cyc.tolist())) == len(set(comp.tolist()))
    for m, idx in enumerate(inst):
        for r, p in enumerate(idx.tolist()):
            j, row = bo.raw_cell(bps, p)
            assert cyc[(1 + A + L + m) * n + r] == cyc[(1 + j) * n + row]


def test_copy_sequence_without_instances_is_the_existing_one():
    k, A, L = 7, 2, 1
    max_rows = (1 << k) - 9
    b = bo.make_builder(np.random.default_rng(2), k, A, L, False, 4, max_rows)
    got, want = io.copy_sequence(k, A, L, max_rows, b), ko.copy_sequence(k, A, L, max_rows, b)
    assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
    # an instance column with no cells adds no copy
    assert np.array_equal(io.copy_sequence(k, A, L, max_rows, b, [np.zeros(0, dtype=np.uint64)])[0], want[0])


def test_instance_panics_at_the_first_failing_cell():
    k, A, L = 7, 2, 0
    max_rows = (1 << k) - 9
    b = bo.make_builder(np.random.default_rng(3), k, A, L, False, 4, max_rows)
    N, u = len(b["selectors"]), (1 << k) - 7
    with pytest.raises(bo.Panic, match="instance not assigned"):
        io.copy_sequence(k, A, L, max_rows, b, [np.array([0, N], dtype=np.uint64)])
    with pytest.raises(bo.Panic, match=r"NotEnoughRowsAvailable \{ current_k: 7 \}"):
        io.copy_sequence(k, A, L, max_rows, b, [np.zeros(u + 1, dtype=np.uint64)])
    bad = np.zeros(u + 1, dtype=np.uint64)
    bad[u] = N  # at row u, halo2-base's lookup of the cell comes before the copy
    with pytest.raises(bo.Panic, match="instance not assigned"):
        io.copy_sequence(k, A, L, max_rows, b, [bad])
    with pytest.raises(bo.Panic, match="NotEnoughRowsAvailable"):
        io.copy_sequence(k, A, L, max_rows, b, [np.zeros(u + 1, dtype=np.uint64), np.array([N], dtype=np.uint64)])


def test_mock_instance_check():
    k, A, L, sel, bits = 7, 2, 1, False, 4
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(4)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
    inst = _instances(rng, b, 2, 10)
    public = [[int(b["values"][int(p)]) for p in idx] for idx in inst]
    res = io.mock_run(k, A, L, sel, bits, max_rows, b, b["values"], inst, public)
    assert res["satisfied"] and res["instances"] == [(0, []), (0, [])]
    base = bo.run(k, A, L, sel, bits, max_rows, b, b["values"])
    assert {key: res[key] for key in base if key != "q"} == {key: v for key, v in base.items() if key != "q"}
    public[1][3] += 1
    res = io.mock_run(k, A, L, sel, bits, max_rows, b, b["values"], inst, public)
    assert not res["satisfied"] and res["instances"] == [(0, []), (1, [3])]
    assert res["instance_cells"][1] == [bo.raw_cell(res["break_points"], int(inst[1][3]))]
    with pytest.raises(bo.Panic, match="InstanceTooLarge"):
        io.mock_run(k, A, L, sel, bits, max_rows, b, b["values"], [np.zeros(122, dtype=np.uint64)], [[0] * 122])
    with pytest.raises(bo.Panic, match="instance not assigned"):
        io.mock_run(k, A, L, sel, bits, max_rows, b, b["values"], [[len(b["values"])]], [[0]])


# ------------------------------------------------------------------------------------------------ the oracle prover with public inputs
def _with_public(k, A, L, sel, seed, I, count):
    """test_oracle_prover.int_instance plus I instance columns of `count` cells each: every instance row is tied (a 2-cycle) to
    the first cell of a distinct gate (row 4i, in no other cycle), and its public value is that cell's"""
    inst = top.int_instance(k, A, L, sel, seed)
    n = 1 << k
    G = (n - 20) // 4 if A == 1 else (n - 24) // 4
    w = pyref.omega_for(k)
    ident = lambda c, r: pow(pyref.DELTA, c, R) * pow(w, r, R) % R
    sig = [list(c) for c in inst["sigma"]] + [[ident(1 + A + L + m, r) for r in range(n)] for m in range(I)]
    cells = random.Random(seed + 7).sample([(j, 4 * i) for j in range(A) for i in range(G)], I * count)
    public = []
    for m in range(I):
        col = []
        for r, (j, row) in enumerate(cells[m * count:(m + 1) * count]):
            sig[1 + j][row], sig[1 + A + L + m][r] = ident(1 + A + L + m, r), ident(1 + j, row)
            col.append(inst["virtual"][j * 4 * G + row])
        public.append(col)
    return dict(inst, sigma=sig), public


def _prove(k, A, L, sel, seed, inst, public, prover=None):
    """test_oracle_prover.run's inputs (random polynomial, blinding rows, bases) through instance_oracle.create_proof"""
    rng = random.Random(seed + 1)
    n = 1 << k
    blind = lambda rows: [rng.randrange(R) for _ in range(rows)]
    args = (k, A, L, sel, inst["fixed"], inst["sigma"], inst["virtual"], inst["break_points"], inst["lookup"],
            [rng.randrange(R) for _ in range(n)], blind, _bases(n, 3, 5), _bases(n, 7, 11))
    res = (prover or io.create_proof)(*args, **({} if prover else {"instances": public}))
    as_limbs = lambda v: np.frombuffer(prover_ref.fr_bytes(v), dtype=np.uint64)
    return {"evals": {(nm, r): as_limbs(v) for nm, r, v in res["evals"]}, "challenges": res["challenges"], "commitments": res["commitments"]}


_bases_memo = {}


def _bases(n, a0, d):
    if (n, a0, d) not in _bases_memo:
        _bases_memo[(n, a0, d)] = top.small_bases(n, a0, d)
    return _bases_memo[(n, a0, d)]


def _identity_or_divisibility_fails(k, A, L, sel, seed, inst, public):
    """a broken instance: the folded terms are not divisible by X^n - 1, so either create_proof's degree assertion fires or the
    identity fails at x (as test_oracle_prover's broken gate)"""
    try:
        bad = _prove(k, A, L, sel, seed, inst, public)
    except AssertionError:
        return True
    left, right = io.quotient_identity(bad, k, A, L, sel, public)
    return left != right


def test_oracle_prover_without_instances_is_prover_ref():
    """no instance columns: the same commitments, evaluations and challenges as oracle/prover_ref (and so the golden proof's
    inputs give the golden proof); the extended identity is prover_check's"""
    from golden import make_golden_prover as g
    for k, A, L, sel, seed in ((g.K, g.A, g.L, g.SEL, g.SEED), (5, 2, 1, True, 31)):
        inst = top.int_instance(k, A, L, sel, seed)
        got, want = _prove(k, A, L, sel, seed, inst, None), _prove(k, A, L, sel, seed, inst, None, prover_ref.create_proof)
        assert got["commitments"] == want["commitments"] and got["challenges"] == want["challenges"]
        assert all(np.array_equal(got["evals"][q], want["evals"][q]) for q in want["evals"]) and list(got["evals"]) == list(want["evals"])
        assert io.quotient_identity(got, k, A, L, sel, []) == pc.quotient_identity(got, k, prover_ref.BLINDING_FACTORS, A, L, sel)
    assert g.proof() == json.loads(json.dumps(json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prover_k5.json")))))


@pytest.mark.parametrize("I", [1, 2])
@pytest.mark.parametrize("A,L,sel", [(1, 0, True), (1, 0, False), (2, 1, True), (3, 2, True)])
def test_oracle_prover_with_public_inputs(A, L, sel, I):
    """the extended quotient identity holds; one public value replaced, or one sigma entry of an instance column, breaks it"""
    k, seed = 6, 500 + 10 * A + L + I
    inst, public = _with_public(k, A, L, sel, seed, I, 3)
    res = _prove(k, A, L, sel, seed, inst, public)
    left, right = io.quotient_identity(res, k, A, L, sel, public)
    assert left == right
    assert res["challenges"]["theta"] == io.theta([np.stack([np.frombuffer(prover_ref.fr_bytes(v), dtype=np.uint64) for v in col])
                                                   for col in public], [np.frombuffer(c, dtype=np.uint64) for c in res["commitments"][:A + L]])
    wrong = [list(col) for col in public]
    wrong[-1][1] = (wrong[-1][1] + 1) % R
    assert _identity_or_divisibility_fails(k, A, L, sel, seed, inst, wrong)
    sig = [list(c) for c in inst["sigma"]]
    c = 1 + A + L + I - 1
    sig[c][0], sig[c][1] = sig[c][1], sig[c][0]  # two instance rows swap their sigma images
    assert _identity_or_divisibility_fails(k, A, L, sel, seed, dict(inst, sigma=sig), public)
    with pytest.raises(ValueError, match="InstanceTooLarge"):
        _prove(k, A, L, sel, seed, inst, [[0] * ((1 << k) - 6)] + public[1:])

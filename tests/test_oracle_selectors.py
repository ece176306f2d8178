"""CPU: halo2's selector compression on plain Python integers (tests/selectors_oracle.py) — hand-worked combinations, halo2's
own property on random activations (each substituted expression is non-zero exactly on its selector's rows, no gate exceeds
max_degree), oracle proofs in the compressed layout that the oracle verifier accepts, rejections of a changed combination-column
evaluation and of the uncompressed fixed order, and the committed golden proof."""
import json
import os
import random
import pytest
from oracle import pyref
import selectors_oracle as so
import test_oracle_halo2_proof as toh

R = pyref.R
HERE = os.path.dirname(os.path.abspath(__file__))
NO = [[False] * 8 for _ in range(8)]


def test_hand_worked_combinations():
    # three mutually exclusive degree-3 selectors: pairs at max_degree 4, all three at 5 (roots by join order)
    assert so.process([3, 3, 3], 4, NO) == [[0, 1], [2]]
    assert so.process([3, 3, 3], 5, NO) == [[0, 1, 2]]
    assert so.process([3, 3, 3], 3, NO) == [[0], [1], [2]]
    # a complex (degree-0) selector is placed first, alone
    assert so.process([3, 0, 3], 4, NO) == [[1], [0, 2]]
    # a selector active beside another stays alone
    c = [[False, True, False], [True, False, False], [False, False, False]]
    assert so.process([3, 3, 3], 4, c) == [[0, 2], [1]]
    # an all-zero selector conflicts with nothing and joins the first combination
    cols = [[1, 0, 1, 0], [1, 1, 0, 0], [0, 0, 0, 0]]
    assert so.process([3, 3, 3], 4, so.conflicts_of(cols)) == [[0, 2], [1]]
    # a degree-2 selector leaves room for a third member at max_degree 4: d stays 1, 1 + 3 = 4
    assert so.process([2, 2, 2], 4, NO) == [[0, 1, 2]]


@pytest.mark.parametrize("seed", range(6))
def test_substitution_is_nonzero_exactly_on_active_rows(seed):
    """halo2's property: with the combination columns, every selector's substituted expression is non-zero exactly on its own
    active rows, and no gate's degree (its combination length + deg - 1) exceeds max_degree"""
    rng = random.Random(seed)
    S, n = rng.randrange(2, 9), 24
    max_degree = rng.choice([3, 4, 5, 6])
    degrees = [rng.choice([0, 2, 3, min(4, max_degree)]) for _ in range(S)]
    cols = [[1 if rng.random() < 0.15 else 0 for _ in range(n)] for _ in range(S)]
    combos = so.process(degrees, max_degree, so.conflicts_of(cols))
    assert sorted(i for c in combos for i in c) == list(range(S))
    for comb in combos:
        col = [0] * n
        for m, si in enumerate(comb):
            for r in range(n):
                if cols[si][r]:
                    assert col[r] == 0, "members of a combination share a row"
                    col[r] = m + 1
        for m, si in enumerate(comb):
            assert [so.substitute(v, m + 1, len(comb)) != 0 for v in col] == [bool(v) for v in cols[si]]
            if degrees[si]:
                assert degrees[si] - 1 + len(comb) <= max_degree
            else:
                assert len(comb) == 1


def _prove(k, A, L, sel, F, inst, seed, vk_repr):
    rng = random.Random(seed)
    g, gl = toh.params(k)
    return so.create_proof(k, A, L, sel, F, inst["fixed"], inst["sigma"], inst["virtual"], inst["break_points"], inst["lookup"],
                           [rng.randrange(R) for _ in range(1 << k)], lambda rows: [rng.randrange(R) for _ in range(rows)], g, gl,
                           inst["public"], vk_repr)


def _vk(k, A, L, sel, F, inst):
    cfixed, lay = so.compress(k, A, L, sel, F, inst["fixed"])
    _, gl = toh.params(k)
    return lay, {"fixed": {nm: pyref.msm_naive(cfixed[nm], gl) for nm in lay["columns"]},
                 "permutation": [pyref.msm_naive(col, gl) for col in inst["sigma"]]}


def _verify(proof, k, A, L, sel, F, inst, lay, vk, vk_repr):
    g, _ = toh.params(k)
    return so.verify_proof(proof, k, A, L, sel, F, lay, vk, inst["public"], vk_repr, g[0], toh.TAU)


@pytest.mark.parametrize("F,I", [(1, 0), (0, 1), (2, 1)])
@pytest.mark.parametrize("A,L,sel", toh.SHAPE_KINDS)
def test_oracle_proofs_verify(A, L, sel, F, I):
    k = 5
    seed = 300 + 10 * A + L + 3 * F + I + k  # the builders of test_oracle_halo2_proof.test_oracle_proofs_verify
    inst = toh.instance(k, A, L, sel, 3, F, I, seed)
    lay, vk = _vk(k, A, L, sel, F, inst)
    if sel:  # convention 12 for the ECDSA shape kind: q_lookup alone first, then q0, reordered only
        assert lay["combinations"] == [["q_lookup"], ["q0"]]
    if not L and not sel:  # degree 3: nothing combines
        assert all(len(c) == 1 for c in lay["combinations"])
    proof = _prove(k, A, L, sel, F, inst, seed, 777)
    assert _verify(proof, k, A, L, sel, F, inst, lay, vk, 777)


def test_rejections():
    from golden import make_golden_compressed_proof as g
    inst, _, _ = g.inputs()
    k, A, L, sel, F = g.K, g.A, g.L, g.SEL, g.F
    lay, vk = _vk(k, A, L, sel, F, inst)
    assert any(len(c) == 2 for c in lay["combinations"])
    proof = _prove(k, A, L, sel, F, inst, 88, 5)
    assert _verify(proof, k, A, L, sel, F, inst, lay, vk, 5)
    s = so.shape(k, A, L, sel, F, 1, lay)
    n_pts = len(s["adv"]) + 2 * s["n_lookups"] + s["n_sets"] + s["n_lookups"] + 1 + s["degree"] - 1
    order = so.hpo.evaluation_order(s)
    bad = bytearray(proof)
    bad[32 * (n_pts + order.index(("s0", 0)))] ^= 1  # the combination column's evaluation
    assert not _verify(bytes(bad), k, A, L, sel, F, inst, lay, vk, 5)
    legacy = dict(lay, queries=list(lay["columns"]))  # the evaluations read in column order instead of query order
    assert legacy["queries"] != lay["queries"]
    assert not _verify(proof, k, A, L, sel, F, inst, legacy, vk, 5)


def test_oracle_reproduces_the_committed_golden_proof():
    """tests/golden/halo2_proof_compressed_k5.json (tests/golden/make_golden_compressed_proof.py): the frozen bytes, which the
    oracle verifier accepts; one pair of selectors shares a column"""
    from golden import make_golden_compressed_proof as g
    want = json.load(open(os.path.join(HERE, "golden", "halo2_proof_compressed_k5.json")))
    assert g.proof() == want
    assert want["combinations"] == [["q0", "q1"], ["q2"]]
    inst, _, _ = g.inputs()
    lay, vk = _vk(g.K, g.A, g.L, g.SEL, g.F, inst)
    assert _verify(bytes.fromhex(want["proof"]), g.K, g.A, g.L, g.SEL, g.F, inst, lay, vk, g.VK_REPR)

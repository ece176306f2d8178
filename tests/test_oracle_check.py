"""CPU: the MockProver restatement of tests/mock_oracle.py on integer instances (tests/test_oracle_prover.py::int_instance):
a satisfied instance reports nothing, and every hand-placed violation reports exactly the cells it breaks."""
import random
import pytest
from oracle import pyref
from test_oracle_prover import int_instance
import mock_oracle as mo

R = pyref.R
K = 6
# (A, L, selector lookup): the selector lookup; lookup-advice columns; no lookup (three one-column permutation sets);
# lookup-advice columns with two chained permutation sets
SHAPES = [(1, 0, True), (3, 2, False), (2, 0, False), (2, 1, True)]


def _setup(A, L, sel, seed=4100):
    inst = int_instance(K, A, L, sel, seed + 10 * A + L)
    cols = mo.assign(K, A, L, inst["virtual"], inst["break_points"], inst["lookup"])
    return inst, cols


def _verify(inst, cols, A, L, sel, max_report=16):
    return mo.verify(K, A, L, sel, inst["fixed"], inst["sigma"], cols, max_report)


def _expect(A, L, sel, gates=None, lookups=None, copies=None):
    """the report dict with the named failing rows (sets) and zero elsewhere"""
    n_lk = L if L else (1 if sel else 0)
    rep = lambda d, i: (len(d.get(i, ())), sorted(d.get(i, ())))
    g, lk, cp = gates or {}, lookups or {}, copies or {}
    out = {"gates": [rep(g, j) for j in range(A)], "lookups": [rep(lk, t) for t in range(n_lk)], "copies": [rep(cp, c) for c in range(1 + A + L)]}
    out["satisfied"] = not (g or lk or cp)
    return out


def _pred(inst, c, r):
    """the cell whose sigma entry names (c, r)"""
    target = pow(pyref.DELTA, c, R) * pow(pyref.omega_for(K), r, R) % R
    hits = [(c2, r2) for c2, col in enumerate(inst["sigma"]) for r2, v in enumerate(col) if v == target]
    assert len(hits) == 1
    return hits[0]


def _add(d, c, r):
    d.setdefault(c, set()).add(r)


@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_satisfied_instance_reports_nothing(A, L, sel):
    inst, cols = _setup(A, L, sel)
    assert _verify(inst, cols, A, L, sel) == _expect(A, L, sel)


@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_gate_output_cell(A, L, sel):
    inst, cols = _setup(A, L, sel)
    j = A - 1
    cols[j][4 * 2 + 3] = (cols[j][4 * 2 + 3] + 1) % R  # gate 2 of the last gate column: its output cell, tied to nothing
    assert _verify(inst, cols, A, L, sel) == _expect(A, L, sel, gates={j: {8}})


@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_bit_cell_breaks_its_gate_and_both_copies(A, L, sel):
    inst, cols = _setup(A, L, sel)
    i = next(i for i in range(1, 10) if cols[0][4 * i + 1])  # a gate whose b operand is not 0, so the bit matters
    r = 4 * i + 2
    cols[0][r] = 1 - cols[0][r]  # the other bit: the gate breaks, and so do the copy into and out of this cell
    cp = {}
    _add(cp, 1, r)
    _add(cp, *_pred(inst, 1, r))
    assert _verify(inst, cols, A, L, sel) == _expect(A, L, sel, gates={0: {4 * i}}, copies=cp)


@pytest.mark.parametrize("A,L,sel", [s for s in SHAPES if s[1] or s[2]])
def test_looked_up_cell_outside_the_table(A, L, sel):
    inst, cols = _setup(A, L, sel)
    i = 3
    big = 1 << 40
    cols[0][4 * i + 1] = big                                               # the b operand of gate i ...
    cols[0][4 * i + 3] = (cols[0][4 * i] + big * cols[0][4 * i + 2]) % R    # ... with the gate still satisfied
    if L:  # lookup cell i is the copy of this cell (synthetic layout: column i mod L, row i div L): the copy still holds
        cols[A + i % L][i // L] = big
        lk = {i % L: {i // L}}
    else:
        lk = {0: {4 * i + 1}}
    assert _verify(inst, cols, A, L, sel) == _expect(A, L, sel, lookups=lk)


@pytest.mark.parametrize("A,L,sel", [s for s in SHAPES if s[1]])
def test_lookup_advice_copy(A, L, sel):
    inst, cols = _setup(A, L, sel)
    t, r = 1 % L, 2
    i = r * L + t                                # lookup cell i, the copy of gate column 0's cell 4 i + 1
    bits = min(8, K - 2)
    cols[A + t][r] = (cols[A + t][r] + 1) % (1 << bits)  # still in the table: only the 2-cycle with its source breaks
    cp = {}
    _add(cp, 1 + A + t, r)
    _add(cp, 1, 4 * i + 1)
    assert _pred(inst, 1 + A + t, r) == (1, 4 * i + 1)
    assert _verify(inst, cols, A, L, sel) == _expect(A, L, sel, copies=cp)


@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_fixed_constant_cell(A, L, sel):
    inst, cols = _setup(A, L, sel)
    inst["fixed"]["c"][1] = 2  # the constant 1 that every bit-1 cell is tied to
    cp = {}
    _add(cp, 0, 1)
    _add(cp, *_pred(inst, 0, 1))
    assert _verify(inst, cols, A, L, sel) == _expect(A, L, sel, copies=cp)


@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_malformed_sigma_entry(A, L, sel):
    inst, cols = _setup(A, L, sel)
    c, r = A + L, 5  # the last permutation column
    inst["sigma"][c][r] = random.Random(7).randrange(R)
    with pytest.raises(ValueError):
        _verify(inst, cols, A, L, sel)
    want = [(0, [])] * (1 + A + L)
    want[c] = (1, [r])
    assert mo.malformed_sigma(K, inst["sigma"]) == want


def test_report_holds_the_smallest_rows_and_the_exact_count():
    A, L, sel = 1, 0, True
    inst, cols = _setup(A, L, sel)
    for i in range(6):
        cols[0][4 * i + 3] = (cols[0][4 * i + 3] + 1) % R
    rep = _verify(inst, cols, A, L, sel, max_report=4)
    assert rep["gates"] == [(6, [0, 4, 8, 12])] and not rep["satisfied"]


def test_rows_past_the_usable_ones_read_as_zero():
    """a gate at row u - 1 reads rows >= u through its rotations: they count as 0, whatever the column holds there"""
    A, L, sel = 1, 0, False
    inst, cols = _setup(A, L, sel)
    n, u = 1 << K, (1 << K) - 7
    q = inst["fixed"]["q0"]
    q[u - 1] = 1
    cols[0][u - 1] = 5
    for r in range(u, n):
        cols[0][r] = 12345  # junk above u: must not matter
    # 5 + 0 * 0 - 0 != 0 -> fails; with a(u - 1) = 0 it holds
    assert _verify(inst, cols, A, L, sel)["gates"] == [(1, [u - 1])]
    cols[0][u - 1] = 0
    assert _verify(inst, cols, A, L, sel)["gates"] == [(0, [])]

"""CPU tests of tests/builder_oracle.py, the yardstick of the device MockProver: hand-written walks (a gate that would cross
max_rows, the forced break at max_rows - 1, empty contexts), every panic of the keygen pass, and hand-placed violations
found at the expected equality indices, rows and raw cells."""
import numpy as np
import pytest
from oracle import pyref
import builder_oracle as bo


def _walk(contexts, A, max_rows):
    return bo.assign_with_constraints([np.asarray(c, dtype=np.uint8) for c in contexts], A, max_rows)


def test_gate_that_would_cross_max_rows_breaks_before_it():
    # max_rows 10: the gate at row 7 would read rows 7..10; the break cell keeps its value in column 0 and its selector moves
    sel = [1, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0]
    bps, raw, q = _walk([sel], 2, 10)
    assert bps == [7]
    assert q == [{0, 3}, {0}]
    assert raw[7] == (0, 7) and raw[8] == (1, 1) and raw[11] == (1, 4)
    assert bps == pyref.break_points_for([sel], 10)
    assert bo.raw_cell(bps, 7) == (0, 7) and bo.raw_cell(bps, 8) == (1, 1)


def test_forced_break_at_max_rows_minus_one():
    bps, raw, q = _walk([[0] * 25], 3, 10)
    assert bps == [9, 9]  # rows 0..9 of column 0, then the copy at row 0 and 8 new cells per column
    assert raw[9] == (0, 9) and raw[10] == (1, 1) and raw[18] == (1, 9) and raw[19] == (2, 1)
    assert bo.spans(bps, 25) == [(0, 10), (9, 10), (18, 7)]


def test_a_selector_two_rows_before_max_rows_breaks_there():
    bps, _, q = _walk([[0] * 8 + [1, 0, 0, 0]], 2, 10)  # row 8 >= max_rows - 3 with the selector set
    assert bps == [8] and q == [set(), {0}]


def test_empty_contexts_change_nothing():
    a = _walk([[], [1, 0, 0, 1, 0, 0, 0], [], [0, 1, 0]], 1, 20)
    b = _walk([[1, 0, 0, 1, 0, 0, 0, 0, 1, 0]], 1, 20)
    assert a == b == ([], a[1], [{0, 3, 8}])


def test_spans_and_raw_cells_agree_with_the_literal_walk():
    rng = np.random.default_rng(5)
    for A, max_rows in ((3, 40), (5, 23), (2, 101)):
        b = bo.make_builder(rng, 9, A, 0, False, 4, max_rows, contexts=3)
        bps, raw, q = bo.assign_with_constraints(b["contexts"], A, max_rows)
        assert bps == pyref.break_points_for(b["contexts"], max_rows)
        N = len(b["values"])
        assert [bo.raw_cell(bps, p) for p in range(N)] == raw
        cols = pyref.assign_witnesses([list(range(N))], bps, A, 1 << 9)
        for j, (s, cnt) in enumerate(bo.spans(bps, N)):
            assert cols[j][:cnt] == list(range(s, s + cnt))
        lit = bo.run(9, A, 0, False, 4, max_rows, b, b["values"])
        fast = bo.run(9, A, 0, False, 4, max_rows, b, b["values"], record=False)
        assert lit["q"] == fast["q"] and lit["satisfied"] and fast["satisfied"]


def test_panics():
    with pytest.raises(bo.Panic, match="NOT ENOUGH ADVICE COLUMNS"):
        _walk([[0] * 10], 1, 10)
    with pytest.raises(bo.Panic, match="We do not support overlaps with delta = 1"):
        _walk([[0] * 6 + [1, 1, 0, 0, 0]], 2, 10)
    with pytest.raises(bo.Panic, match="We do not support overlaps with delta = 2"):
        _walk([[0] * 5 + [1, 0, 1, 0, 0, 0]], 2, 10)
    rng = np.random.default_rng(1)
    b = bo.make_builder(rng, 8, 1, 1, False, 4, 240)
    b["lookups"] = np.arange(241, dtype=np.uint64)
    with pytest.raises(bo.Panic, match="range lookups would be assigned to unusable rows"):
        bo.run(8, 1, 1, False, 4, 240, b, b["values"])
    b = bo.make_builder(rng, 8, 2, 0, False, 4, 240)
    b["lookups"] = np.arange(3, dtype=np.uint64)
    with pytest.raises(bo.Panic, match="range lookups require lookup advice columns"):
        bo.run(8, 2, 0, False, 4, 240, b, b["values"])
    for key in ("advice_equalities", "constant_index", "lookups"):
        b = bo.make_builder(rng, 8, 1, 0, True, 4, 240)
        b[key] = b[key].copy()
        b[key].reshape(-1)[0] = len(b["values"])
        with pytest.raises(bo.Panic, match="virtual cell not assigned"):
            bo.run(8, 1, 0, True, 4, 240, b, b["values"])
    b = {"contexts": [np.zeros(3, dtype=np.uint8)], "advice_equalities": np.zeros((0, 2), dtype=np.uint64), "lookups": [],
         "constants": np.arange(10, dtype=np.uint64), "constant_index": np.zeros(10, dtype=np.uint64)}
    assert bo.run(4, 1, 0, False, 2, 9, dict(b, constants=b["constants"][:9]), [0, 0, 0])["constants"][0] == 8
    with pytest.raises(bo.Panic, match="NotEnoughRowsAvailable"):  # 10 distinct constants, 2^4 - 7 = 9 usable rows
        bo.run(4, 1, 0, False, 2, 9, b, [0, 0, 0])
    with pytest.raises(bo.Panic, match="range lookup assigned to an unusable row"):
        bo.assign_lookups_in_phase([3], lambda p: (0, 12), 10, 1, 0, True, 12)


@pytest.mark.parametrize("A,L,sel", [(1, 0, True), (3, 2, False), (2, 0, False)])
def test_hand_placed_violations(A, L, sel):
    rng = np.random.default_rng(10 + A)
    k, bits = 8, 4
    max_rows = (1 << k) - 9
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
    assert bo.run(k, A, L, sel, bits, max_rows, b, b["values"])["satisfied"]
    m = b["meta"]
    bps = bo.run(k, A, L, sel, bits, max_rows, b, b["values"])["break_points"]
    v = b["values"].copy()
    y = int(m["y"][3])
    v[y] += 1
    got = bo.run(k, A, L, sel, bits, max_rows, b, v)
    assert got["equalities"] == (1, [3]) and got["equality_cells"] == [(bo.raw_cell(bps, y - 1), bo.raw_cell(bps, y))]
    assert not any(c for c, _ in got["gates"]) and got["constants"][0] == 0
    v = b["values"].copy()
    t = int(np.flatnonzero(m["c"] == 1)[2])
    c_cell = int(m["x"][t]) + 2
    v[c_cell] = 0  # a bit tied to the constant 1: its constant equality, and its gate unless b_t = 0
    i = int(np.flatnonzero(b["constant_index"] == c_cell)[0])
    got = bo.run(k, A, L, sel, bits, max_rows, b, v)
    assert got["constants"] == (1, [i]) and got["constant_cells"] == [bo.raw_cell(bps, c_cell)]
    col, row = bo.raw_cell(bps, int(m["x"][t]))
    gate_fails = int(b["values"][int(m["x"][t]) + 1]) != 0
    assert got["gates"][col] == ((1, [row]) if gate_fails else (0, []))
    if b["lookups"].size:
        v = b["values"].copy()
        j = 5
        v[int(b["lookups"][j])] = 1 << bits
        got = bo.run(k, A, L, sel, bits, max_rows, b, v)
        lk_t, lk_row = (0, bo.raw_cell(bps, int(b["lookups"][j]))[1]) if L == 0 else (j % L, j // L)
        assert got["lookups"][lk_t] == (1, [lk_row])

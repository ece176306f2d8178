"""CPU tests of the C restatement of halo2-base's own witness form (tests/cpp/assigned_witness_oracle.c through
tests/assigned_oracle.py): batch_invert_assigned over the Vec<Assigned> that (values, Rational pairs) stand for, then
assign_raw over the lookup indices, pinned against plain-integer formulas (assigned_oracle.apply_rational,
oracle/pyref.py's assign_lookups)."""
import numpy as np
import pytest
from oracle import pyref, oracle as orc
from util import *
import assigned_oracle as ao

R = pyref.R


def _case(rng, N, n_rat, zero_den=0, zero_num=0):
    """N cells; n_rat of them Rational (sorted distinct indices), the first zero_den with d = 0, the next zero_num with n = 0;
    about a quarter of the others Zero (value 0)"""
    values = rand_ints(rng, N, R)
    for j in rng.choice(N, size=N // 4, replace=False):
        values[j] = 0
    index = sorted(int(i) for i in rng.choice(N, size=n_rat, replace=False))
    den = rand_ints(rng, n_rat, R)
    for i in range(min(zero_den, n_rat)):
        den[i] = 0
    for i in range(zero_den, min(zero_den + zero_num, n_rat)):
        values[index[i]] = 0
    return values, index, den


def _run(values, index, den, lk, k, L):
    return ao.assigned_witness(mont(values, R), np.array(index, dtype=np.uint64), mont(den, R).reshape(-1, 4),
                                np.array(lk, dtype=np.uint64), k, L)


@pytest.mark.parametrize("N,n_rat,zero_den,zero_num,n_lookup,k,L", [
    (200, 20, 0, 0, 37, 5, 2),     # Zero / Trivial / Rational mix; n_lookup not divisible by L
    (200, 20, 3, 4, 64, 6, 1),     # d = 0 cells and n = 0 cells with d != 0
    (150, 0, 0, 0, 10, 4, 3),      # R = 0
    (96, 96, 5, 5, 30, 4, 2),      # R = N: every cell Rational
    (1, 1, 0, 0, 4, 2, 3),         # a single cell, looked up four times
    (300, 50, 2, 0, 0, 6, 0),      # no lookups at all
])
def test_oracle_matches_plain_integers(N, n_rat, zero_den, zero_num, n_lookup, k, L):
    rng = np.random.default_rng(N + n_rat + 7 * n_lookup)
    values, index, den = _case(rng, N, n_rat, zero_den, zero_num)
    lk = [int(x) for x in rng.integers(0, N, size=n_lookup)]
    if n_lookup >= 3:
        lk[0] = lk[1] = lk[2]      # one cell looked up repeatedly
        lk[-1] = N - 1             # the last cell of the virtual column
    rc, out, cols = _run(values, index, den, lk, k, L)
    assert rc == 0
    want = ao.apply_rational(values, list(zip(index, den)))
    assert unmont(out, R) == want
    for i, d in zip(index, den):
        assert want[i] == (values[i] * pow(d, -1, R) % R if d else 0)
    if L:
        want_cols = pyref.assign_lookups([want[i] for i in lk], L, 1 << k)
        assert [unmont(c, R) for c in cols] == want_cols
    # with no Rational cell and value lookups the oracle is the existing assign_lookups
    if n_rat == 0 and L:
        rc2, cols2 = orc.assign_lookups(mont([values[i] for i in lk], R), k, L)
        assert rc2 == 0 and np.array_equal(cols, cols2)


def test_rational_with_zero_denominator_is_zero_and_nonzero_numerator_survives_elsewhere():
    values = [5, 7, 11, 13]
    rc, out, _ = _run(values, [1, 3], [0, 2], [], 3, 0)
    assert rc == 0 and unmont(out, R) == [5, 0, 11, 13 * pow(2, -1, R) % R]


@pytest.mark.parametrize("index,lk,k,L,want", [
    ([0, 10], [], 3, 1, -2),          # a Rational index == N
    ([3], [10], 3, 1, -2),            # a lookup index == N
    ([2, 2], [], 3, 1, -3),           # repeated Rational index
    ([5, 3], [], 3, 1, -3),           # decreasing Rational indices
    ([], list(range(9)), 3, 1, -1),   # 9 lookups in one column of 2^3 rows
    ([], list(range(10)) * 2, 2, 4, -1),  # 20 lookups over 4 columns of 4 rows
    ([], [1], 3, 0, -1),              # lookups but no lookup column
])
def test_oracle_rejects(index, lk, k, L, want):
    rng = np.random.default_rng(5)
    values = rand_ints(rng, 10, R)
    rc, _, _ = _run(values, index, rand_ints(rng, len(index), R), lk, k, L)
    assert rc == want

"""The operand families of tests/field_edges.py reach what the device and host field tests rely on, so that a later edit
cannot quietly weaken them: both sides of the final conditional subtraction within 2^32 of m for every product op, the
largest values before that subtraction, limbs with the top limb of m, and every value below m."""
import pytest
import field_edges as fe

SIDE = 1 << 32


@pytest.mark.parametrize("field", ["Fq", "Fr"])
def test_every_operand_is_below_the_modulus(field):
    m = fe.FIELDS[field][1]
    for op, groups in fe.samples(field).items():
        for group, tuples in groups.items():
            assert tuples, (op, group)
            assert all(len(t) == fe.ARITY[op] and all(0 <= v < m for v in t) for t in tuples), (op, group)


@pytest.mark.parametrize("op", fe.PRODUCT_OPS)
@pytest.mark.parametrize("field", ["Fq", "Fr"])
def test_products_reach_both_sides_of_the_final_subtraction(field, op):
    """t = (S + M m) / 2^256 lands in [m, m + 2^32) (subtracted) and in [m - 2^32, m) (not) for some samples.  from_mont
    (op 4) is the one exception: its second factor is 1, so t < (m + (2^256 - 1) m) / 2^256 = m and the subtraction is
    never taken; for it the test asserts exactly that."""
    m = fe.FIELDS[field][1]
    groups = {g: ts for g, ts in fe.samples(field)[op].items() if g != "pattern"}  # the 2^18 limb patterns reach neither edge
    ts = {g: [fe.unreduced(op, m, t) for t in tuples] for g, tuples in groups.items()}
    every = [t for v in ts.values() for t in v]
    assert all(t < 2 * m for t in every)
    below = sum(m - SIDE <= t < m for t in every)
    above = sum(m <= t < m + SIDE for t in every)
    assert below >= 2, (op, below)
    if op == 4:
        assert max(every) < m
    else:
        assert above >= 2, (op, above)
    # the targeted results are what the solver aimed at (t and the result agree mod m)
    targets = set(fe.TARGETS(m)) | ({j for j in range(3, 40)} | {m - j for j in range(3, 40)} if op == 6 else set())
    for tup, t in zip(groups["boundary"], ts["boundary"]):
        assert t % m == fe.reference(op, m, tup) and t % m in targets
    if op == 0:
        assert max(every) >= 1.15 * m
    if op == 10:
        assert max(every) >= 1.3 * m


@pytest.mark.parametrize("field", ["Fq", "Fr"])
def test_add_sub_boundaries_are_reached(field):
    m = fe.FIELDS[field][1]
    s = fe.samples(field)
    sums = {a + b for a, b in s[1]["add/sub boundary"]}
    assert {m - 1, m, m + 1, 2 * m - 2} <= sums
    diffs = {a - b for a, b in s[2]["add/sub boundary"]}
    assert {0, -1, -(m - 1), m - 1} <= diffs
    assert {b for _, b in s[8]["add/sub boundary"]} >= {0, m - 1}  # neg(0) and neg(m - 1) inside mul_sub_mul


@pytest.mark.parametrize("field", ["Fq", "Fr"])
def test_limb_patterns_have_the_shapes_asked_for(field):
    """the top limb equals MOD(7) in a good share, with the lower limbs both saturated and cleared, and bit 31 is set
    in every limb below the top one"""
    m = fe.FIELDS[field][1]
    pat = fe.pattern_family(m, 1 << 14, 1)
    top = [v for v in pat if fe.limb(v, 7) == fe.limb(m, 7)]
    assert len(top) >= len(pat) // 3
    assert any(all(fe.limb(v, j) == 0xFFFFFFFF for j in range(3)) for v in top)
    assert any(all(fe.limb(v, j) == 0 for j in range(3)) for v in top)
    assert any(fe.limb(v, 6) == fe.limb(m, 6) and fe.limb(v, 5) == fe.limb(m, 5) for v in top)
    for j in range(7):  # limb 7 stays <= MOD(7) < 2^31
        assert sum(fe.limb(v, j) >> 31 for v in pat) > len(pat) // 8, j
    fixed = fe.fixed_family(m)
    assert {0, 1, 2, 3, m - 1, m - 2, (m - 1) // 2, (m + 1) // 2, fe.W % m, m - fe.W % m} <= set(fixed)
    assert all(v < m for v in fixed + pat)


def test_square_roots_and_inversion_inputs():
    for m in (fe.P, fe.R):
        for x in (2, 3, 5, 7, fe.W % m, m - 1):
            r = fe.sqrt_mod(x, m)
            assert r is None or r * r % m == x
            assert (r is None) == (pow(x, (m - 1) // 2, m) != 1)
        inv = [t[0] for t in fe.inversion_samples(m)]
        assert 1 in inv and m - 1 in inv and (m + 1) // 2 in inv and 1 << 253 in inv
        with pytest.raises(ValueError):
            fe.checked([m], m)

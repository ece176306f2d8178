"""CPU tests of the keygen oracles (tests/keygen_oracle.py) on the copy graphs of tests/forest_cases.py: halo2's Assembly in
Python, the same in C and the closed form (Kruskal's forest by call index and its walk) give one mapping, and that mapping is a
permutation whose cycles are exactly the copy graph's connected components.  The GPU tests of the device forest
(tests/test_gpu_keygen_forest.py) trust these oracles on the same graphs at larger sizes."""
import numpy as np
import pytest
import forest_cases as fc
import keygen_oracle as ko


@pytest.mark.parametrize("E", [1, 7, 300])
@pytest.mark.parametrize("name", sorted(fc.GENERATORS))
def test_the_three_oracles_agree_and_cycles_are_components(name, E):
    rng = np.random.default_rng(E * 31 + len(name))
    V = fc.need(name, E) + int(rng.integers(0, 40))
    pairs = fc.GENERATORS[name](rng, V, E)
    assert pairs.shape == (E, 2) and pairs.dtype == np.uint32 and int(pairs.max()) < V
    want = ko.assembly(V, pairs)
    assert np.array_equal(ko.assembly_c(V, pairs), want)
    assert np.array_equal(ko.closed_form(V, pairs), want)
    fc.check_cycles(V, pairs, want)


def test_star_with_many_leaves():
    """2^17 leaves: the hub's cycle holds every leaf"""
    rng = np.random.default_rng(17)
    E = 1 << 17
    V = E + 1000
    for hub in ("left", "right", "mixed"):
        pairs = fc.star(rng, V, E, hub)
        want = ko.assembly_c(V, pairs)
        fc.check_cycles(V, pairs, want)
        if hub != "mixed":
            assert np.array_equal(ko.assembly(V, pairs), want)


def test_a_clique_among_other_components():
    rng = np.random.default_rng(64)
    V, E = 3000, 2016 + 1500
    pairs = fc.clique(rng, V, E)
    # the 64-cell clique is there, in full
    _, lab = fc.components(V, pairs)
    sizes = np.bincount(lab)
    assert sizes.max() >= 64
    want = ko.assembly(V, pairs)
    assert np.array_equal(ko.assembly_c(V, pairs), want)
    assert np.array_equal(ko.closed_form(V, pairs), want)
    fc.check_cycles(V, pairs, want)


@pytest.mark.parametrize("where", ["after", "before", "mixed"])
def test_redundant_copies_leave_the_forest_alone(where):
    """the copies that join nothing (duplicates, reversed duplicates, self-copies, cycle closers) change no entry: the mapping
    of the graph equals that of its spanning forest alone, which the Assembly keeps"""
    rng = np.random.default_rng(5)
    V, E = 900, 800
    pairs = fc.redundant(rng, V, E, where)
    want = ko.assembly(V, pairs)
    # Kruskal by call index: the copies that join two classes when made
    parent = list(range(V))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    keep = []
    for x, y in pairs.tolist():
        rx, ry = find(x), find(y)
        if rx != ry:
            parent[rx] = ry
            keep.append((x, y))
    assert len(keep) < E
    assert np.array_equal(ko.assembly(V, np.array(keep, dtype=np.uint32)), want)
    assert np.array_equal(ko.closed_form(V, pairs), want)
    fc.check_cycles(V, pairs, want)


def test_long_decreasing_path_walks_the_whole_component():
    """from the path's first cell the closed form's walk crosses every copy; the mapping is one cycle through all of them"""
    rng = np.random.default_rng(9)
    V, E = 1200, 1000
    cells = rng.choice(V, size=E + 1, replace=False)
    pairs = fc.path(rng, V, E, "decreasing", cells=cells)
    want = ko.assembly(V, pairs)
    assert np.array_equal(ko.closed_form(V, pairs), want)
    fc.check_cycles(V, pairs, want)
    # every copy goes first in the transposition product: sigma(first cell) = the far end of the path
    assert want[cells[0]] == cells[-1]


def test_one_edge_components_leave_the_other_cells_fixed():
    rng = np.random.default_rng(2)
    V, E = 5000, 1200
    pairs = fc.one_edge(rng, V, E)
    want = ko.assembly(V, pairs)
    a, b = pairs[:, 0].astype(np.int64), pairs[:, 1].astype(np.int64)
    assert np.array_equal(want[a], b) and np.array_equal(want[b], a)
    untouched = np.setdiff1d(np.arange(V), pairs.reshape(-1))
    assert len(untouched) == V - 2 * E and np.array_equal(want[untouched], untouched)


def test_extreme_cell_ids_past_2_24():
    """ids 0, V - 1 and around 2^24 in a 2^25-cell graph: the C Assembly and the closed form agree"""
    rng = np.random.default_rng(24)
    V, E = 8 << 22, 3000
    pairs = fc.extremes(rng, V, E)
    assert {0, V - 1, 1 << 24} <= set(pairs.reshape(-1).tolist())
    want = ko.assembly_c(V, pairs)
    assert np.array_equal(ko.closed_form(V, pairs), want)
    fc.check_cycles(V, pairs, want)


def test_the_invariant_catches_a_wrong_mapping():
    """check_cycles fails on a mapping that splits or merges components, or that is not a permutation"""
    rng = np.random.default_rng(1)
    V, E = 400, 300
    pairs = fc.random_graph(rng, V, E)
    good = ko.assembly(V, pairs)
    fc.check_cycles(V, pairs, good)
    x = int(pairs[0, 0]) if pairs[0, 0] != pairs[0, 1] else int(pairs[1, 0])
    split = good.copy()  # x leaves its cycle
    y = int(np.nonzero(good == x)[0][0])
    split[y], split[x] = good[x], x
    assert good[x] != x
    dup = good.copy()  # good[x] twice
    dup[y] = good[x]
    bad = {"split": split, "not a permutation": dup}
    fixed = np.nonzero(good == np.arange(V))[0]
    if len(fixed) >= 2:
        merged = good.copy()
        merged[fixed[0]], merged[fixed[1]] = fixed[1], fixed[0]
        bad["merged"] = merged
    for name, m in bad.items():
        with pytest.raises(AssertionError):
            fc.check_cycles(V, pairs, m)

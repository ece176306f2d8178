"""CPU tests of tests/keygen_oracle.py, the yardstick of the device keygen: the closed form of halo2's permutation Assembly
equals the literal Assembly on random multigraphs (self-loops, duplicate, reversed and redundant copies) and on the copy
sequences of synthetic halo2-base builders of every shape; every sigma cycle is exactly one copy class
(scipy.sparse.csgraph.connected_components, independent of both); the C restatement equals the Python one; the copy
sequence does not depend on the builder's order of its equalities."""
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components
import builder_oracle as bo
import keygen_oracle as ko

SHAPES = [(1, 0, True), (3, 2, False), (2, 0, False), (2, 1, True)]


def _random_pairs(rng, V, E):
    p = rng.integers(0, V, size=(E, 2))
    loops = rng.random(E) < 0.05
    p[loops, 1] = p[loops, 0]                                   # self-loops
    dup = rng.integers(0, E, size=E // 10)
    p = np.concatenate([p, p[dup], p[dup][:, ::-1]])           # duplicates and reversed duplicates
    return p[rng.permutation(len(p))]


def _cycles_are_classes(sigma, pairs):
    V = len(sigma)
    p = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    g = sp.coo_matrix((np.ones(len(p)), (p[:, 0], p[:, 1])), shape=(V, V))
    _, cls = connected_components(g, directed=False)
    # a permutation whose cycles are the classes: sigma stays inside each class and one cycle covers it
    assert (cls[sigma.astype(np.int64)] == cls).all()
    seen = np.zeros(V, dtype=bool)
    for x in range(V):
        if seen[x]:
            continue
        cyc = [x]
        seen[x] = True
        y = int(sigma[x])
        while y != x:
            assert not seen[y]
            seen[y] = True
            cyc.append(y)
            y = int(sigma[y])
        assert len(cyc) == int((cls == cls[x]).sum())


@pytest.mark.parametrize("seed", range(40))
def test_closed_form_equals_the_assembly_on_random_multigraphs(seed):
    rng = np.random.default_rng(seed)
    V = int(rng.integers(2, 200))
    pairs = _random_pairs(rng, V, int(rng.integers(0, 3 * V)))
    lit = ko.assembly(V, pairs)
    assert np.array_equal(ko.closed_form(V, pairs), lit)
    assert np.array_equal(ko.assembly_c(V, pairs), lit)
    _cycles_are_classes(lit, pairs)


@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_closed_form_equals_the_assembly_on_builders(A, L, sel):
    k, bits = 8, 6
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(40 + A + L)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, contexts=3)
    pairs, c_rows, bps = ko.copy_sequence(k, A, L, max_rows, b)
    assert bps == bo.run(k, A, L, sel, bits, max_rows, b, b["values"])["break_points"]
    assert c_rows == bo.assign_constants(zip(b["constants"], b["constant_index"]), (1 << k) - 7, k)
    V = (1 + A + L) << k
    lit = ko.assembly(V, pairs)
    assert np.array_equal(ko.closed_form(V, pairs), lit)
    _cycles_are_classes(lit, pairs)
    # halo2-base sorts the equalities: the builder's order of them does not matter
    perm, cperm = rng.permutation(len(b["advice_equalities"])), rng.permutation(len(b["constants"]))
    shuffled = dict(b, advice_equalities=b["advice_equalities"][perm],
                    constants=b["constants"][cperm], constant_index=b["constant_index"][cperm])
    assert np.array_equal(ko.copy_sequence(k, A, L, max_rows, shuffled)[0], pairs)


@pytest.mark.parametrize("k", [10, 12])
def test_the_c_assembly_equals_python(k):
    A, L, sel, bits = 3, 2, False, 8
    max_rows = (1 << k) - 9
    b = bo.make_builder(np.random.default_rng(k), k, A, L, sel, bits, max_rows)
    pairs = ko.copy_sequence(k, A, L, max_rows, b)[0]
    V = (1 + A + L) << k
    assert np.array_equal(ko.assembly_c(V, pairs), ko.assembly(V, pairs))


def test_sigma_values_are_delta_and_omega_powers():
    from oracle import pyref
    from util import unmont
    k, n_cols = 4, 4
    m = np.random.default_rng(0).permutation(n_cols << k).astype(np.uint32)
    v = unmont(ko.sigma_values(m, n_cols, k).reshape(-1, 4), pyref.R)
    w = pyref.omega_for(k)
    assert v == [pow(pyref.DELTA, int(x) >> k, pyref.R) * pow(w, int(x) & 15, pyref.R) % pyref.R for x in m]

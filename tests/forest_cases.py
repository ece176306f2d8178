"""Copy graphs shaped to stress keygen's spanning forest, its walk and its dart sort (csrc/keygen.cu), for
tests/test_oracle_keygen_forest.py and tests/test_gpu_keygen_forest.py.  Random builders make shallow components; these make
long paths whose walks cross a whole component and whose hook chains need many pointer-jumping launches, wide stars, a dense
clique, redundant copies before and after the forest, many one-edge components and cell ids whose high bytes vary.

Every generator takes (rng, V, E) and returns exactly E copies as an (E, 2) uint32 array of cell ids < V in call order
(cell id c 2^k + r; V = n_cols 2^k).  need(name, E) is the least V a generator accepts.  components(V, pairs) and
check_cycles(V, pairs, mapping) state the invariant every mapping must meet: it is a permutation whose cycles are exactly the
connected components of the copy graph."""
from __future__ import annotations
import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components


def _orient(rng, pairs: np.ndarray) -> np.ndarray:
    """each copy written (x, y) or (y, x) at random"""
    flip = rng.random(len(pairs)) < 0.5
    pairs[flip] = pairs[flip][:, ::-1]
    return pairs


def _u32(pairs) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(pairs, dtype=np.int64).reshape(-1, 2).astype(np.uint32))


def interleave(rng, *parts) -> np.ndarray:
    """the copies of every part in their own order, the parts shuffled among one another"""
    parts = [np.asarray(p, dtype=np.int64).reshape(-1, 2) for p in parts]
    tags = np.concatenate([np.full(len(p), i) for i, p in enumerate(parts)]).astype(np.int64)
    rng.shuffle(tags)
    out = np.empty((len(tags), 2), dtype=np.int64)
    for i, p in enumerate(parts):
        out[tags == i] = p
    return out


# ------------------------------------------------------------------------------------------------------------ paths
def _path_ranks(order: str, m: int, rng) -> np.ndarray:
    """call-order rank of the i-th edge along the path"""
    if order == "increasing":
        return np.arange(m)
    if order == "decreasing":  # a walk from the path's first cell crosses every edge
        return np.arange(m)[::-1].copy()
    if order == "alternating":  # small, large, small, large, .. along the path
        r = np.empty(m, dtype=np.int64)
        r[0::2] = np.arange((m + 1) // 2)
        r[1::2] = m - 1 - np.arange(m // 2)
        return r
    assert order == "shuffled"
    return rng.permutation(m)


def path(rng, V: int, E: int, order: str, cells=None) -> np.ndarray:
    """one path through E + 1 cells taken in a random order; edge i along the path is copy number ranks[i]"""
    cells = rng.choice(V, size=E + 1, replace=False) if cells is None else np.asarray(cells, dtype=np.int64)
    along = np.stack([cells[:-1], cells[1:]], axis=1).astype(np.int64)
    out = np.empty_like(along)
    out[_path_ranks(order, E, rng)] = along
    return _u32(_orient(rng, out))


# ------------------------------------------------------------------------------------------------------------ stars
def star(rng, V: int, E: int, hub: str) -> np.ndarray:
    """one hub copied to E leaves in random id order; the hub is the left cell, the right one, or either"""
    cells = rng.choice(V, size=E + 1, replace=False).astype(np.int64)
    out = np.stack([np.full(E, cells[0]), cells[1:]], axis=1)
    if hub == "right":
        out = out[:, ::-1]
    elif hub == "mixed":
        out = _orient(rng, out)
    return _u32(out)


# ----------------------------------------------------------------------------------------------------------- clique
def clique(rng, V: int, E: int, m: int = 64) -> np.ndarray:
    """every pair of m cells (m = 64: 2016 copies, 1953 of them redundant) in random order, among a random graph on the
    other cells that makes up the rest of the E copies; m shrinks when E has no room for the whole clique"""
    while m * (m - 1) // 2 > E:
        m //= 2
    cells = rng.permutation(V).astype(np.int64)
    kc, rest = cells[:m], cells[m:]
    i, j = np.triu_indices(m, 1)
    cl = _orient(rng, np.stack([kc[i], kc[j]], axis=1)[rng.permutation(len(i))])
    e2 = E - len(cl)
    other = np.stack([rest[rng.integers(0, len(rest), e2)], rest[rng.integers(0, len(rest), e2)]], axis=1)
    return _u32(interleave(rng, cl, other))


# -------------------------------------------------------------------------------------------------- redundant copies
def _tree(rng, V: int, E: int):
    """(cells, copies): E copies that each join a new cell to a random earlier one, one random tree of every depth"""
    cells = rng.choice(V, size=E + 1, replace=False).astype(np.int64)
    parent = (rng.random(E) * np.arange(1, E + 1)).astype(np.int64)
    return cells, _orient(rng, np.stack([cells[1:], cells[parent]], axis=1))


def forest_of_trees(rng, V: int, E: int) -> np.ndarray:
    return _u32(_tree(rng, V, E)[1])


def redundant(rng, V: int, E: int, where: str) -> np.ndarray:
    """a random tree of about E / 2 copies and, for the rest, exact and reversed duplicates of its copies, self-copies (x, x)
    and copies between two of its cells, which close a cycle when made after the tree's; placed after the tree's copies,
    before them, or mixed among them"""
    F = max(1, E // 2)
    cells, tree = _tree(rng, V, F)
    n_red = E - F
    q = n_red // 4
    pick = lambda m: cells[rng.integers(0, len(cells), m)]
    dup = tree[rng.integers(0, F, q)]
    rev = tree[rng.integers(0, F, q)][:, ::-1]
    selfc = np.repeat(pick(q)[:, None], 2, axis=1)
    cyc = np.stack([pick(n_red - 3 * q), pick(n_red - 3 * q)], axis=1)
    extra = np.concatenate([dup, rev, selfc, cyc])[rng.permutation(n_red)]
    if where == "after":
        out = np.concatenate([tree, extra])
    elif where == "before":
        out = np.concatenate([extra, tree])
    else:
        out = interleave(rng, tree, extra)
    return _u32(out)


# ------------------------------------------------------------------------------------------- small components, random
def one_edge(rng, V: int, E: int) -> np.ndarray:
    """E components of one copy each on 2E distinct cells; the V - 2E cells left over are untouched"""
    cells = rng.choice(V, size=2 * E, replace=False).astype(np.int64)
    return _u32(cells.reshape(-1, 2))


def random_graph(rng, V: int, E: int) -> np.ndarray:
    """E copies between uniformly random cells (self-copies and duplicates included); V sets the density"""
    return _u32(rng.integers(0, V, size=(E, 2)))


def extremes(rng, V: int, E: int) -> np.ndarray:
    """copies among cell 0, cell V - 1, the cells around 2^16 and 2^24 (where V reaches past them) and random cells, so that
    the high bytes of the dart keys' vertex half vary: a chain through the extreme cells, then random copies half of whose
    ends are extreme cells"""
    pool = [0, 1, V - 2, V - 1]
    for b in (1 << 16, 1 << 24):
        if V > b + 2:
            pool += [b - 1, b, b + 1]
    pool = rng.permutation(np.unique(np.array(pool, dtype=np.int64)))
    chain = np.stack([pool[:-1], pool[1:]], axis=1)[:E]
    r = E - len(chain)
    draw = lambda: np.where(rng.random(r) < 0.5, pool[rng.integers(0, len(pool), r)], rng.integers(0, V, r))
    return _u32(interleave(rng, chain, np.stack([draw(), draw()], axis=1)))


# ----------------------------------------------------------------------------------------------------------- catalog
GENERATORS = {
    "path_increasing": lambda rng, V, E: path(rng, V, E, "increasing"),
    "path_decreasing": lambda rng, V, E: path(rng, V, E, "decreasing"),
    "path_alternating": lambda rng, V, E: path(rng, V, E, "alternating"),
    "path_shuffled": lambda rng, V, E: path(rng, V, E, "shuffled"),
    "star_hub_left": lambda rng, V, E: star(rng, V, E, "left"),
    "star_hub_right": lambda rng, V, E: star(rng, V, E, "right"),
    "star_hub_mixed": lambda rng, V, E: star(rng, V, E, "mixed"),
    "clique": clique,
    "redundant_after": lambda rng, V, E: redundant(rng, V, E, "after"),
    "redundant_before": lambda rng, V, E: redundant(rng, V, E, "before"),
    "redundant_mixed": lambda rng, V, E: redundant(rng, V, E, "mixed"),
    "tree": forest_of_trees,
    "one_edge": one_edge,
    "random_sparse": random_graph,   # E = V / 2
    "random_even": random_graph,     # E = V
    "random_dense": random_graph,    # E = 4 V
    "extremes": extremes,
}

# the least V for E copies: enough distinct cells for the paths, stars and one-edge components; the random graphs' density
_DENSITY = {"random_sparse": 2.0, "random_even": 1.0, "random_dense": 0.25, "one_edge": 2.0}


def need(name: str, E: int) -> int:
    return int(np.ceil(_DENSITY.get(name, 1.0) * E)) + 2


# ---------------------------------------------------------------------------------------------------------- invariant
def components(V: int, pairs) -> tuple[int, np.ndarray]:
    """(count, label per cell) of the copy graph's connected components"""
    p = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    g = sp.coo_matrix((np.ones(len(p), dtype=np.int8), (p[:, 0], p[:, 1])), shape=(V, V)).tocsr()
    return connected_components(g, directed=False)


def check_cycles(V: int, pairs, mapping) -> None:
    """mapping is a permutation of the V cells whose cycles are exactly the copy graph's components"""
    m = np.asarray(mapping, dtype=np.int64)
    assert len(m) == V
    seen = np.zeros(V, dtype=bool)
    seen[m] = True
    assert seen.all(), "the mapping is not a permutation"
    nc, lab = components(V, pairs)
    assert np.array_equal(lab[m], lab), "a cycle leaves its component"
    nk, _ = components(V, np.stack([np.arange(V, dtype=np.int64), m], axis=1))
    assert nk == nc, "%d cycles for %d components" % (nk, nc)  # each component is one cycle

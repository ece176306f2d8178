"""GPU tests (-m gpu) of keygen's permutation kernels (csrc/keygen.cu, include/h2b200.h's keygen section) through the C ABI,
with torch tensors as device buffers, every comparison exact:
  sigma_map      the copy graphs of tests/forest_cases.py against halo2's Assembly (tests/keygen_oracle.py), at dart counts
                 that put the cooperative radix sort (csrc/lookup.cu) in each of its grid regimes, one 2^25-cell graph, and
                 the edges (no copies, k = 1, one column, a cell id out of range);
  sigma_values   every cell against keygen_oracle.sigma_values at small k, sampled cells against plain integers at k = 20, 23;
  copies_nf      the copy calls and constants block against a numpy restatement of the order the header documents, on inputs
                 that make the byte-skipping key sort, the stable second sort of the constants and the row limit bite;
  instance_edges the rows at and past `usable`."""
import ctypes as C
import numpy as np
import pytest
from oracle import pyref
from util import mont
import forest_cases as fc
import keygen_oracle as ko

pytestmark = pytest.mark.gpu
R = pyref.R
vp = C.c_void_p
RS_T = 256  # elements per tile of lookup.cu's radix sort


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def h2b():
    import halo2_lib_b200 as h
    return h


@pytest.fixture(scope="module")
def lib(h2b):
    from halo2_lib_b200._capi import lib as l
    return l


@pytest.fixture(scope="module")
def ctx(h2b):
    c = h2b.Context(0)
    yield c
    c.close()


def _dev(torch, a, dtype):
    """a device copy of host array a (viewed as the signed type torch knows), complete before the library's stream reads it"""
    a = np.ascontiguousarray(a, dtype=dtype)
    t = torch.from_numpy(a.view({np.uint32: np.int32, np.uint64: np.int64}[np.dtype(dtype).type])).cuda()
    torch.cuda.synchronize()
    return t


def _host(t, dtype):
    return t.cpu().numpy().view(dtype)


def _ptr(t):
    return vp(t.data_ptr()) if t is not None else None


def sigma_map(torch, ctx, lib, pairs, n_cols, k):
    pairs = np.asarray(pairs, dtype=np.uint32).reshape(-1, 2)
    d_e = _dev(torch, pairs.reshape(-1), np.uint32) if len(pairs) else None
    d_m = torch.full(((n_cols << k) + 64,), -1, dtype=torch.int32, device="cuda")  # 64 guard words past the map
    ctx.check(lib.h2b_keygen_sigma_map_dev(ctx.h, _ptr(d_e), len(pairs), n_cols, k, _ptr(d_m)))
    got = _host(d_m, np.uint32)
    assert (got[n_cols << k:] == 0xFFFFFFFF).all(), "written past the map"
    return got[: n_cols << k]


def _shape(V: int, n_cols: int):
    """(n_cols, k): the least k with n_cols 2^k >= V"""
    k = max(1, int(np.ceil(np.log2(max(2, -(-V // n_cols))))))
    return n_cols, k


# ---------------------------------------------------------------------------------------------- sort-grid regimes
# E copies make D = 2E darts and ceil(D / 256) tiles; sort_column_ctas launches min(SMs x min(occupancy, 4), tiles) CTAs.
# k_radix_sort holds 6 CTAs of 256 threads per SM (40 registers, 11 KB of shared memory on sm_90a), so the cap is 4 per SM.
SIZES = {
    "one_cta": 100,                     # D = 200: one tile
    "rows_per_cta": (1 << 11) + 3,      # D = 2^12 + 6: 17 CTAs, each scans several rows of the bin table
    "row_scan_wraps": (1 << 15) + 5,    # D = 2^16 + 10: 257 CTAs, the row scan's loop over j0 runs twice
    "segments": (1 << 19) + 7,          # D = 2^20 + 14: more tiles than CTAs, base[] carried from tile to tile
    "segments_2^24": (1 << 23) + 1,     # D = 2^24 + 2
}
# at the largest size, the shapes whose walks, hook chains or key bytes differ most
LARGEST = ["path_decreasing", "path_increasing", "star_hub_mixed", "redundant_before", "one_edge", "random_sparse", "extremes"]


def sort_ctas(torch, D: int) -> tuple[int, int]:
    """(CTAs, tiles) of the sort of D keys, as the library sizes the cooperative grid"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = -(-D // RS_T)
    return min(sms * 4, tiles), tiles


def test_the_sizes_reach_every_sort_grid_regime(torch):
    got = {name: sort_ctas(torch, 2 * E) for name, E in SIZES.items()}
    assert all((2 * E) % RS_T for E in SIZES.values())
    assert got["one_cta"] == (1, 1)
    ctas, tiles = got["rows_per_cta"]
    assert 1 < ctas < 256 and ctas == tiles and 256 % ctas
    ctas, tiles = got["row_scan_wraps"]
    assert ctas > 256 and ctas == tiles
    for name in ("segments", "segments_2^24"):
        ctas, tiles = got[name]
        assert tiles >= 4 * ctas and tiles % ctas, name


CASES = [(name, size) for size in SIZES for name in sorted(fc.GENERATORS) if size != "segments_2^24" or name in LARGEST]


@pytest.mark.parametrize("name,size", CASES)
def test_sigma_map_matches_the_assembly(torch, ctx, lib, name, size):
    E = SIZES[size]
    rng = np.random.default_rng(100 * sorted(fc.GENERATORS).index(name) + list(SIZES).index(size))
    n_cols = [1, 3, 4, 5, 8][len(name) % 5]
    n_cols, k = (5, 22) if name == "extremes" else _shape(fc.need(name, E), n_cols)
    V = n_cols << k
    pairs = fc.GENERATORS[name](rng, V, E)
    assert pairs.shape == (E, 2)
    want = ko.assembly(V, pairs) if V <= 1 << 14 else ko.assembly_c(V, pairs)
    got = sigma_map(torch, ctx, lib, pairs, n_cols, k)
    assert np.array_equal(got, want), "%d of %d entries differ" % (int((got != want).sum()), V)


def test_sigma_map_on_a_2_25_cell_graph(torch, ctx, lib):
    """k = 22, 8 columns: a path through a quarter of the cells with decreasing copy indices, merged with a random graph"""
    rng = np.random.default_rng(2225)
    n_cols, k = 8, 22
    V = n_cols << k
    walk = fc.path(rng, V, V // 4, "decreasing")
    pairs = fc._u32(fc.interleave(rng, walk, fc.random_graph(rng, V, V // 4)))
    want = ko.assembly_c(V, pairs)
    got = sigma_map(torch, ctx, lib, pairs, n_cols, k)
    assert np.array_equal(got, want), "%d of %d entries differ" % (int((got != want).sum()), V)
    fc.check_cycles(V, pairs, got)


def test_sigma_map_edges(torch, ctx, lib, h2b):
    from halo2_lib_b200._capi import H2B_ERR_ARG
    rng = np.random.default_rng(4)
    # no copies: the identity
    assert np.array_equal(sigma_map(torch, ctx, lib, np.zeros((0, 2)), 3, 4), np.arange(3 << 4, dtype=np.uint32))
    # k = 1
    for n_cols in (1, 2, 7):
        V = n_cols << 1
        pairs = fc.random_graph(rng, V, 3 * V)
        assert np.array_equal(sigma_map(torch, ctx, lib, pairs, n_cols, 1), ko.assembly(V, pairs))
    # one column
    for name in ("path_decreasing", "star_hub_right", "random_even"):
        pairs = fc.GENERATORS[name](rng, 1 << 12, 3000)
        assert np.array_equal(sigma_map(torch, ctx, lib, pairs, 1, 12), ko.assembly(1 << 12, pairs))
    # a copy naming a cell outside the columns: H2B_ERR_ARG with its message, and the context stays usable
    n_cols, k = 3, 6
    V = n_cols << k
    good = fc.random_graph(rng, V, 200)
    for bad_cell in (V, V + 1, 0xFFFFFFFF):
        for at in (0, 1, 157, 199):
            bad = good.copy()
            bad[at, at % 2] = bad_cell
            with pytest.raises(h2b.H2BError, match="keygen_sigma_map: a copy names a cell outside the permutation columns") as e:
                sigma_map(torch, ctx, lib, bad, n_cols, k)
            assert e.value.code == H2B_ERR_ARG
            assert np.array_equal(sigma_map(torch, ctx, lib, good, n_cols, k), ko.assembly(V, good))


# -------------------------------------------------------------------------------------------------------- values
def _sigma_values(torch, ctx, lib, d_map, n_cols, k):
    d_s = torch.empty(((n_cols << k) * 4,), dtype=torch.int64, device="cuda")
    ctx.check(lib.h2b_keygen_sigma_values_dev(ctx.h, _ptr(d_map), n_cols, k, _ptr(d_s)))
    return d_s


@pytest.mark.parametrize("n_cols,k", [(1, 1), (5, 1), (3, 4), (2, 7), (7, 9)])
def test_sigma_values_match_the_oracle(torch, ctx, lib, n_cols, k):
    rng = np.random.default_rng(n_cols * 100 + k)
    V = n_cols << k
    pairs = fc.random_graph(rng, V, V)
    mapping = ko.assembly(V, pairs)
    got = _host(_sigma_values(torch, ctx, lib, _dev(torch, mapping, np.uint32), n_cols, k), np.uint64).reshape(n_cols, 1 << k, 4)
    assert np.array_equal(got, ko.sigma_values(mapping, n_cols, k))


@pytest.mark.parametrize("n_cols,k", [(40, 20), (40, 23)])
def test_sigma_values_at_sampled_cells(torch, ctx, lib, n_cols, k):
    """delta^c omega^r at cells whose map entries sit at the ends of the columns and around the split of the domain's
    two-level power table (2^h entries of omega^i and of omega^(i 2^h), h = ceil(k / 2))"""
    rng = np.random.default_rng(k)
    V, n, h = n_cols << k, 1 << k, (k + 1) // 2
    rows = [0, 1, 2, (1 << h) - 1, 1 << h, (1 << h) + 1, (3 << h) + 5, n - 2, n - 1]
    cols = [0, 1, n_cols // 2, n_cols - 1]
    targets = [c * n + r for c in cols for r in rows] + rng.integers(0, V, 200).tolist()
    where = rng.permutation(np.unique(rng.integers(1, V - 1, len(targets) + 400)))[: len(targets) + 300]
    where = np.concatenate([[0, V - 1], where]).astype(np.int64)
    d_map = (torch.arange(V, dtype=torch.int64, device="cuda") * 2654435761 % V).to(torch.int32)  # a permutation of the cells
    d_map[torch.from_numpy(where[: len(targets)]).cuda()] = torch.tensor(targets, dtype=torch.int32, device="cuda")
    d_s = _sigma_values(torch, ctx, lib, d_map, n_cols, k)
    idx = torch.from_numpy(where).cuda()
    m = _host(d_map[idx], np.uint32).astype(np.int64)
    got = _host(d_s.view(-1, 4)[idx], np.uint64)
    assert set(targets) <= set(m.tolist())
    w = pyref.omega_for(k)
    want = mont([pow(pyref.DELTA, int(x) >> k, R) * pow(w, int(x) & (n - 1), R) % R for x in m.tolist()], R)
    assert np.array_equal(got, want)
    del d_s, d_map
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------- copies (the _nf form)
def _limbs(v: int):
    return [(v >> (64 * i)) & ((1 << 64) - 1) for i in range(4)]


def copies_want(N, bps, k, F, A, L, lookups, pairs, consts, cidx):
    """(edges, c block, status) in the order include/h2b200.h documents for h2b_keygen_copies_nf_dev; consts canonical ints"""
    n = 1 << k
    bps = np.asarray(bps, dtype=np.int64)
    ends = np.cumsum(bps)
    starts = np.concatenate([[0], ends])

    def raw(p):
        p = np.asarray(p, dtype=np.int64)
        j = np.searchsorted(ends, p, side="left")
        return (F + j) * n + (p - starts[j])
    st0 = 0
    parts = [np.stack([(F + 1 + np.arange(len(bps))) * n, (F + np.arange(len(bps))) * n + bps], axis=1)]
    lk = np.asarray(lookups, dtype=np.uint64).astype(np.int64) if len(lookups) else np.zeros(0, dtype=np.int64)
    if len(lk):
        st0 |= 1 if (lk >= N).any() else 0
        i = np.arange(len(lk))
        parts.append(np.stack([np.where(lk < N, raw(np.where(lk < N, lk, 0)), 0), (F + A + i % max(L, 1)) * n + i // max(L, 1)], axis=1))
    pr = np.asarray(pairs, dtype=np.uint64).reshape(-1, 2)
    if len(pr):
        ok = (pr[:, 0] < N) & (pr[:, 1] < N)
        st0 |= 0 if ok.all() else 2
        key = np.where(ok, pr[:, 0] << np.uint64(32) | pr[:, 1], np.uint64(0))
        key = key[np.argsort(key, kind="stable")]
        parts.append(np.stack([raw((key >> np.uint64(32)).astype(np.int64)), raw((key & np.uint64(0xFFFFFFFF)).astype(np.int64))], axis=1))
    c_block = np.zeros((F * n, 4), dtype=np.uint64)
    distinct = 0
    if len(consts):
        ci = np.asarray(cidx, dtype=np.uint64)
        st0 |= 0 if (ci < N).all() else 2
        cell_key = np.where(ci < N, ci, 0).astype(np.int64)
        limbs = np.array([_limbs(int(v)) for v in consts], dtype=np.uint64)
        order = np.lexsort((np.arange(len(consts)), cell_key, limbs[:, 0], limbs[:, 1], limbs[:, 2], limbs[:, 3]))
        srt = limbs[order]
        head = np.ones(len(order), dtype=bool)
        head[1:] = (srt[1:] != srt[:-1]).any(axis=1)
        d = np.cumsum(head) - 1
        distinct = int(head.sum())
        in_c = d < F * n
        cell = np.where(in_c, (d % max(F, 1)) * n + d // max(F, 1), 0)
        hm = head & in_c
        c_block[cell[hm]] = mont([int(consts[j]) for j in order[hm]], R)
        parts.append(np.stack([cell, np.where(ci[order] < N, raw(cell_key[order]), 0)], axis=1))
    return np.concatenate(parts).astype(np.uint32), c_block, [st0, distinct]


def copies_run(torch, ctx, lib, N, bps, k, F, A, L, lookups, pairs, consts, cidx):
    """(edges, c block, status) of the device; 64 guard entries past the edges and the c block stay unwritten"""
    n = 1 << k
    bps_h = np.ascontiguousarray(bps, dtype=np.uint64)
    E = len(bps) + len(lookups) + len(pairs) + len(consts)
    lk = _dev(torch, lookups, np.uint64) if len(lookups) else None
    pr = _dev(torch, np.asarray(pairs, dtype=np.uint64).reshape(-1), np.uint64) if len(pairs) else None
    cv = _dev(torch, mont([int(v) for v in consts], R).reshape(-1), np.uint64) if len(consts) else None
    ci = _dev(torch, cidx, np.uint64) if len(consts) else None
    d_c = torch.full(((F * n + 64) * 4,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
    d_e = torch.full(((E + 64) * 2,), -1, dtype=torch.int32, device="cuda")
    d_st = torch.full((4,), -1, dtype=torch.int32, device="cuda")
    ctx.check(lib.h2b_keygen_copies_nf_dev(ctx.h, N, vp(bps_h.ctypes.data) if len(bps_h) else None, len(bps_h), k, F, A, L, _ptr(lk),
                                           len(lookups), _ptr(pr), len(pairs), _ptr(cv), _ptr(ci), len(consts),
                                           _ptr(d_c) if F else None, _ptr(d_e), _ptr(d_st)))
    e = _host(d_e, np.uint32).reshape(-1, 2)
    c = _host(d_c, np.uint64).reshape(-1, 4)
    st = _host(d_st, np.uint32)
    assert (e[E:] == 0xFFFFFFFF).all(), "written past the edges"
    assert (c[F * n:] == 0x5A5A5A5A5A5A5A5A).all(), "written past the constants block"
    assert st[2] == st[3] == 0xFFFFFFFF, "written past the status words"
    return e[:E], c[: F * n], st[:2].tolist()


def _check_copies(torch, ctx, lib, N, bps, k, F, A, L=0, lookups=(), pairs=(), consts=(), cidx=()):
    got = copies_run(torch, ctx, lib, N, bps, k, F, A, L, lookups, pairs, consts, cidx)
    want = copies_want(N, bps, k, F, A, L, lookups, pairs, consts, cidx)
    assert np.array_equal(got[0], want[0]), "%d of %d copies differ" % (int((got[0] != want[0]).any(axis=1).sum()), len(want[0]))
    assert np.array_equal(got[1], want[1]), "constants block"
    assert got[2] == want[2], "status"
    return want


def _wide_layout(k=22, A=9):
    """break points near 2^k so that virtual indices reach past 2^25 and raw cells past 2^26"""
    n = 1 << k
    bps = [n - 3 - 2 * j for j in range(A - 1)]
    return sum(bps) + n - 11, bps


def test_copies_pair_keys_that_differ_in_one_byte(torch, ctx, lib):
    """advice equalities whose endpoints (>= 2^24) differ in a single byte of a or of b: the sort passes over that byte only"""
    rng = np.random.default_rng(11)
    k, A = 22, 9
    N, bps = _wide_layout(k, A)
    for side in (0, 1):
        for byte in range(4):
            m = 3000
            base = np.array([(1 << 24) + 0x123456, (1 << 24) + 0x0ABCDE], dtype=np.uint64)
            pr = np.tile(base, (m, 1))
            digits = rng.integers(0, 2 if byte == 3 else 256, m).astype(np.uint64)
            pr[:, side] = (pr[:, side] & ~np.uint64(0xFF << (8 * byte))) | (digits << np.uint64(8 * byte))
            assert (pr < N).all() and len(np.unique(pr[:, side] >> np.uint64(8 * byte) & np.uint64(0xFF))) > 1
            _check_copies(torch, ctx, lib, N, bps, k, 1, A, pairs=pr)
    # endpoints differing anywhere, with break copies and lookups before them
    pr = rng.integers(0, N, size=(70_000, 2)).astype(np.uint64)
    lk = rng.integers(0, N, size=5000).astype(np.uint64)
    _check_copies(torch, ctx, lib, N, bps, k, 2, A, L=3, lookups=lk, pairs=pr)


def _const_variants(rng):
    """canonical constants that differ only in byte 0, only in byte 31 (up to r - 1), only in limb 1 or only in limb 2"""
    top = (R - 1) >> 248
    low = (R - 1) & ((1 << 248) - 1)
    mid = 0x1111222233334444 | 0x5555666677778888 << 64 | 0x0999AAAABBBBCCCC << 128 | 0x0102030405060708 << 192
    return {
        "byte0": [(mid & ~0xFF) | int(d) for d in rng.integers(0, 256, 40)],
        "byte31": [low + (int(d) << 248) for d in rng.integers(0, top + 1, 40)] + [R - 1, low + (top << 248)],
        "limb1": [(mid & ~(((1 << 64) - 1) << 64)) | int(d) << 64 for d in rng.integers(0, 1 << 62, 40, dtype=np.int64)],
        "limb2": [(mid & ~(((1 << 64) - 1) << 128)) | int(d) << 128 for d in rng.integers(0, 1 << 62, 40, dtype=np.int64)],
    }


@pytest.mark.parametrize("variant", ["byte0", "byte31", "limb1", "limb2"])
def test_copies_constants_that_differ_in_one_place(torch, ctx, lib, variant):
    rng = np.random.default_rng(31)
    k, A, F = 8, 3, 2
    bps = [200, 180]
    N = sum(bps) + 150
    vals = _const_variants(rng)[variant]
    assert all(0 <= v < R for v in vals)
    m = 3000  # each value many times, at random cells
    consts = [vals[i] for i in rng.integers(0, len(vals), m)]
    cidx = rng.integers(0, N, m).astype(np.uint64)
    _check_copies(torch, ctx, lib, N, bps, k, F, A, consts=consts, cidx=cidx)


@pytest.mark.parametrize("values", [1, 2, 5])
def test_copies_equal_constants_in_descending_cell_order(torch, ctx, lib, values):
    """the second sort (by constant) keeps the first one's order (by cell) among equal constants: ties come out by ascending
    cell although the builder supplies them descending"""
    rng = np.random.default_rng(values)
    k, A, F = 12, 2, 1
    bps = [4000]
    N = 4000 + 4000
    m = 6000
    cidx = np.sort(rng.choice(N, size=m, replace=False))[::-1].astype(np.uint64)
    pool = [7 + 1000003 * i for i in range(values)]
    consts = [pool[i] for i in rng.integers(0, values, m)]
    want = _check_copies(torch, ctx, lib, N, bps, k, F, A, consts=consts, cidx=cidx)
    c_edges = want[0][len(bps):]
    for v in range(values):  # the run of each constant: ascending raw cells
        run = c_edges[c_edges[:, 0] == v][:, 1].astype(np.int64)
        assert len(run) > 1 and (np.diff(run) > 0).all()


@pytest.mark.parametrize("F,extra", [(F, x) for F in (0, 1, 3) for x in (-1, 0, 1) if F or x >= 0])
def test_copies_distinct_constants_at_the_row_limit(torch, ctx, lib, F, extra):
    """D = F 2^k + extra distinct constants: status[1] = D; ranks >= F 2^k get no row and write nothing"""
    k, A = 3, 2
    n = 1 << k
    D = F * n + extra
    rng = np.random.default_rng(F * 10 + extra + 1)
    bps = [5]
    N = 5 + 7
    vals = rng.choice(1 << 40, size=D, replace=False).tolist()
    consts = vals + [vals[i] for i in rng.integers(0, D, 2 * D)] if D else []
    cidx = rng.integers(0, N, len(consts)).astype(np.uint64)
    want = _check_copies(torch, ctx, lib, N, bps, k, F, A, consts=consts, cidx=cidx)
    assert want[2][1] == D


@pytest.mark.parametrize("M,Mc", [(5, (1 << 17) + 3), ((1 << 17) + 3, 5), (0, 300), (300, 0), (1, 1)])
def test_copies_unbalanced_pairs_and_constants(torch, ctx, lib, M, Mc):
    """both sorts run on the grid sized for the larger one: the smaller one has more CTAs than tiles"""
    rng = np.random.default_rng(M + Mc)
    k, A, F = 16, 4, 2
    bps = [60000, 61000, 59000]
    N = sum(bps) + 50000
    pr = rng.integers(0, N, size=(M, 2)).astype(np.uint64)
    vals = rng.integers(0, 1 << 62, 1000).tolist() + [R - 1, R - 2, 0]
    consts = [vals[i] for i in rng.integers(0, len(vals), Mc)]
    cidx = rng.integers(0, N, Mc).astype(np.uint64)
    _check_copies(torch, ctx, lib, N, bps, k, F, A, pairs=pr, consts=consts, cidx=cidx)


def test_copies_indices_out_of_range_set_the_status(torch, ctx, lib):
    rng = np.random.default_rng(77)
    k, A, F, L = 8, 3, 1, 2
    bps = [250, 240]
    N = 490 + 200
    lk = rng.integers(0, N, 300).astype(np.uint64)
    pr = rng.integers(0, N, size=(400, 2)).astype(np.uint64)
    consts = rng.integers(1, 50, 300).tolist()
    cidx = rng.integers(0, N, 300).astype(np.uint64)
    base = dict(L=L, lookups=lk, pairs=pr, consts=consts, cidx=cidx)
    assert _check_copies(torch, ctx, lib, N, bps, k, F, A, **base)[2][0] == 0
    lk2 = lk.copy(); lk2[[0, 299]] = [N, 1 << 40]
    assert _check_copies(torch, ctx, lib, N, bps, k, F, A, **dict(base, lookups=lk2))[2][0] == 1
    pr2 = pr.copy(); pr2[5, 1] = N; pr2[17, 0] = N + 3
    assert _check_copies(torch, ctx, lib, N, bps, k, F, A, **dict(base, pairs=pr2))[2][0] == 2
    ci2 = cidx.copy(); ci2[[3, 4]] = [N, (1 << 64) - 1]
    assert _check_copies(torch, ctx, lib, N, bps, k, F, A, **dict(base, cidx=ci2))[2][0] == 2
    assert _check_copies(torch, ctx, lib, N, bps, k, F, A, **dict(base, lookups=lk2, pairs=pr2, cidx=ci2))[2][0] == 3


# ------------------------------------------------------------------------------------------------------- instance edges
def test_instance_edges_past_the_usable_rows(torch, ctx, lib):
    """rows >= usable are written (0, 0) and set bit 1; an index >= N at a row <= usable sets bit 0"""
    rng = np.random.default_rng(12)
    k, F, A, L = 5, 2, 3, 1
    n = 1 << k
    usable = n - 7
    bps = [30, 29]
    N = 59 + 20
    n_index = [usable + 3, 5, 0, usable, usable + 1]
    cols = [rng.integers(0, N, m).astype(np.uint64) for m in n_index]
    cols[0][[usable, usable + 2]] = [N, N + 1]  # row == usable: bit 0; row > usable: no bit 0
    cols[1][3] = N                              # row < usable: bit 0
    cols[3][usable - 1] = 1 << 63
    cols[4][usable] = N
    want_e, want_s = [], []
    ends = np.cumsum(bps)
    starts = np.concatenate([[0], ends])
    for m, col in enumerate(cols):
        s = 0
        for r, p in enumerate(col.tolist()):
            if p >= N and r <= usable:
                s |= 1
            if r >= usable:
                s |= 2
            if p < N and r < usable:
                j = int(np.searchsorted(ends, p, side="left"))
                want_e.append(((F + j) * n + p - int(starts[j]), (F + A + L + m) * n + r))
            else:
                want_e.append((0, 0))
        want_s.append(s)
    assert want_s == [3, 1, 0, 1, 3]
    I, E = len(cols), sum(n_index)
    d_i = _dev(torch, np.concatenate(cols), np.uint64)
    d_e = torch.full(((E + 64) * 2,), -1, dtype=torch.int32, device="cuda")
    d_st = torch.full((I + 2,), -1, dtype=torch.int32, device="cuda")
    nix = (C.c_size_t * I)(*n_index)
    bps_h = np.array(bps, dtype=np.uint64)
    ctx.check(lib.h2b_keygen_instance_edges_nf_dev(ctx.h, N, vp(bps_h.ctypes.data), len(bps), k, F, A, L, usable, I, nix, _ptr(d_i),
                                                   _ptr(d_e), _ptr(d_st)))
    e = _host(d_e, np.uint32).reshape(-1, 2)
    st = _host(d_st, np.uint32)
    assert np.array_equal(e[:E], np.array(want_e, dtype=np.uint32)) and (e[E:] == 0xFFFFFFFF).all()
    assert st[:I].tolist() == want_s and (st[I:] == 0xFFFFFFFF).all()

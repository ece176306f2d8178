"""GPU tests of halo2_lib_b200.keygen (include/h2b200_keygen.hpp, csrc/keygen.cu), keygen of a halo2-base builder on the
device: its break points equal MockProver's, its fixed columns (q_j, q_lookup, table, c) the ones the oracle's layout gives,
its sigma bit for bit the mapping of halo2's permutation Assembly on halo2-base's copy calls (tests/keygen_oracle.py:
Python at small k, C at full size), its coefficient / extended forms those of a Circuit built from the downloaded columns,
its vk each column's commit_lagrange; on builders that stress the spanning forest; end to end, a ProverSession on the keygen
circuit gives the same proof bytes and check reports as one on the circuit built from the downloaded columns; halo2-base's
panics raise its messages and leave the context usable."""
import numpy as np
import pytest
from oracle import pyref
from util import mont, rand_ints, affine_to_limbs
import builder_oracle as bo
import keygen_oracle as ko

pytestmark = pytest.mark.gpu
R = pyref.R
SHAPES = [(1, 0, True), (3, 2, False), (2, 0, False), (2, 1, True)]


@pytest.fixture(scope="module")
def h2b():
    import halo2_lib_b200 as h
    return h


@pytest.fixture(scope="module")
def ctx(h2b):
    c = h2b.Context(0)
    yield c
    c.close()


_params = {}


@pytest.fixture(scope="module", autouse=True)
def _close_params(ctx):
    yield
    for p in _params.values():
        p.close()
    _params.clear()


def _params_for(ctx, h2b, k):
    if k not in _params:
        n = 1 << k
        g = affine_to_limbs([pyref.G1])[0]
        bm = ctx.g1_fixed_base_mul(g, mont([3 + 5 * i for i in range(n)], R))
        bl = ctx.g1_fixed_base_mul(g, mont([7 + 11 * i for i in range(n)], R))
        _params[k] = h2b.ParamsKZG(ctx, k, g=bm, g_lagrange=bl)
    return _params[k]


def _mont_small(ctx, v):
    v = np.ascontiguousarray(v, dtype=np.uint64)
    z = np.zeros(len(v), dtype=np.uint64)
    return ctx.field_op(1, 5, np.stack([v, z, z, z], axis=1)) if len(v) else np.zeros((0, 4), dtype=np.uint64)


def _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, **kw):
    return h2b.keygen(ctx, _params_for(ctx, h2b, k), k, A, L, sel, bits, max_rows, b["selectors"], b["advice_equalities"],
                      (_mont_small(ctx, b["constants"]), b["constant_index"]), b["lookups"], **kw)


def _want_fixed(k, A, L, sel, bits, max_rows, b):
    """q_j, q_lookup, table and c from builder_oracle's layout"""
    n = 1 << k
    lay = bo.run(k, A, L, sel, bits, max_rows, b, np.zeros(len(b["selectors"]), dtype=np.uint64), gate_rows={}, record=False)
    one = mont([1], R)[0]
    fixed = {}
    for j in range(A):
        q = np.zeros((n, 4), dtype=np.uint64)
        q[sorted(lay["q"][j])] = one
        fixed["q%d" % j] = q
    if L == 0 and sel:
        ql = np.zeros((n, 4), dtype=np.uint64)
        ql[sorted(lay["q_lookup"] or ())] = one
        fixed["q_lookup"] = ql
    if L or sel:
        t = np.zeros((n, 4), dtype=np.uint64)
        t[: 1 << bits] = mont(list(range(1 << bits)), R)
        fixed["table"] = t
    c = np.zeros((n, 4), dtype=np.uint64)
    rows = bo.assign_constants(zip(b["constants"], b["constant_index"]), n - 7, k)
    if rows:
        c[list(rows.values())] = mont(list(rows.keys()), R)
    fixed["c"] = c
    return fixed, lay["break_points"]


def _sigma_map(cs):
    return cs.sigma_map.download().view(np.uint32).reshape(-1)[: len(cs.perm_cols) << cs.k]


def _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, oracle="python", values=True, forms=True):
    cs, vk, bps = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b)
    fixed, want_bps = _want_fixed(k, A, L, sel, bits, max_rows, b)
    assert bps == want_bps
    assert cs.fixed_names == list(fixed)
    got_fixed = {nm: cs.lagr[nm].download() for nm in cs.fixed_names}
    for nm in fixed:
        assert np.array_equal(got_fixed[nm], fixed[nm]), nm
    pairs, _, _ = ko.copy_sequence(k, A, L, max_rows, b)
    V = (1 + A + L) << k
    want_map = ko.assembly(V, pairs) if oracle == "python" else ko.assembly_c(V, pairs)
    assert np.array_equal(_sigma_map(cs), want_map)
    sigma = [cs.lagr[nm].download() for nm in cs.sigma_names]
    if values:
        assert np.array_equal(np.stack(sigma), ko.sigma_values(want_map, 1 + A + L, k))
    if forms:  # the proving key's forms: the existing constructor on the downloaded columns
        ref = h2b.Circuit(ctx, k, got_fixed, sigma, A=A, L=L, selector_lookup=sel)
        for nm in cs.fixed_names + cs.sigma_names:
            for table in ("coeff", "ext"):
                assert np.array_equal(getattr(cs, table)[nm].download(), getattr(ref, table)[nm].download()), (table, nm)
        ref.free()
        params = _params_for(ctx, h2b, k)
        for nm, col in list(got_fixed.items()) + list(zip(cs.sigma_names, sigma)):
            want = h2b.prover.g1_normalize_host(params.commit_lagrange(col))
            got = vk["fixed"][nm] if nm in vk["fixed"] else vk["permutation"][cs.sigma_names.index(nm)]
            assert np.array_equal(got, want), nm
    return cs, vk, bps, sigma


@pytest.mark.parametrize("k", [8, 12])
@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_keygen_matches_the_oracle(ctx, h2b, k, A, L, sel):
    rng = np.random.default_rng(700 + k + 10 * A + L)
    bits = min(8, k - 2)
    max_rows = (1 << k) - 9
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, contexts=3)
    cs, vk, bps, sigma = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b)
    # a second run gives the same bytes
    cs2, vk2, bps2 = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b)
    assert bps2 == bps
    for nm in cs.fixed_names + cs.sigma_names:
        for table in ("lagr", "coeff", "ext"):
            assert np.array_equal(getattr(cs, table)[nm].download(), getattr(cs2, table)[nm].download())
    assert all(np.array_equal(vk["fixed"][nm], vk2["fixed"][nm]) for nm in vk["fixed"])
    assert all(np.array_equal(x, y) for x, y in zip(vk["permutation"], vk2["permutation"]))
    cs.free(); cs2.free()


@pytest.mark.parametrize("k,A,L,sel,bits", [(19, 1, 0, True, 18), (19, 1, 0, False, 18), (20, 11, 2, False, 19)])
def test_keygen_at_full_size(ctx, h2b, k, A, L, sel, bits):
    """sigma against the C Assembly; its values at sampled cells against Python integers"""
    rng = np.random.default_rng(k + A)
    max_rows = (1 << k) - 9
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
    cs, vk, bps, sigma = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, oracle="c", values=False, forms=False)
    m = _sigma_map(cs)
    pick = rng.choice(len(m), size=2000, replace=False)
    w = pyref.omega_for(k)
    flat = np.concatenate(sigma)
    for x in pick.tolist():
        c, r = int(m[x]) >> k, int(m[x]) & ((1 << k) - 1)
        assert np.array_equal(flat[x], mont([pow(pyref.DELTA, c, R) * pow(w, r, R) % R], R)[0])
    cs.free()


def _stress_builder(rng, k, A, L, max_rows):
    """make_builder plus the equalities that stress the forest: duplicate, reversed and self equalities, equalities that
    close cycles, break cells and looked-up cells inside equalities"""
    b = bo.make_builder(rng, k, A, L, False, 6, max_rows)
    N = len(b["selectors"])
    E = b["advice_equalities"]
    bps = bo.assign_with_constraints(b["contexts"], A, max_rows, record=False)[0]
    brk = np.cumsum(bps).astype(np.uint64)
    extra = [E[:20], E[:20][:, ::-1], np.stack([E[:10, 0], E[:10, 0]], axis=1)]
    ring = rng.choice(N, size=30, replace=False).astype(np.uint64)
    extra.append(np.stack([ring, np.roll(ring, 1)], axis=1))                           # a cycle
    if len(brk):
        extra.append(np.stack([brk, rng.choice(N, size=len(brk)).astype(np.uint64)], axis=1))  # break cells
    lk = b["lookups"][: 40]
    extra.append(np.stack([lk, rng.choice(N, size=len(lk)).astype(np.uint64)], axis=1))    # looked-up cells
    return dict(b, advice_equalities=np.concatenate([E] + extra).astype(np.uint64))


@pytest.mark.parametrize("A,L", [(3, 2), (2, 0)])
def test_keygen_on_builders_that_stress_the_forest(ctx, h2b, A, L):
    k = 10
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(31 + A)
    b = _stress_builder(rng, k, A, L, max_rows)
    cs, _, _, _ = _check_keygen(ctx, h2b, k, A, L, False, 6, max_rows, b)
    m = _sigma_map(cs)
    # the builder's order of its equalities does not change the keys
    perm, cperm = rng.permutation(len(b["advice_equalities"])), rng.permutation(len(b["constants"]))
    sh = dict(b, advice_equalities=b["advice_equalities"][perm], constants=b["constants"][cperm], constant_index=b["constant_index"][cperm])
    cs2, _, _ = _keygen(ctx, h2b, k, A, L, False, 6, max_rows, sh)
    assert np.array_equal(_sigma_map(cs2), m)
    for nm in cs.sigma_names + cs.fixed_names:
        assert np.array_equal(cs.lagr[nm].download(), cs2.lagr[nm].download())
    cs.free(); cs2.free()


def test_keygen_with_a_constant_tied_to_many_cells(ctx, h2b):
    k, A, L = 17, 1, 0
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(5)
    b = bo.make_builder(rng, k, A, L, False, 8, max_rows)
    N = len(b["selectors"])
    tied = rng.choice(N, size=110_000, replace=False).astype(np.uint64)
    b = dict(b, lookups=np.zeros(0, dtype=np.uint64), constants=np.concatenate([b["constants"], np.full(len(tied), 12345, dtype=np.uint64)]),
             constant_index=np.concatenate([b["constant_index"], tied]))
    cs, _, _, _ = _check_keygen(ctx, h2b, k, A, L, False, 8, max_rows, b, oracle="c", values=False, forms=False)
    cs.free()


def test_a_session_on_the_keygen_circuit(ctx, h2b):
    """the same proof bytes and check reports as the circuit built from the downloaded columns; MockProver's verdicts"""
    k, bits = 10, 6
    for A, L, sel in SHAPES:
        max_rows = (1 << k) - 9
        rng = np.random.default_rng(90 + A + L)
        b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
        cs, _, bps, sigma = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, values=False, forms=False)
        ref = h2b.Circuit(ctx, k, {nm: cs.lagr[nm].download() for nm in cs.fixed_names}, sigma, A=A, L=L, selector_lookup=sel)
        params = _params_for(ctx, h2b, k)
        rnd = mont(rand_ints(rng, 1 << k, R), R)
        mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows)
        lk = np.ascontiguousarray(b["lookups"] if L else np.zeros(0, dtype=np.uint64))
        proofs = []
        for circuit in (cs, ref):
            sess = h2b.ProverSession(ctx, params, circuit)
            cells = _mont_small(ctx, b["values"])
            draws = np.random.default_rng(1)
            sess.blind_source = lambda rows: mont(rand_ints(draws, rows, R), R)
            kw = dict(break_points=np.array(bps, dtype=np.uint64), lookup_index_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))
            proofs.append(sess.prove(cells.ctypes.data, len(cells), rnd.ctypes.data, **kw))
            assert sess.check(cells.ctypes.data, len(cells), **kw)["satisfied"]
            v = bo.plant(np.random.default_rng(3), b, bits)
            bad = _mont_small(ctx, v)
            chk = sess.check(bad.ctypes.data, len(bad), **kw)
            got = mp.run(bad, b["selectors"], b["advice_equalities"], (_mont_small(ctx, b["constants"]), b["constant_index"]), b["lookups"])
            assert chk["gates"] == got["gates"] and chk["lookups"] == got["lookups"]
            assert (sum(c for c, _ in chk["copies"]) > 0) == (got["equalities"][0] + got["constants"][0] > 0)
            sess.free()
        a, r = proofs
        assert all(np.array_equal(x, y) for x, y in zip(a["commitments"], r["commitments"]))
        assert all(np.array_equal(a["evals"][q], r["evals"][q]) for q in a["evals"]) and a["challenges"] == r["challenges"]
        mp.free(); ref.free(); cs.free()


def test_errors_carry_halo2_base_messages_and_leave_the_context_usable(ctx, h2b):
    rng = np.random.default_rng(3)
    k, bits = 8, 4
    max_rows = (1 << k) - 9
    b = bo.make_builder(rng, k, 2, 1, False, bits, max_rows)

    def expect(msg, A=2, L=1, **changes):
        with pytest.raises(h2b.H2BError, match=msg):
            _keygen(ctx, h2b, k, A, L, False, bits, max_rows, dict(b, **changes))
        cs = _keygen(ctx, h2b, k, 2, 1, False, bits, max_rows, b)[0]
        cs.free()

    expect("NOT ENOUGH ADVICE COLUMNS", A=1)
    s = np.zeros_like(b["selectors"])
    s[max_rows - 3] = s[max_rows - 4] = 1
    expect("We do not support overlaps with delta = 1", selectors=s)
    s[max_rows - 4], s[max_rows - 5] = 0, 1
    expect("We do not support overlaps with delta = 2", selectors=s)
    expect("range lookups would be assigned to unusable rows", lookups=np.arange(max_rows + 1, dtype=np.uint64))
    N = len(b["selectors"])
    e = b["advice_equalities"].copy()
    e[7, 1] = N
    expect("virtual cell not assigned", advice_equalities=e)
    ci = b["constant_index"].copy()
    ci[-1] = N + 5
    expect("virtual cell not assigned", constant_index=ci)
    expect("virtual cell not assigned", lookups=np.concatenate([b["lookups"][:5], [N]]).astype(np.uint64))
    u = (1 << k) - 7
    expect(r"NotEnoughRowsAvailable \{ current_k: 8 \}", constants=np.arange(u + 1, dtype=np.uint64), constant_index=np.zeros(u + 1, dtype=np.uint64))
    expect("range lookups require lookup advice columns", L=0)

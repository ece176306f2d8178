"""GPU tests of several constants columns (BaseCircuitParams::num_fixed = F, F >= 0) for halo2-base builders: keygen places the
distinct constants left to right, then top to bottom over c, c1.. and builds sigma as halo2's Assembly does (tests/constants_oracle.py),
the resident prover proves the quotient identity with the constants columns in the permutation, check and MockProver report a
broken constant of c1 where halo2 would, the capacity panics carry halo2's and halo2-base's texts, and F = 1 gives the bytes
the calls without F give."""
import os
import subprocess
import numpy as np
import pytest
from oracle import pyref
from util import mont, unmont, rand_ints, affine_to_limbs
import builder_oracle as bo
import keygen_oracle as ko
import constants_oracle as co

pytestmark = pytest.mark.gpu
R = pyref.R
SHAPES = [(1, 0, True), (3, 2, False), (2, 0, False), (2, 1, True)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def _builder(rng, k, A, L, sel, bits, max_rows, F, fill=1.0, extra=True):
    """builder_oracle.make_builder; with `extra`, duplicated constant equalities and cells tied to a second constant; F = 0:
    no constants at all"""
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, fill=fill)
    if F == 0:
        return dict(b, constants=np.zeros(0, dtype=np.uint64), constant_index=np.zeros(0, dtype=np.uint64))
    if not extra:
        return b
    m, N = len(b["constants"]), len(b["selectors"])
    dup = rng.choice(m, size=min(m, 6), replace=False)
    cells = rng.choice(N, size=6, replace=False).astype(np.uint64)
    extra_c = np.concatenate([b["constants"][dup], rng.integers(2, 1 << 40, size=6, dtype=np.int64).astype(np.uint64)])
    return dict(b, constants=np.concatenate([b["constants"], extra_c]),
                constant_index=np.concatenate([b["constant_index"], b["constant_index"][dup], cells]))


def _consts(ctx, b):
    return (_mont_small(ctx, b["constants"]), b["constant_index"])


def _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, **kw):
    return h2b.keygen(ctx, _params_for(ctx, h2b, k), k, A, L, sel, bits, max_rows, b["selectors"], b["advice_equalities"], _consts(ctx, b),
                      b["lookups"], **kw)


def _instances(rng, b, I, count):
    return [rng.choice(len(b["selectors"]), size=count).astype(np.uint64) for _ in range(I)]


def _sigma_of(mapping, k, cells):
    """delta^c' omega^r' (canonical) of the mapping at the given flat cells"""
    w = pyref.omega_for(k)
    return [pow(pyref.DELTA, int(mapping[x]) >> k, R) * pow(w, int(mapping[x]) & ((1 << k) - 1), R) % R for x in cells]


def _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, F, inst=(), oracle="python", sample=None):
    """keygen with F constants columns against the oracles: sigma map, c columns, every vk commitment, repeatability"""
    I = len(inst)
    kw = dict(F=F, I=I, instances=list(inst) if I else None)
    cs, vk, bps = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, **kw)
    pairs, cells, want_bps = co.copy_sequence(k, A, L, max_rows, b, F, list(inst))
    assert bps == want_bps
    assert cs.F == F and cs.I == I and cs.const_names == co.const_names(F)
    assert cs.perm_cols == co.const_names(F) + cs.adv_names + ["i%d" % m for m in range(I)]
    assert cs.fixed_names[len(cs.fixed_names) - F:] == co.const_names(F)
    npc = F + A + L + I
    V = npc << k
    want = ko.assembly(V, pairs) if oracle == "python" else ko.assembly_c(V, pairs)
    got = cs.sigma_map.download().view(np.uint32).reshape(-1)[:V]
    assert np.array_equal(got, want)
    for nm, col in zip(co.const_names(F), co.const_columns(k, F, cells)):
        assert unmont(cs.lagr[nm].download(), R) == col, nm
    if sample is None:
        sigma = [cs.lagr[nm].download() for nm in cs.sigma_names]
        assert np.array_equal(np.stack(sigma), ko.sigma_values(want, npc, k))
        params = _params_for(ctx, h2b, k)
        for nm in cs.fixed_names:
            assert np.array_equal(vk["fixed"][nm], h2b.prover.g1_normalize_host(params.commit_lagrange(cs.lagr[nm].download()))), nm
        for c in range(npc):
            assert np.array_equal(vk["permutation"][c], h2b.prover.g1_normalize_host(params.commit_lagrange(sigma[c]))), c
    else:  # sigma values on sampled cells
        n = 1 << k
        xs = np.random.default_rng(k).choice(V, size=sample, replace=False)
        got_v = [unmont(cs.lagr[cs.sigma_names[int(x) >> k]].download(int(x) & (n - 1), 1), R)[0] for x in xs]
        assert got_v == _sigma_of(want, k, xs)
    assert len(vk["permutation"]) == npc and list(vk["fixed"]) == cs.fixed_names
    return cs, vk, bps


def _same_keys(a, b):
    assert list(a["fixed"]) == list(b["fixed"]) and all(np.array_equal(a["fixed"][nm], b["fixed"][nm]) for nm in a["fixed"])
    assert len(a["permutation"]) == len(b["permutation"]) and all(np.array_equal(x, y) for x, y in zip(a["permutation"], b["permutation"]))


@pytest.mark.parametrize("I", [0, 1])
@pytest.mark.parametrize("F", [0, 2, 3, 7])
@pytest.mark.parametrize("k", [8, 12])
@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_keygen_with_constants_columns_matches_the_assembly(ctx, h2b, A, L, sel, k, F, I):
    rng = np.random.default_rng(600 + k + 10 * A + L + 3 * F + I)
    bits = min(8, k - 2)
    max_rows = (1 << k) - 9
    b = _builder(rng, k, A, L, sel, bits, max_rows, F)
    inst = _instances(rng, b, I, 12)
    cs, vk, bps = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, F, inst)
    cs2, vk2, bps2 = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, F=F, I=I, instances=inst if I else None)
    assert bps2 == bps
    _same_keys(vk, vk2)
    assert all(np.array_equal(cs.lagr[nm].download(), cs2.lagr[nm].download()) for nm in cs.fixed_names + cs.sigma_names)
    cs.free(); cs2.free()


def _prove(ctx, h2b, cs, k, b, bps, L, rnd, public=None, draws_seed=1, cells=None):
    sess = h2b.ProverSession(ctx, _params_for(ctx, h2b, k), cs)
    cells = _mont_small(ctx, b["values"]) if cells is None else cells
    draws = np.random.default_rng(draws_seed)
    sess.blind_source = lambda rows: mont(rand_ints(draws, rows, R), R)
    lk = np.ascontiguousarray(b["lookups"] if L else np.zeros(0, dtype=np.uint64))
    kw = dict(break_points=np.array(bps, dtype=np.uint64), lookup_index_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))
    res = sess.prove(cells.ctypes.data, len(cells), rnd.ctypes.data, instances=public, **kw)
    chk = sess.check(cells.ctypes.data, len(cells), instances=public, **kw)
    return sess, res, chk


def _public(ctx, b, inst):
    return [_mont_small(ctx, b["values"][idx.astype(np.int64)]) for idx in inst]


# halo2-ecc's bench configurations that need several constants columns (bench_fixed_msm.config, bench_ecdsa.config):
# (k, num_advice, num_lookup_advice, num_fixed, lookup_bits)
ECC_SHAPES = [(19, 20, 2, 2, 18), (17, 83, 9, 7, 16), (12, 139, 24, 2, 11)]


@pytest.mark.parametrize("k,A,L,F,bits", ECC_SHAPES)
def test_halo2_ecc_shapes(ctx, h2b, k, A, L, F, bits):
    """keygen against the C Assembly (sigma values on 2000 sampled cells), then a proof that satisfies the quotient identity"""
    rng = np.random.default_rng(k + A)
    max_rows = (1 << k) - 9
    b = _builder(rng, k, A, L, False, bits, max_rows, F, extra=False)
    cs, _, bps = _check_keygen(ctx, h2b, k, A, L, False, bits, max_rows, b, F, oracle="c", sample=2000)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    sess, res, chk = _prove(ctx, h2b, cs, k, b, bps, L, rnd)
    assert chk["satisfied"], {key: [x for x in v if x[0]] for key, v in chk.items() if key != "satisfied"}
    left, right = co.quotient_identity(res, k, A, L, False, F)
    assert left == right
    sess.free(); cs.free()


@pytest.mark.parametrize("F", [0, 2, 3])
@pytest.mark.parametrize("A,L,sel,I", [(1, 0, True, 0), (3, 2, False, 1), (2, 1, True, 1)])
def test_proofs_on_keygen_circuits(ctx, h2b, A, L, sel, I, F):
    k, bits = 12, 8
    rng = np.random.default_rng(700 + 10 * A + L + F + I)
    max_rows = (1 << k) - 9
    b = _builder(rng, k, A, L, sel, bits, max_rows, F, fill=0.7, extra=False)
    inst = _instances(rng, b, I, 16)
    cs, _, bps = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, F, inst, sample=500)
    public = _public(ctx, b, inst) if I else None
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    sess, res, chk = _prove(ctx, h2b, cs, k, b, bps, L, rnd, public)
    assert chk["satisfied"] and len(chk["copies"]) == F + A + L + I
    left, right = co.quotient_identity(res, k, A, L, sel, F, [unmont(p, R) for p in public or []])
    assert left == right
    sess.free(); cs.free()


@pytest.mark.parametrize("F,I", [(0, 0), (2, 1)])
def test_proof_matches_the_oracle_prover(ctx, h2b, F, I):
    """a proof on a keygen circuit at k = 8 with F constants columns, fixed blinding rows: every commitment, evaluation and
    challenge the bytes of constants_oracle.create_proof (Python integers)"""
    import test_oracle_prover as top
    from oracle import prover_ref
    k, A, L, sel, bits = 8, 2, 1, False, 6
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(51 + F)
    b = _builder(rng, k, A, L, sel, bits, max_rows, F, fill=0.5, extra=False)
    inst = _instances(rng, b, I, 5)
    cs, _, bps = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, F, inst, sample=100)
    public = _public(ctx, b, inst) if I else None
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    sess, res, _ = _prove(ctx, h2b, cs, k, b, bps, L, rnd, public)
    draws = np.random.default_rng(1)
    blind = lambda rows: rand_ints(draws, rows, R)
    want = co.create_proof(k, A, L, sel, F, {nm: unmont(cs.lagr[nm].download(), R) for nm in cs.fixed_names},
                           [unmont(cs.lagr[nm].download(), R) for nm in cs.sigma_names], [int(v) for v in b["values"]], list(bps),
                           [int(b["values"][int(i)]) for i in b["lookups"]], unmont(rnd, R), blind,
                           top.small_bases(1 << k, 3, 5), top.small_bases(1 << k, 7, 11), instances=[unmont(p, R) for p in public or []])
    assert res["challenges"] == want["challenges"]
    assert [np.asarray(c, dtype=np.uint64).tobytes() for c in res["commitments"]] == want["commitments"]
    assert [(nm, r) for nm, r in res["evals"]] == [(nm, r) for nm, r, _ in want["evals"]]
    assert [np.asarray(v, dtype=np.uint64).tobytes() for v in res["evals"].values()] == [prover_ref.fr_bytes(v) for _, _, v in want["evals"]]
    sess.free(); cs.free()


def _broken_c1(b, cells, k):
    """values with the cell of one constant equality of column c1 changed, and that equality's index"""
    n = 1 << k
    i = next(i for i, c in enumerate(b["constants"].tolist()) if cells[int(c)] // n == 1)
    v = b["values"].copy()
    v[int(b["constant_index"][i])] += 1
    return v, i


def test_a_broken_constant_in_c1(ctx, h2b):
    k, A, L, sel, bits, F = 8, 2, 1, True, 6, 3
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(61)
    b = _builder(rng, k, A, L, sel, bits, max_rows, F, fill=0.6, extra=False)
    cs, _, bps = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, F)
    _, cells, _ = co.copy_sequence(k, A, L, max_rows, b, F)
    vals, i = _broken_c1(b, cells, k)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    sess, res, chk = _prove(ctx, h2b, cs, k, b, bps, L, rnd, cells=_mont_small(ctx, vals))
    c_cols = [unmont(cs.lagr[nm].download(), R) for nm in cs.const_names]
    cols = [unmont(sess.lagr[nm].download(), R) for nm in cs.adv_names]
    sigma = [unmont(cs.lagr[nm].download(), R) for nm in cs.sigma_names]
    want = co.check(k, F, c_cols, sigma, cols)
    assert not chk["satisfied"] and chk["copies"] == want and sum(c for c, _ in want) == 2
    mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows, F=F)
    got = mp.run(_mont_small(ctx, vals), b["selectors"], b["advice_equalities"], _consts(ctx, b), b["lookups"])
    ref = co.mock_run(k, A, L, sel, bits, max_rows, b, vals, F)
    assert got["constants"] == ref["constants"] and i in got["constants"][1]
    assert got["constant_cells"] == ref["constant_cells"] and not got["satisfied"]
    assert got["distinct_constants"] == ref["distinct_constants"] == len(cells)
    mp.free(); sess.free(); cs.free()


def test_capacity_errors_carry_halo2_messages_and_leave_the_context_usable(ctx, h2b):
    k, A, L, sel, bits = 8, 2, 0, False, 4
    max_rows = (1 << k) - 9
    u = (1 << k) - 7
    rng = np.random.default_rng(71)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, fill=0.5)
    N = len(b["selectors"])
    cells = _mont_small(ctx, b["values"])
    args = lambda bb: (cells, bb["selectors"], bb["advice_equalities"], _consts(ctx, bb), bb["lookups"])

    def with_distinct(D):
        return dict(b, constants=np.arange(10, 10 + D, dtype=np.uint64), constant_index=(np.arange(D) % N).astype(np.uint64))

    def ok(F):
        cs, _, _ = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, F=F)
        cs.free()
        mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows, F=F)
        assert mp.run(*args(b))["satisfied"]
        mp.free()
    for F in (1, 2, 3):
        full, over = with_distinct(F * u), with_distinct(F * u + 1)
        cs, _, _ = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, full, F, sample=200)
        cs.free()
        mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows, F=F)
        assert mp.run(*args(full))["distinct_constants"] == F * u
        for call in (lambda: _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, over, F=F), lambda: mp.run(*args(over))):
            with pytest.raises(h2b.H2BError, match=r"NotEnoughRowsAvailable \{ current_k: 8 \}: %d distinct constants for the %d usable cells"
                                                   % (F * u + 1, F * u)):
                call()
            ok(F)
        mp.free()
    none = dict(b, constants=np.zeros(0, dtype=np.uint64), constant_index=np.zeros(0, dtype=np.uint64))
    mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows, F=0)
    for call in (lambda: _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, F=0), lambda: mp.run(*args(b))):
        with pytest.raises(h2b.H2BError, match="index out of bounds: the len is 0 but the index is 0"):
            call()
        cs, _, _ = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, none, F=0)
        assert cs.const_names == [] and cs.perm_cols[0] == "a0"
        cs.free()
    res = mp.run(*args(none))
    assert res["satisfied"] and res["distinct_constants"] == 0
    mp.free()


def test_one_constants_column_gives_the_existing_bytes(ctx, h2b):
    k, A, L, sel, bits = 8, 2, 1, False, 6
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(81)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    out = []
    for kw in ({}, dict(F=1)):
        cs, vk, bps = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, **kw)
        sess, res, chk = _prove(ctx, h2b, cs, k, b, bps, L, rnd)
        mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows, **kw)
        mres = mp.run(_mont_small(ctx, b["values"]), b["selectors"], b["advice_equalities"], _consts(ctx, b), b["lookups"])
        out.append((vk, res, chk, mres, [cs.lagr[nm].download() for nm in cs.fixed_names + cs.sigma_names], cs.perm_cols, cs.fixed_names))
        mp.free(); sess.free(); cs.free()
    (vk0, r0, c0, m0, s0, p0, f0), (vk1, r1, c1, m1, s1, p1, f1) = out
    _same_keys(vk0, vk1)
    assert p0 == p1 and p0[0] == "c" and f0 == f1 and f0[-1] == "c"
    assert all(np.array_equal(x, y) for x, y in zip(s0, s1))
    assert all(np.array_equal(x, y) for x, y in zip(r0["commitments"], r1["commitments"]))
    assert all(np.array_equal(r0["evals"][q], r1["evals"][q]) for q in r0["evals"]) and r0["challenges"] == r1["challenges"]
    assert r0["h2d_bytes"] == r1["h2d_bytes"] and r0["d2h_bytes"] == r1["d2h_bytes"]
    assert c0 == c1 and m0 == m1


def test_cpp_front_end_matches_python(ctx, h2b, tmp_path):
    """tests/cpp/constants_test.cpp runs keygen, MockProver and a proof with F = 3 and one instance column through the C++
    headers; its break points, vk, MockProver constants report and proof bytes equal the Python front end's"""
    k, A, L, sel, bits, I, count, max_report, F = 8, 2, 1, False, 6, 1, 6, 8, 3
    n, max_rows = 1 << k, (1 << k) - 9
    rng = np.random.default_rng(91)
    b = _builder(rng, k, A, L, sel, bits, max_rows, F, fill=0.5, extra=False)
    inst = _instances(rng, b, I, count)
    public = _public(ctx, b, inst)
    _, cells, _ = co.copy_sequence(k, A, L, max_rows, b, F)
    bad_vals, _ = _broken_c1(b, cells, k)
    rnd = mont(rand_ints(rng, n, R), R)
    g = affine_to_limbs([pyref.G1])[0]
    d = str(tmp_path)
    files = {"cells": _mont_small(ctx, b["values"]), "bad_cells": _mont_small(ctx, bad_vals), "selectors": b["selectors"],
             "eq": b["advice_equalities"], "consts": _mont_small(ctx, b["constants"]), "const_index": b["constant_index"], "lookups": b["lookups"],
             "rnd": rnd, "g": ctx.g1_fixed_base_mul(g, mont([3 + 5 * i for i in range(n)], R)),
             "gl": ctx.g1_fixed_base_mul(g, mont([7 + 11 * i for i in range(n)], R))}
    for m in range(I):
        files.update({"inst%d" % m: inst[m], "pub%d" % m: public[m]})
    for name, arr in files.items():
        np.ascontiguousarray(arr).tofile(os.path.join(d, name + ".bin"))
    with open(os.path.join(d, "manifest.txt"), "w") as f:
        f.write(" ".join(str(x) for x in (k, A, L, int(sel), bits, max_rows, len(b["values"]), len(b["advice_equalities"]), len(b["constants"]),
                                          len(b["lookups"]), I, count, max_report, F)))
    exe = os.path.join(d, "constants_test")
    libdir = os.path.join(ROOT, "halo2-lib_b200")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "cpp", "constants_test.cpp"), "-o", exe,
                           f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])
    out = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    cs, vk, bps = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, F=F, I=I, instances=inst)
    want = [np.array([len(bps)] + bps, dtype=np.uint64)] + [np.asarray(vk["fixed"][nm], dtype=np.uint64) for nm in cs.fixed_names]
    want += [np.asarray(p, dtype=np.uint64) for p in vk["permutation"]]
    mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows, I=I, F=F)
    r = mp.run(files["bad_cells"], b["selectors"], b["advice_equalities"], (files["consts"], b["constant_index"]), b["lookups"],
               instances=inst, public=public, max_report=max_report)
    assert r["constants"][0] >= 1
    cnt, rows = r["constants"]
    want.append(np.array([cnt, len(rows)] + rows + [x for c in r["constant_cells"] for x in c] + [r["distinct_constants"]], dtype=np.uint64))
    sess = h2b.ProverSession(ctx, _params_for(ctx, h2b, k), cs)
    counter = iter(range(1, 1 << 30))
    sess.blind_source = lambda rows: np.array([[next(counter), 0, 0, 0] for _ in range(rows)], dtype=np.uint64)
    lk = np.ascontiguousarray(b["lookups"])
    res = sess.prove(files["cells"].ctypes.data, len(files["cells"]), rnd.ctypes.data, break_points=np.array(bps, dtype=np.uint64),
                     lookup_index_ptr=lk.ctypes.data, n_lookup=len(lk), instances=public)
    want += [np.asarray(c, dtype=np.uint64) for c in res["commitments"]] + [np.asarray(v, dtype=np.uint64) for v in res["evals"].values()]
    want += [np.asarray(h2b.prover.to_limbs(res["challenges"][c]), dtype=np.uint64) for c in ("theta", "beta", "gamma", "y", "x")]
    assert open(os.path.join(d, "out.bin"), "rb").read() == b"".join(a.tobytes() for a in want)
    sess.free(); mp.free(); cs.free()

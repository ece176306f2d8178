"""GPU tests of public inputs (instance columns) for halo2-base builders: keygen appends assign_instances' copies (sigma and
the vk against halo2's Assembly, tests/instance_oracle.py), the resident prover absorbs the public values before the advice
commitments and proves the extended quotient identity, check and MockProver report a wrong public value where halo2 would,
a session without instance columns gives the bytes it gave before, and the errors carry halo2's and halo2-base's texts."""
import numpy as np
import pytest
from oracle import pyref
from util import mont, unmont, rand_ints, affine_to_limbs
import builder_oracle as bo
import keygen_oracle as ko
import instance_oracle as io

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


def _instances(rng, b, I, count):
    return [rng.choice(len(b["selectors"]), size=count).astype(np.uint64) for _ in range(I)]


def _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, inst, oracle="python", values=True):
    I = len(inst)
    cs, vk, bps = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, I=I, instances=inst)
    pairs, _, want_bps = io.copy_sequence(k, A, L, max_rows, b, inst)
    assert bps == want_bps
    assert cs.I == I and cs.perm_cols[1 + A + L:] == ["i%d" % m for m in range(I)]
    V = (1 + A + L + I) << k
    want = ko.assembly(V, pairs) if oracle == "python" else ko.assembly_c(V, pairs)
    got = cs.sigma_map.download().view(np.uint32).reshape(-1)[:V]
    assert np.array_equal(got, want)
    sigma = [cs.lagr[nm].download() for nm in cs.sigma_names]
    if values:
        assert np.array_equal(np.stack(sigma), ko.sigma_values(want, 1 + A + L + I, k))
    params = _params_for(ctx, h2b, k)
    assert len(vk["permutation"]) == 1 + A + L + I
    for m in range(I):  # the instance columns' sigma commitments, last in perm_cols order
        c = 1 + A + L + m
        assert np.array_equal(vk["permutation"][c], h2b.prover.g1_normalize_host(params.commit_lagrange(sigma[c])))
    return cs, vk, bps


@pytest.mark.parametrize("I", [1, 2])
@pytest.mark.parametrize("k", [8, 12])
@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_keygen_with_instances_matches_the_assembly(ctx, h2b, k, A, L, sel, I):
    rng = np.random.default_rng(300 + k + 10 * A + L + I)
    bits = min(8, k - 2)
    max_rows = (1 << k) - 9
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, contexts=3)
    cs, _, _ = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, _instances(rng, b, I, 16))
    cs.free()


def _prove(ctx, h2b, cs, k, b, bps, L, public, rnd, draws_seed=1):
    sess = h2b.ProverSession(ctx, _params_for(ctx, h2b, k), cs)
    cells = _mont_small(ctx, b["values"])
    draws = np.random.default_rng(draws_seed)
    sess.blind_source = lambda rows: mont(rand_ints(draws, rows, R), R)
    lk = np.ascontiguousarray(b["lookups"] if L else np.zeros(0, dtype=np.uint64))
    kw = dict(break_points=np.array(bps, dtype=np.uint64), lookup_index_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))
    res = sess.prove(cells.ctypes.data, len(cells), rnd.ctypes.data, instances=public, **kw)
    chk = sess.check(cells.ctypes.data, len(cells), instances=public, **kw)
    return sess, res, chk


def _public(ctx, b, inst):
    return [_mont_small(ctx, b["values"][idx.astype(np.int64)]) for idx in inst]


@pytest.mark.parametrize("k,A,L,sel,bits,count", [(8, 2, 1, True, 6, 16), (12, 3, 2, False, 8, 16), (19, 1, 0, True, 18, 64)])
def test_proof_with_public_inputs(ctx, h2b, k, A, L, sel, bits, count):
    """keygen with one instance column (the ECDSA shape at k = 19 against the C Assembly), then a proof: theta is the transcript
    over the public values and the advice commitments, the extended quotient identity holds, the check is satisfied"""
    rng = np.random.default_rng(k + A)
    max_rows = (1 << k) - 9
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, fill=0.5 if k < 19 else 1.0)
    inst = _instances(rng, b, 1, count)
    cs, _, bps = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, inst, oracle="c" if k >= 19 else "python", values=k < 19)
    public = _public(ctx, b, inst)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    sess, res, chk = _prove(ctx, h2b, cs, k, b, bps, L, public, rnd)
    assert chk["satisfied"], chk
    assert res["challenges"]["theta"] == io.theta(public, res["commitments"][:A + L])
    left, right = io.quotient_identity(res, k, A, L, sel, [unmont(p, R) for p in public])
    assert left == right
    assert res["h2d_bytes"] >= 32 * count
    sess.free(); cs.free()


def test_a_wrong_public_value(ctx, h2b):
    k, A, L, sel, bits = 8, 2, 1, True, 6
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(17)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, fill=0.5)
    inst = _instances(rng, b, 2, 16)
    cs, _, bps = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, inst, values=False)
    public = _public(ctx, b, inst)
    vals = [unmont(p, R) for p in public]
    vals[1][5] = (vals[1][5] + 1) % R
    bad = [mont(v, R).reshape(-1, 4) for v in vals]
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    sess, res, chk = _prove(ctx, h2b, cs, k, b, bps, L, bad, rnd)
    # check: the instance row, and the cell whose sigma names it
    c_col = unmont(cs.lagr["c"].download(), R)
    cols = [unmont(sess.lagr[nm].download(), R) for nm in cs.adv_names]
    sigma = [unmont(cs.lagr[nm].download(), R) for nm in cs.sigma_names]
    want = io.check(k, c_col, sigma, cols, vals)
    assert not chk["satisfied"] and chk["copies"] == want
    assert chk["copies"][1 + A + L + 1] == (1, [5]) and sum(c for c, _ in chk["copies"]) == 2
    # MockProver: that row and its raw cell
    mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows, I=2)
    got = mp.run(_mont_small(ctx, b["values"]), b["selectors"], b["advice_equalities"], (_mont_small(ctx, b["constants"]), b["constant_index"]),
                 b["lookups"], instances=inst, public=bad)
    ref = io.mock_run(k, A, L, sel, bits, max_rows, b, b["values"], inst, vals)
    assert got["instances"] == ref["instances"] == [(0, []), (1, [5])]
    assert got["instance_cells"] == ref["instance_cells"] == [[], [bo.raw_cell(bps, int(inst[1][5]))]]
    assert not got["satisfied"]
    # the proof of the wrong value does not satisfy the identity
    left, right = io.quotient_identity(res, k, A, L, sel, vals)
    assert left != right
    mp.free(); sess.free(); cs.free()


def test_no_instance_columns_give_the_existing_bytes(ctx, h2b):
    k, A, L, sel, bits = 8, 2, 1, False, 6
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(23)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    out = []
    for kw in ({}, dict(I=0, instances=[])):
        cs, vk, bps = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, **kw)
        sess, res, chk = _prove(ctx, h2b, cs, k, b, bps, L, None if not kw else [], rnd)
        mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows, **({"I": 0} if kw else {}))
        mres = mp.run(_mont_small(ctx, b["values"]), b["selectors"], b["advice_equalities"], (_mont_small(ctx, b["constants"]), b["constant_index"]),
                      b["lookups"])
        out.append((vk, res, chk, mres, [cs.lagr[nm].download() for nm in cs.sigma_names]))
        mp.free(); sess.free(); cs.free()
    (vk0, r0, c0, m0, s0), (vk1, r1, c1, m1, s1) = out
    assert all(np.array_equal(x, y) for x, y in zip(vk0["permutation"], vk1["permutation"]))
    assert all(np.array_equal(x, y) for x, y in zip(s0, s1))
    assert all(np.array_equal(x, y) for x, y in zip(r0["commitments"], r1["commitments"]))
    assert all(np.array_equal(r0["evals"][q], r1["evals"][q]) for q in r0["evals"]) and r0["challenges"] == r1["challenges"]
    assert r0["h2d_bytes"] == r1["h2d_bytes"] and r0["d2h_bytes"] == r1["d2h_bytes"]
    assert c0 == c1 and m0 == m1 and m0["instances"] == []


def test_errors_carry_halo2_messages_and_leave_the_context_usable(ctx, h2b):
    k, A, L, sel, bits = 8, 2, 0, False, 4
    max_rows = (1 << k) - 9
    u = (1 << k) - 7
    rng = np.random.default_rng(29)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, fill=0.5)
    N = len(b["selectors"])
    inst = _instances(rng, b, 1, 8)

    def keygen_ok():
        return _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, inst, values=False)

    for bad, msg in (([np.array([1, N], dtype=np.uint64)], "instance not assigned"),
                     ([np.zeros(u + 1, dtype=np.uint64)], r"NotEnoughRowsAvailable \{ current_k: 8 \}")):
        with pytest.raises(h2b.H2BError, match=msg):
            _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, I=1, instances=bad)
        keygen_ok()[0].free()
    cs, _, bps = keygen_ok()
    public = _public(ctx, b, inst)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    too_many = [np.zeros((u + 1, 4), dtype=np.uint64)]
    sess = h2b.ProverSession(ctx, _params_for(ctx, h2b, k), cs)
    cells = _mont_small(ctx, b["values"])
    kw = dict(break_points=np.array(bps, dtype=np.uint64))
    with pytest.raises(h2b.H2BError, match="InstanceTooLarge"):
        sess.prove(cells.ctypes.data, len(cells), rnd.ctypes.data, instances=too_many, **kw)
    with pytest.raises(h2b.H2BError, match="InstanceTooLarge"):
        sess.check(cells.ctypes.data, len(cells), instances=too_many, **kw)
    assert sess.check(cells.ctypes.data, len(cells), instances=public, **kw)["satisfied"]
    sess.free(); cs.free()
    mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows, I=1)
    args = (_mont_small(ctx, b["values"]), b["selectors"], b["advice_equalities"], (_mont_small(ctx, b["constants"]), b["constant_index"]),
            b["lookups"])
    with pytest.raises(h2b.H2BError, match="InstanceTooLarge"):
        mp.run(*args, instances=[np.zeros(u + 1, dtype=np.uint64)], public=too_many)
    with pytest.raises(h2b.H2BError, match="instance not assigned"):
        mp.run(*args, instances=[np.array([N], dtype=np.uint64)], public=[np.zeros((1, 4), dtype=np.uint64)])
    assert mp.run(*args, instances=inst, public=public)["satisfied"]
    mp.free()


def test_proof_with_public_inputs_matches_the_oracle_prover(ctx, h2b):
    """a proof with two instance columns on a keygen circuit at k = 8, fixed blinding rows: every commitment, evaluation and
    challenge the bytes of instance_oracle.create_proof (oracle/prover_ref's flow with instance columns, Python integers)"""
    import test_oracle_prover as top
    from oracle import prover_ref
    k, A, L, sel, bits = 8, 2, 1, False, 6
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(41)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, fill=0.5)
    inst = _instances(rng, b, 2, 6)
    cs, _, bps = _check_keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, inst, values=False)
    public = _public(ctx, b, inst)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    sess, res, _ = _prove(ctx, h2b, cs, k, b, bps, L, public, rnd)
    draws = np.random.default_rng(1)  # _prove's blinding rows, replayed
    blind = lambda rows: rand_ints(draws, rows, R)
    want = io.create_proof(k, A, L, sel, {nm: unmont(cs.lagr[nm].download(), R) for nm in cs.fixed_names},
                           [unmont(cs.lagr[nm].download(), R) for nm in cs.sigma_names], [int(v) for v in b["values"]], list(bps),
                           [int(b["values"][int(i)]) for i in b["lookups"]], unmont(rnd, R), blind,
                           top.small_bases(1 << k, 3, 5), top.small_bases(1 << k, 7, 11), instances=[unmont(p, R) for p in public])
    assert res["challenges"] == want["challenges"]
    assert [np.asarray(c, dtype=np.uint64).tobytes() for c in res["commitments"]] == want["commitments"]
    assert [(nm, r) for nm, r in res["evals"]] == [(nm, r) for nm, r, _ in want["evals"]]
    assert [np.asarray(v, dtype=np.uint64).tobytes() for v in res["evals"].values()] == [prover_ref.fr_bytes(v) for _, _, v in want["evals"]]
    sess.free(); cs.free()


def test_cpp_front_end_matches_python(ctx, h2b, tmp_path):
    """tests/cpp/instance_test.cpp runs keygen, MockProver and a proof with instance columns through include/h2b200_keygen.hpp;
    its break points, vk, MockProver instance reports and proof bytes equal the Python front end's"""
    import os, subprocess
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    k, A, L, sel, bits, I, count, max_report = 8, 2, 1, False, 6, 2, 6, 8
    n, max_rows = 1 << k, (1 << k) - 9
    rng = np.random.default_rng(43)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, fill=0.5)
    inst = _instances(rng, b, I, count)
    public = _public(ctx, b, inst)
    vals = [unmont(p, R) for p in public]
    vals[1][2] = (vals[1][2] + 1) % R
    bad = [mont(v, R).reshape(-1, 4) for v in vals]
    rnd = mont(rand_ints(rng, n, R), R)
    g = affine_to_limbs([pyref.G1])[0]
    d = str(tmp_path)
    files = {"cells": _mont_small(ctx, b["values"]), "selectors": b["selectors"], "eq": b["advice_equalities"],
             "consts": _mont_small(ctx, b["constants"]), "const_index": b["constant_index"], "lookups": b["lookups"], "rnd": rnd,
             "g": ctx.g1_fixed_base_mul(g, mont([3 + 5 * i for i in range(n)], R)),
             "gl": ctx.g1_fixed_base_mul(g, mont([7 + 11 * i for i in range(n)], R))}
    for m in range(I):
        files.update({"inst%d" % m: inst[m], "pub%d" % m: public[m], "bad%d" % m: bad[m]})
    for name, arr in files.items():
        np.ascontiguousarray(arr).tofile(os.path.join(d, name + ".bin"))
    with open(os.path.join(d, "manifest.txt"), "w") as f:
        f.write(" ".join(str(x) for x in (k, A, L, int(sel), bits, max_rows, len(b["values"]), len(b["advice_equalities"]), len(b["constants"]),
                                          len(b["lookups"]), I, count, max_report)))
    exe = os.path.join(d, "instance_test")
    libdir = os.path.join(ROOT, "halo2-lib_b200")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "cpp", "instance_test.cpp"), "-o", exe,
                           f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])
    out = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    # the same through Python
    cs, vk, bps = _keygen(ctx, h2b, k, A, L, sel, bits, max_rows, b, I=I, instances=inst)
    want = [np.array([len(bps)] + bps, dtype=np.uint64)] + [np.asarray(p, dtype=np.uint64) for p in vk["permutation"]]
    mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows, I=I)
    r = mp.run(files["cells"], b["selectors"], b["advice_equalities"], (files["consts"], b["constant_index"]), b["lookups"],
               instances=inst, public=bad, max_report=max_report)
    assert r["instances"][1] == (1, [2])
    for (cnt, rows), cells in zip(r["instances"], r["instance_cells"]):
        want.append(np.array([cnt, len(rows)] + rows + [x for c in cells for x in c], dtype=np.uint64))
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

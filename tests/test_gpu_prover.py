"""GPU tests of the resident prover path (halo2-lib_b200/prover.py over the h2b_poly / product-column entry points):
a SATISFIED synthetic halo2-base circuit is proven with every column resident on the device; checked are
 - every commitment == the oracle's MSM of the polynomial that was committed (downloaded), with the real bases,
 - the product columns against plain-integer recurrences,
 - the quotient identity at the challenge point (tests/prover_check.py), and that a broken witness violates it,
 - the evaluations against Horner re-evaluation of downloaded coefficients."""
import ctypes as C
import numpy as np
import pytest
from oracle import pyref, oracle as orc
from util import *
import prover_check as pc

pytestmark = pytest.mark.gpu
R = pyref.R


@pytest.fixture(scope="module")
def h2b():
    import halo2_lib_b200 as h
    return h


@pytest.fixture(scope="module")
def ctx(h2b):
    c = h2b.Context(0)
    yield c
    c.close()


def _setup(ctx, h2b, k, seed, A=1, L=0, sel=True):
    rng = np.random.default_rng(seed)
    n = 1 << k
    g = affine_to_limbs([pyref.G1])[0]
    bases_m = ctx.g1_fixed_base_mul(g, mont([3 + 5 * i for i in range(n)], R))
    bases_l = ctx.g1_fixed_base_mul(g, mont([7 + 11 * i for i in range(n)], R))
    params = h2b.ParamsKZG(ctx, k, g=bases_m, g_lagrange=bases_l)
    inst = h2b.synthetic_circuit(ctx, k, rng, A=A, L=L, selector_lookup=sel)
    cs = h2b.Circuit(ctx, k, inst["fixed"], inst["sigma"], A=A, L=L, selector_lookup=sel)
    sess = h2b.ProverSession(ctx, params, cs)
    return rng, params, cs, sess, inst, (bases_m, bases_l)


def _prove(sess, inst, rnd, seed=5, virtual=None):
    v = np.ascontiguousarray(inst["virtual"] if virtual is None else virtual)
    lk = np.ascontiguousarray(inst["lookup"])
    return sess.prove(v.ctypes.data, len(v), rnd.ctypes.data, seed=seed, break_points=inst["break_points"],
                      lookup_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))


@pytest.mark.parametrize("k,A,L,sel", [(8, 1, 0, True), (11, 1, 0, True), (8, 1, 0, False), (9, 2, 1, True), (10, 3, 2, True), (9, 8, 2, True)])
def test_resident_proof_commitments_and_quotient_identity(ctx, h2b, k, A, L, sel):
    """shapes: the ECDSA / pairing configs (1 gate column, selector lookup), the inner_product bench (no lookup at all,
    degree 3, extended domain 2^(k+1)) and the multi-column configs of BASELINE.json (8 / 2 and 11 / 2 in the reference's
    config files; 8 / 2 here at a small k)"""
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 3100 + k + 10 * A, A, L, sel)
    nlk = cs.n_lookups
    n = 1 << k
    rnd = mont(rand_ints(rng, n, R), R)
    sess.keep = {}
    res = _prove(sess, inst, rnd)
    # advice | permuted pairs | product columns + random | h pieces | two openings
    want_cm = (A + L) + 2 * nlk + (cs.n_sets + nlk + 1) + (cs.degree - 1) + 2
    assert len(res["commitments"]) == want_cm and len(sess.keep["committed"]) == want_cm
    # the assignment produced the columns of the instance (rows below the blinding rows)
    for j, nm in enumerate(cs.adv_names):
        assert np.array_equal(sess.keep["committed"][j][1][: cs.u], inst["cols"][j][: cs.u]), nm
    for cm, (basis, poly) in zip(res["commitments"], sess.keep["committed"]):
        want = orc.msm_pippenger(poly, bases[basis])
        got = ctx.g1_normalize(np.asarray(cm).reshape(1, 12))[0]
        assert np.array_equal(got, want)
    left, right = pc.quotient_identity(res, k, cs.bf, A, L, sel)
    assert left == right
    # the evaluations are what Horner gives on the downloaded coefficients (an advice column, a product column, an h piece)
    x = res["challenges"]["x"]
    w = pyref.omega_for(k)
    assert pc.fr(res["evals"][("a0", 2)]) == pc.horner(sess.coef["a0"].download(), x * pow(w, 2, R) % R)
    assert pc.fr(res["evals"][("zp0", 1)]) == pc.horner(sess.coef["zp0"].download(), x * w % R)
    if cs.n_sets > 1:
        assert pc.fr(res["evals"][("zp0", -(cs.bf + 1))]) == pc.horner(sess.coef["zp0"].download(), x * pow(w, n - (cs.bf + 1), R) % R)
    assert pc.fr(res["evals"][("h1", 0)]) == pc.horner(sess.h.download(n, n), x)
    # PCIe accounting: witness + looked-up cells + random polynomial + blinding rows up, commitments + evaluations down
    ncols = (A + L) + 2 * nlk + cs.n_sets + nlk
    assert res["h2d_bytes"] <= (len(inst["virtual"]) + len(inst["lookup"]) + n) * 32 + 8 * 32 * ncols
    assert res["d2h_bytes"] <= want_cm * 96 + (len(res["evals"]) + nlk) * 32
    # second proof on the same session (buffers reused) with a broken gate: the identity must fail
    bad = np.ascontiguousarray(inst["virtual"]).copy()
    bad[3] = mont([12345], R)[0]
    sess.keep = None
    res2 = _prove(sess, inst, rnd, virtual=bad)
    l2, r2 = pc.quotient_identity(res2, k, cs.bf, A, L, sel)
    assert l2 != r2
    # a looked-up cell that is not in the table: ConstraintSystemFailure, reported with the phase's commitments
    bad = np.ascontiguousarray(inst["virtual"]).copy()
    bad[1] = mont([(1 << 40) + 7], R)[0]
    if not nlk:
        pass
    elif L:
        lk_bad = dict(inst); lk_bad["lookup"] = inst["lookup"].copy(); lk_bad["lookup"][0] = bad[1]
        with pytest.raises(h2b.H2BError):
            _prove(sess, lk_bad, rnd)
    else:
        with pytest.raises(h2b.H2BError):
            _prove(sess, inst, rnd, virtual=bad)
    sess.free(); cs.free(); params.close()


@pytest.mark.parametrize("k,A,L,sel", [(5, 1, 0, True), (5, 1, 0, False), (5, 2, 1, True), (6, 3, 2, True)])
def test_resident_prover_matches_the_oracle_prover(ctx, h2b, k, A, L, sel):
    """the parity test proper of row a1: the resident prover (every phase on the device, through the C ABI) against the
    oracle's restatement of the whole create_proof flow on plain Python integers (oracle/prover_ref.py: recursive NTTs,
    naive MSMs, row-by-row quotient, schoolbook divisions) — same instance, SRS, random polynomial and blinding rows:
    every commitment (affine form) and every evaluation must be the same bytes, every challenge the same integer."""
    from oracle import prover_ref
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 3700 + k + 10 * A, A, L, sel)
    n = 1 << k
    rnd = mont(rand_ints(rng, n, R), R)
    sess.blind_log = []
    res = _prove(sess, inst, rnd)
    blinds = [unmont(b, R) for b in sess.blind_log]
    sess.blind_log = None
    it = iter(blinds)

    def blind(rows):
        b = next(it)
        assert len(b) == rows
        return b
    aff = lambda B: [None if (x == 0 and y == 0) else (x, y) for x, y in zip(unmont(B[:, :4], pyref.P), unmont(B[:, 4:], pyref.P))]
    want = prover_ref.create_proof(k, A, L, sel, {nm: unmont(inst["fixed"][nm], R) for nm in cs.fixed_names},
                                   [unmont(sg, R) for sg in inst["sigma"]], unmont(inst["virtual"], R), [int(b) for b in inst["break_points"]],
                                   unmont(inst["lookup"], R) if len(inst["lookup"]) else [], unmont(rnd, R), blind, aff(bases[0]), aff(bases[1]))
    assert next(it, None) is None  # every blinding draw of the device prover was consumed, in the same order
    assert res["challenges"] == want["challenges"]
    assert [np.asarray(c, dtype=np.uint64).tobytes() for c in res["commitments"]] == want["commitments"]
    assert [(nm, r) for nm, r in res["evals"]] == [(nm, r) for nm, r, _ in want["evals"]]
    assert [np.asarray(v, dtype=np.uint64).tobytes() for v in res["evals"].values()] == [prover_ref.fr_bytes(v) for _, _, v in want["evals"]]
    sess.free(); cs.free(); params.close()


def test_resident_prover_reproduces_the_committed_golden_proof(ctx, h2b):
    """tests/golden/prover_k5.json (made by tests/golden/make_golden_prover.py from the oracle prover on an integer-built
    circuit): the CUDA path fed with the same instance, SRS, random polynomial and blinding rows writes the same bytes"""
    import json, os, random
    import test_oracle_prover as top
    from golden import make_golden_prover as g
    want = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prover_k5.json")))
    k, A, L, sel, seed = g.K, g.A, g.L, g.SEL, g.SEED
    n = 1 << k
    inst = top.int_instance(k, A, L, sel, seed)
    rr = random.Random(seed + 1)  # the draw order of test_oracle_prover.run: random polynomial first, then the blinding rows
    rnd = mont([rr.randrange(R) for _ in range(n)], R)
    to_limbs_pts = lambda pts: np.stack([np.concatenate([mont([x], pyref.P)[0], mont([y], pyref.P)[0]]) for x, y in pts])
    bases_m, bases_l = to_limbs_pts(top.small_bases(n, 3, 5)), to_limbs_pts(top.small_bases(n, 7, 11))
    params = h2b.ParamsKZG(ctx, k, g=bases_m, g_lagrange=bases_l)
    fixed = {nm: mont(v, R) for nm, v in inst["fixed"].items()}
    cs = h2b.Circuit(ctx, k, fixed, [mont(sg, R) for sg in inst["sigma"]], A=A, L=L, selector_lookup=sel)
    sess = h2b.ProverSession(ctx, params, cs)
    sess.blind_source = lambda rows: mont([rr.randrange(R) for _ in range(rows)], R)
    v, lk = mont(inst["virtual"], R), mont(inst["lookup"], R)
    res = sess.prove(v.ctypes.data, len(v), rnd.ctypes.data, break_points=np.array(inst["break_points"], dtype=np.uint64),
                     lookup_ptr=lk.ctypes.data, n_lookup=len(lk))
    assert {c: hex(x) for c, x in res["challenges"].items()} == want["challenges"]
    assert [np.asarray(c, dtype=np.uint64).tobytes().hex() for c in res["commitments"]] == want["commitments_affine_montgomery"]
    assert [[nm, r, np.asarray(x, dtype=np.uint64).tobytes().hex()] for (nm, r), x in res["evals"].items()] == want["evals_montgomery"]
    sess.free(); cs.free(); params.close()


@pytest.mark.parametrize("k,A,L,sel", [(8, 1, 0, True), (8, 1, 0, False), (9, 7, 2, True)])
def test_cpp_prover_matches_python(ctx, h2b, k, A, L, sel, tmp_path):
    """the two front ends of the compiled prover pass identical inputs: a C++ program (include/h2b200_prover.hpp over
    std::vector inputs and its own Context / ParamsKZG) and halo2-lib_b200/prover.py (the library's binding, host pointers)
    give the SAME BYTES for the same instance, SRS, random polynomial and blinding rows: commitments, evaluations and
    challenges are compared byte for byte.  The Python proof is the one the protocol-level checks above run on."""
    import os, subprocess
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 3500 + k + 10 * A, A, L, sel)
    n = 1 << k
    rnd = mont(rand_ints(rng, n, R), R)
    sess.blind_log = []
    res = _prove(sess, inst, rnd)
    blind = np.concatenate(sess.blind_log) if sess.blind_log else np.zeros((0, 4), dtype=np.uint64)
    sess.blind_log = None
    left, right = pc.quotient_identity(res, k, cs.bf, A, L, sel)
    assert left == right
    d = str(tmp_path)
    w = lambda name, arr: np.ascontiguousarray(arr, dtype=np.uint64).tofile(os.path.join(d, name))
    for nm in cs.fixed_names:
        w("fixed_%s.bin" % nm, inst["fixed"][nm])
    for i, sg in enumerate(inst["sigma"]):
        w("sigma_%d.bin" % i, sg)
    w("witness.bin", inst["virtual"]); w("breaks.bin", inst["break_points"]); w("lookup.bin", inst["lookup"])
    w("random.bin", rnd); w("blind.bin", blind); w("bases_m.bin", bases[0]); w("bases_l.bin", bases[1])
    with open(os.path.join(d, "manifest.txt"), "w") as f:
        f.write("%d %d %d %d %d %d %d %d\n" % (k, A, L, 1 if sel else 0, len(inst["virtual"]), len(inst["break_points"]), len(inst["lookup"]), len(blind)))
    import test_cpp_mirror as tcm
    exe = os.path.join(tcm.ROOT, "build", "prover_mirror_test")
    tcm.test_cpp_prover_mirror_compiles_and_links()
    out = subprocess.run([exe, d], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    raw = np.fromfile(os.path.join(d, "proof.bin"), dtype=np.uint64)
    nc = int(raw[0])
    cms = raw[1:1 + 12 * nc].reshape(nc, 12)
    ne = int(raw[1 + 12 * nc])
    evs = raw[2 + 12 * nc: 2 + 12 * nc + 4 * ne].reshape(ne, 4)
    chal = raw[2 + 12 * nc + 4 * ne:].reshape(5, 4)
    assert nc == len(res["commitments"]) and np.array_equal(cms, np.stack(res["commitments"]))
    assert ne == len(res["evals"]) and np.array_equal(evs, np.stack(list(res["evals"].values())))
    want = [res["challenges"][c] for c in ("theta", "beta", "gamma", "y", "x")]
    assert [pc.fr(c) for c in chal] == want
    sess.free(); cs.free(); params.close()


def test_shard_over_the_whole_range_matches_the_unsharded_proof(ctx, h2b):
    """the multi-GPU path on one GPU: shard(0, n, allreduce) with a callback that records its calls and leaves the points as
    they are.  It must be called once per batched MSM (at most 16 commitments; 17 advice columns make phase 0 two batches)
    with that batch's size, and the proof must be the same bytes as an unsharded one."""
    k, A, L = 8, 15, 2
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 3900, A, L, True)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    want = _prove(sess, inst, rnd)
    calls = []
    sharded = h2b.ProverSession(ctx, params, cs)
    sharded.shard(0, 1 << k, lambda ptr, m: calls.append((ptr, m)))
    got = _prove(sharded, inst, rnd)
    nlk = cs.n_lookups
    assert [m for _, m in calls] == [16, A + L - 16, 2 * nlk, cs.n_sets + nlk + 1, cs.degree - 1, 1, 1]
    assert calls[0][0] and len(set(p for p, _ in calls)) == 1
    assert [c.tobytes() for c in got["commitments"]] == [c.tobytes() for c in want["commitments"]]
    assert [(q, v.tobytes()) for q, v in got["evals"].items()] == [(q, v.tobytes()) for q, v in want["evals"].items()]
    assert got["challenges"] == want["challenges"]
    assert (got["h2d_bytes"], got["d2h_bytes"]) == (want["h2d_bytes"], want["d2h_bytes"])
    sharded.free(); sess.free(); cs.free(); params.close()


def test_product_columns_vs_integer_recurrence(ctx, h2b):
    from halo2_lib_b200._capi import lib
    k, bf = 7, 6
    n = 1 << k
    u = n - (bf + 1)
    rng = np.random.default_rng(3300)
    beta, gamma = rand_ints(rng, 2, R)
    bl, gl = mont([beta], R)[0], mont([gamma], R)[0]
    w = pyref.omega_for(k)
    # permutation: 3 columns in two sets (2 + 1), random sigma values (the recurrence does not need a valid permutation)
    cols = [rand_ints(rng, n, R) for _ in range(3)]
    sig = [rand_ints(rng, n, R) for _ in range(3)]
    P = [h2b.Poly(ctx, n) for _ in range(8)]
    for j in range(3):
        P[j].upload(mont(cols[j], R)); P[3 + j].upload(mont(sig[j], R))
    zs = []
    carry = 1
    for s, (first, cnt) in enumerate([(0, 2), (2, 1)]):
        z = [carry]
        for i in range(u):
            num = den = 1
            for j in range(first, first + cnt):
                num = num * (cols[j][i] + beta * pow(pyref.DELTA, j, R) * pow(w, i, R) + gamma) % R
                den = den * (cols[j][i] + beta * sig[j][i] + gamma) % R
            z.append(z[-1] * num % R * pow(den, -1, R) % R)
        carry = z[u]
        zs.append(z)
    vp = C.c_void_p
    tc = (C.c_void_p * 2)(P[0].ptr, P[1].ptr); ts = (C.c_void_p * 2)(P[3].ptr, P[4].ptr)
    ctx.check(lib.h2b_permutation_product_dev(ctx.h, tc, ts, 2, 0, vp(bl.ctypes.data), vp(gl.ctypes.data), k, bf, None, vp(P[6].ptr)))
    tc2 = (C.c_void_p * 1)(P[2].ptr); ts2 = (C.c_void_p * 1)(P[5].ptr)
    ctx.check(lib.h2b_permutation_product_dev(ctx.h, tc2, ts2, 1, 2, vp(bl.ctypes.data), vp(gl.ctypes.data), k, bf, vp(P[6].at(u)), vp(P[7].ptr)))
    assert unmont(P[6].download()[: u + 1], R) == zs[0]
    assert unmont(P[7].download()[: u + 1], R) == zs[1]
    # lookup product
    inp, tab, pin, ptab = (rand_ints(rng, n, R) for _ in range(4))
    for j, col in enumerate((inp, tab, pin, ptab)):
        P[j].upload(mont(col, R))
    ctx.check(lib.h2b_lookup_product_dev(ctx.h, vp(P[0].ptr), vp(P[1].ptr), vp(P[2].ptr), vp(P[3].ptr), vp(bl.ctypes.data), vp(gl.ctypes.data), k, bf, vp(P[4].ptr)))
    z = [1]
    for i in range(u):
        z.append(z[-1] * (inp[i] + beta) % R * (tab[i] + gamma) % R * pow((pin[i] + beta) * (ptab[i] + gamma) % R, -1, R) % R)
    assert unmont(P[4].download()[: u + 1], R) == z
    # handle API: ranges are checked, zero works
    with pytest.raises(h2b.H2BError):
        P[0].download(n - 1, 2)
    ctx.check(lib.h2b_poly_zero(ctx.h, P[0].h))
    assert not P[0].download().any()
    for p in P:
        p.free()

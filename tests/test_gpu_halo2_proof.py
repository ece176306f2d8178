"""GPU tests of halo2's proof bytes from the resident prover (ProverSession.gen_proof, h2b::ProverSession::create_proof_halo2):
byte equality with tests/halo2_proof_oracle.py at k = 8 with fixed blinding rows and with the committed golden proof (Python and
C++ front ends), the oracle's verify_proof on keygen'd circuits at k = 12 and 16 and on the ECDSA shape at k = 19 with each
mutation rejected, h2b_kate_division_multi against sequential kate_division in both its forms, and `prove` unaffected by a
gen_proof on the same session."""
import numpy as np
import pytest
from oracle import pyref
from util import mont, unmont, rand_ints
import halo2_proof_oracle as hp
import params_oracle as po
import test_gpu_constants as tgc
import test_oracle_halo2_proof as toh

pytestmark = pytest.mark.gpu
R, P = pyref.R, pyref.P
TAU = po.seeded_tau()
VK_REPR = 0x1234567890ABCDEF


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


def params_for(ctx, h2b, k):
    if k not in _params:
        _params[k] = h2b.ParamsKZG.setup_seeded(ctx, k)
    return _params[k]


def point(limbs):
    """12 Montgomery limbs (affine x, y, 1; identity all zero) -> canonical affine point"""
    b = np.ascontiguousarray(limbs, dtype=np.uint64).tobytes()
    x, y = (pyref.from_mont(int.from_bytes(b[32 * j:32 * j + 32], "little"), P) for j in (0, 1))
    return None if x == 0 and y == 0 else (x, y)


def keygen_proof(ctx, h2b, k, A, L, sel, bits, F, I, seed, fill=0.6):
    """a keygen'd builder circuit on params of tau, its vk (canonical points), one gen_proof with fixed blinding rows"""
    rng = np.random.default_rng(seed)
    max_rows = (1 << k) - 9
    b = tgc._builder(rng, k, A, L, sel, bits, max_rows, F, fill=fill, extra=False)
    inst = tgc._instances(rng, b, I, 5)
    params = params_for(ctx, h2b, k)
    cs, vk, bps = h2b.keygen(ctx, params, k, A, L, sel, bits, max_rows, b["selectors"], b["advice_equalities"], tgc._consts(ctx, b),
                             b["lookups"], F=F, I=I, instances=inst if I else None)
    public = tgc._public(ctx, b, inst) if I else None
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    sess = h2b.ProverSession(ctx, params, cs)
    draws = np.random.default_rng(seed + 1)
    sess.blind_source = lambda rows: mont(rand_ints(draws, rows, R), R)
    cells = tgc._mont_small(ctx, b["values"])
    lk = np.ascontiguousarray(b["lookups"] if L else np.zeros(0, dtype=np.uint64))
    kw = dict(break_points=np.array(bps, dtype=np.uint64), lookup_index_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))
    proof = sess.gen_proof(cells.ctypes.data, len(cells), rnd.ctypes.data, VK_REPR, instances=public, **kw)
    vkp = {"fixed": {nm: point(c) for nm, c in vk["fixed"].items()}, "permutation": [point(c) for c in vk["permutation"]]}
    return dict(b=b, cs=cs, sess=sess, bps=bps, rnd=rnd, proof=proof, vk=vkp, public=[unmont(p, R) for p in public or []], kw=kw,
                cells=cells, public_limbs=public)


@pytest.mark.parametrize("A,L,sel", toh.SHAPE_KINDS)
def test_gen_proof_is_the_oracles_bytes(ctx, h2b, A, L, sel):
    k, F, I, bits = 8, 2, 1, 6
    r = keygen_proof(ctx, h2b, k, A, L, sel, bits, F, I, 51 + A + L, fill=0.5)
    cs = r["cs"]
    g, gl, _, _ = po.params_setup(k, TAU)
    draws = np.random.default_rng(51 + A + L + 1)
    want = hp.create_proof(k, A, L, sel, F, {nm: unmont(cs.lagr[nm].download(), R) for nm in cs.fixed_names},
                           [unmont(cs.lagr[nm].download(), R) for nm in cs.sigma_names], [int(v) for v in r["b"]["values"]], list(r["bps"]),
                           [int(r["b"]["values"][int(i)]) for i in r["b"]["lookups"]] if L else [], unmont(r["rnd"], R),
                           lambda rows: rand_ints(draws, rows, R), g, gl, r["public"], VK_REPR)
    assert r["proof"] == want
    assert hp.verify_proof(r["proof"], k, A, L, sel, F, r["vk"], r["public"], VK_REPR, pyref.G1, TAU)
    r["sess"].free(); cs.free()


# the lookup-advice shape (3 / 2, degree 4) at k = 12 and 16, and the ECDSA shape (1 / 0 with the selector lookup: degree 5,
# permutation chunks of 3, 4 h pieces; bench_ecdsa.config) at k = 19
@pytest.mark.parametrize("k,A,L,sel,F,bits", [(12, 3, 2, False, 2, 8), (16, 3, 2, False, 2, 8), (19, 1, 0, True, 1, 18)])
def test_oracle_verifies_gpu_proofs(ctx, h2b, k, A, L, sel, F, bits):
    I = 1
    r = keygen_proof(ctx, h2b, k, A, L, sel, bits, F, I, 70 + k)
    verify = lambda proof, repr_=VK_REPR, public=None: hp.verify_proof(proof, k, A, L, sel, F, r["vk"], r["public"] if public is None else public,
                                                                        repr_, pyref.G1, TAU)
    assert verify(r["proof"])
    for what, at in toh.mutations(k, A, L, sel, F, I).items():
        bad = bytearray(r["proof"])
        bad[at] ^= 1
        assert not verify(bytes(bad)), what
    assert not verify(r["proof"], VK_REPR + 1)
    public = [list(c) for c in r["public"]]
    public[0][0] = (public[0][0] + 1) % R
    assert not verify(r["proof"], public=public)
    assert not verify(toh.swapped_openings(r["proof"]))
    r["sess"].free(); r["cs"].free()


def _golden():
    """the committed golden proof and its inputs as the device takes them (Montgomery limbs)"""
    import json, os
    from golden import make_golden_halo2_proof as g
    want = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "halo2_proof_k5.json")))
    inst, rnd, rr = g.inputs()
    return g, bytes.fromhex(want["proof"]), inst, mont(rnd, R), rr


def _golden_gen_proof(ctx, h2b, g, inst, rnd, rr):
    cs = h2b.Circuit(ctx, g.K, {nm: mont(v, R) for nm, v in inst["fixed"].items()}, [mont(sg, R) for sg in inst["sigma"]], A=g.A, L=g.L,
                     selector_lookup=g.SEL, I=g.I, F=g.F)
    sess = h2b.ProverSession(ctx, params_for(ctx, h2b, g.K), cs)
    sess.blind_source = lambda rows: mont([rr.randrange(R) for _ in range(rows)], R)
    v, lk = mont(inst["virtual"], R), mont(inst["lookup"], R)
    proof = sess.gen_proof(v.ctypes.data, len(v), rnd.ctypes.data, g.VK_REPR, instances=[mont(p, R) for p in inst["public"]],
                           break_points=np.array(inst["break_points"], dtype=np.uint64), lookup_ptr=lk.ctypes.data, n_lookup=len(lk))
    sess.free(); cs.free()
    return proof


def test_gen_proof_reproduces_the_committed_golden_proof(ctx, h2b):
    """tests/golden/halo2_proof_k5.json (tests/golden/make_golden_halo2_proof.py, Python integers): the CUDA path fed the same
    instance, params, random polynomial and blinding rows writes the same bytes"""
    g, want, inst, rnd, rr = _golden()
    assert _golden_gen_proof(ctx, h2b, g, inst, rnd, rr) == want


def test_cpp_front_end_matches_python(ctx, h2b, tmp_path):
    """tests/cpp/halo2_proof_test.cpp runs ProverSession::create_proof_halo2 through the C++ headers on the golden instance; its
    bytes equal the Python front end's and the committed golden proof"""
    import os, subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    g, want, inst, rnd, rr = _golden()
    blinds = [rr.randrange(R) for _ in range(4096)]  # the stream the prover draws from, after the random polynomial
    gb, glb, _, _ = po.params_setup(g.K, TAU)
    pts = lambda ps: np.stack([np.concatenate([mont([x], P)[0], mont([y], P)[0]]) for x, y in ps])
    d = str(tmp_path)
    s = hp.shape(g.K, g.A, g.L, g.SEL, g.F, g.I)
    files = {"cells": mont(inst["virtual"], R), "break_points": np.array(inst["break_points"], dtype=np.uint64),
             "lookup": mont(inst["lookup"], R), "rnd": rnd, "g": pts(gb), "gl": pts(glb), "vk_repr": mont([g.VK_REPR], R),
             "blind": mont(blinds, R)}
    files.update({"fixed_" + nm: mont(inst["fixed"][nm], R) for nm in s["fixed"]})
    files.update({"sigma%d" % c: mont(col, R) for c, col in enumerate(inst["sigma"])})
    files.update({"pub%d" % m: mont(col, R) for m, col in enumerate(inst["public"])})
    for name, arr in files.items():
        np.ascontiguousarray(arr).tofile(os.path.join(d, name + ".bin"))
    with open(os.path.join(d, "fixed_names.txt"), "w") as f:
        f.write(" ".join(s["fixed"]))
    with open(os.path.join(d, "manifest.txt"), "w") as f:
        f.write(" ".join(str(x) for x in (g.K, g.A, g.L, int(g.SEL), g.I, g.F, len(inst["virtual"]), len(inst["break_points"]),
                                          len(inst["lookup"]), len(inst["public"][0]), len(blinds))))
    exe = os.path.join(d, "halo2_proof_test")
    libdir = os.path.join(root, "halo2-lib_b200")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-Wall", os.path.join(root, "tests", "cpp", "halo2_proof_test.cpp"), "-o", exe,
                           f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])
    out = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    got = open(os.path.join(d, "out.bin"), "rb").read()
    _, _, inst2, rnd2, rr2 = _golden()
    assert got == want == _golden_gen_proof(ctx, h2b, g, inst2, rnd2, rr2)


def test_prove_is_unchanged_by_gen_proof(ctx, h2b):
    """prove on a session before and after a gen_proof gives the bytes of a fresh session"""
    k, A, L, sel, F, I, bits = 10, 2, 1, False, 2, 1, 6
    r = keygen_proof(ctx, h2b, k, A, L, sel, bits, F, I, 91)
    sess, cells, rnd = r["sess"], r["cells"], r["rnd"]

    def prove(s):
        s.blind_source = None
        return s.prove(cells.ctypes.data, len(cells), rnd.ctypes.data, seed=3, instances=r["public_limbs"], **r["kw"])
    before = prove(sess)
    again = sess.gen_proof(cells.ctypes.data, len(cells), rnd.ctypes.data, VK_REPR, instances=r["public_limbs"], seed=4, **r["kw"])
    after = prove(sess)
    fresh_sess = h2b.ProverSession(ctx, params_for(ctx, h2b, k), r["cs"])
    fresh = prove(fresh_sess)
    for res in (before, after):
        assert all(np.array_equal(x, y) for x, y in zip(res["commitments"], fresh["commitments"]))
        assert all(np.array_equal(res["evals"][q], fresh["evals"][q]) for q in fresh["evals"]) and res["challenges"] == fresh["challenges"]
    again2 = fresh_sess.gen_proof(cells.ctypes.data, len(cells), rnd.ctypes.data, VK_REPR, instances=r["public_limbs"], seed=4, **r["kw"])
    assert again == again2
    fresh_sess.free(); sess.free(); r["cs"].free()


def _rand_fr(rng, n):
    """n elements below r as Montgomery limbs (any value below r is the Montgomery form of some element)"""
    a = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.int64).astype(np.uint64)
    a[:, 3] &= np.uint64((1 << 60) - 1)
    return a


@pytest.mark.parametrize("n", [1 << 10, 1 << 19, 1 << 20])
def test_kate_division_multi(ctx, h2b, n):
    import ctypes as C
    import torch
    from halo2_lib_b200._capi import lib
    rng = np.random.default_rng(n)
    a = _rand_fr(rng, n)
    vp = lambda arr: C.c_void_p(arr.ctypes.data)
    for m in (1, 2, 3, 4):
        zs = rand_ints(rng, m, R)
        ws = []
        for j in range(m):
            d = 1
            for t in range(m):
                if t != j:
                    d = d * (zs[j] - zs[t]) % R
            ws.append(pow(d, -1, R))
        pts, wts = mont(zs, R), mont(ws, R)
        q = np.zeros((n - 1, 4), dtype=np.uint64)
        ctx.check(lib.h2b_kate_division_multi(ctx.h, vp(a), n, vp(pts), m, vp(wts), vp(q)))
        seq = a
        for z in pts:
            seq = h2b.kate_division(ctx, seq, z)
        assert np.array_equal(q[:n - m], seq) and not q[n - m:].any(), m
        if n == 1 << 10:
            want = unmont(a, R)
            for z in zs:
                want = pyref.kate_division(want, z)
            assert unmont(q[:n - m], R) == want
        da = torch.from_numpy(a.view(np.int64).copy()).cuda()
        dq = torch.zeros((n - 1, 4), dtype=torch.int64, device="cuda")
        ctx.check(lib.h2b_kate_division_multi_dev(ctx.h, C.c_void_p(da.data_ptr()), n, vp(pts), m, vp(wts), C.c_void_p(dq.data_ptr())))
        ctx.synchronize()
        assert np.array_equal(dq.cpu().numpy().view(np.uint64), q)
    one = mont([1], R)
    assert lib.h2b_kate_division_multi(ctx.h, vp(a), n, vp(mont(rand_ints(rng, 5, R), R)), 5, vp(mont([1] * 5, R)), vp(q)) != 0
    assert lib.h2b_kate_division_multi(ctx.h, vp(a), 0, vp(one), 1, vp(one), vp(q)) != 0

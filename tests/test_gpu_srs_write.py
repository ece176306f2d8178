"""GPU tests (-m gpu) of halo2-lib's params on the device (gen_srs, ParamsKZG::setup with ChaCha20Rng, ParamsKZG::write,
Params::downsize): the G1 encoding kernel against Python integers and as the inverse of the decoder; the params gen_srs(4)
creates against the committed golden image in both formats; written images read back by the existing readers and committing
as the closed form at halo2-lib's tau says; downsizing from resident bases and from an image; gen_srs's file cache, its errors
and the keys keygen builds on it; a proof on it; the C++ front end against the Python one."""
import ctypes as C
import json
import os
import subprocess
import numpy as np
import pytest
from oracle import pyref, oracle as orc
import params_oracle as po
from util import mont, rand_ints, affine_to_limbs
import builder_oracle as bo
import prover_check as pc

pytestmark = pytest.mark.gpu
R, P = pyref.R, pyref.P
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RINV = pow(1 << 256, -1, R)


@pytest.fixture(scope="module")
def h2b():
    import halo2_lib_b200 as h
    return h


@pytest.fixture(scope="module")
def ctx(h2b):
    c = h2b.Context(0)
    yield c
    c.close()


def _compress_host(ctx, pts_limbs):
    from halo2_lib_b200._capi import lib
    a = np.ascontiguousarray(pts_limbs, dtype=np.uint64).reshape(-1, 8)
    out = np.zeros((len(a), 32), dtype=np.uint8)
    ctx.check(lib.h2b_g1_compress(ctx.h, C.c_void_p(a.ctypes.data), len(a), C.c_void_p(out.ctypes.data)))
    return out


def test_compress_matches_python_integers(ctx, h2b):
    from halo2_lib_b200._capi import lib
    rng = np.random.default_rng(4100)
    pts = [pyref.g1_mul(s, pyref.G1) for s in rand_ints(rng, 60, R)] + [None, pyref.G1, pyref.g1_neg(pyref.G1), None]
    assert {p[1] & 1 for p in pts if p} == {0, 1}
    limbs = affine_to_limbs(pts)
    got = _compress_host(ctx, limbs)
    assert [bytes(r) for r in got] == [pyref.g1_compress(p) for p in pts]
    # the `_dev` form gives the same bytes
    dp, db = h2b.Poly(ctx, 2 * len(pts)), h2b.Poly(ctx, len(pts))
    dp.upload(limbs.reshape(-1, 4))
    ctx.check(lib.h2b_g1_compress_dev(ctx.h, C.c_void_p(dp.ptr), len(pts), C.c_void_p(db.ptr)))
    assert np.array_equal(db.download().view(np.uint8).reshape(-1, 32), got)
    dp.free(); db.free()


def test_decompress_inverts_compress_on_a_seeded_srs_of_2_20(ctx, h2b):
    from halo2_lib_b200._capi import lib
    k = 20
    n = 1 << k
    params = h2b.ParamsKZG.setup_seeded(ctx, k)
    enc, back = h2b.Poly(ctx, n), h2b.Poly(ctx, 2 * n)
    for base in (params._g, params._gl):
        ctx.check(lib.h2b_g1_compress_dev(ctx.h, C.c_void_p(base.ptr), n, C.c_void_p(enc.ptr)))
        bad = C.c_size_t(7)
        ctx.check(lib.h2b_g1_decompress_dev(ctx.h, C.c_void_p(enc.ptr), n, C.c_void_p(back.ptr), C.byref(bad)))
        assert bad.value == 0
        ctx.synchronize()
        want = np.empty((2 * n, 4), dtype=np.uint64)
        ctx.check(lib.h2b_poly_download(ctx.h, base.h, 0, C.c_void_p(want.ctypes.data), 2 * n))
        assert np.array_equal(back.download(), want)
        # host twin == `_dev` form
        sl = want.reshape(-1, 8)[:4096]
        assert np.array_equal(_compress_host(ctx, sl), enc.download(0, 4096).view(np.uint8).reshape(-1, 32))
    enc.free(); back.free(); params.close()


def test_setup_seeded_write_equals_the_golden_image(ctx, h2b):
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "srs_seeded_k4.json")))
    params = h2b.ParamsKZG.setup_seeded(ctx, 4)
    assert params.write("processed") == bytes.fromhex(want["processed"])
    assert params.write("raw") == bytes.fromhex(want["raw"])
    assert np.array_equal(h2b.seeded_tau(), mont([int(want["tau"], 16)], R)[0])
    params.close()


def _closed_form(coeff_limbs, tau):
    """commit(coeffs) with g[i] = tau^i G is p(tau) G; the limbs are Montgomery"""
    acc = 0
    for row in coeff_limbs[::-1]:
        acc = (acc * tau + (int(row[0]) | int(row[1]) << 64 | int(row[2]) << 128 | int(row[3]) << 192)) % R
    return pyref.g1_mul(acc * RINV % R, pyref.G1)


def _affine(ctx, jac):
    from util import jac_limbs_to_affine
    return jac_limbs_to_affine(ctx.g1_normalize(np.asarray(jac).reshape(1, 12))[0])


@pytest.mark.parametrize("k", [16, 20])
def test_written_images_read_back_and_commit_as_the_closed_form(ctx, h2b, k):
    from halo2_lib_b200._capi import lib
    n = 1 << k
    tau = po.seeded_tau()
    params = h2b.ParamsKZG.setup_seeded(ctx, k)
    proc, raw = params.write("processed"), params.write("raw")
    assert len(proc) == 4 + 64 * n + 128 and len(raw) == 4 + 128 * n + 256
    assert proc[-128:] == params.g2_processed and raw[-256:] == params.g2_raw
    # RawBytes: h2b_params_raw_view, then an SRS uploaded from the arrays of the image
    img = np.frombuffer(raw, dtype=np.uint8).copy()
    kk, o = C.c_uint32(), [C.c_size_t() for _ in range(4)]
    assert lib.h2b_params_raw_view(C.c_void_p(img.ctypes.data), len(img), C.byref(kk), *[C.byref(x) for x in o]) == 0 and kk.value == k
    g = img[o[0].value:o[1].value].view(np.uint64).reshape(n, 8)
    gl = img[o[1].value:o[2].value].view(np.uint64).reshape(n, 8)
    from_raw = h2b.ParamsKZG(ctx, k, g=g, g_lagrange=gl)
    from_proc = h2b.ParamsKZG.read(ctx, proc)  # h2b_srs_read_processed
    rng = np.random.default_rng(4200 + k)
    coeffs = rng.integers(0, 1 << 62, size=(n, 4), dtype=np.int64).astype(np.uint64)
    coeffs[:, 3] &= np.uint64((1 << 60) - 1)
    evals = h2b.EvaluationDomain(ctx, 2, k).coeff_to_lagrange(coeffs)
    want = _closed_form(coeffs, tau)
    for p in (params, from_raw, from_proc):
        assert _affine(ctx, p.commit(coeffs)) == want
        assert _affine(ctx, p.commit_lagrange(evals)) == want
    from_raw.close(); from_proc.close(); params.close()


@pytest.mark.parametrize("big,small", [(12, 8), (20, 16)])
def test_downsize_from_resident_bases_and_from_an_image(ctx, h2b, big, small):
    want = h2b.ParamsKZG.setup_seeded(ctx, small)
    want_raw, want_proc = want.write("raw"), want.write("processed")
    want.close()
    p = h2b.ParamsKZG.setup_seeded(ctx, big)
    image = p.write("processed")
    p.downsize(small)
    assert p.k == small and p.write("raw") == want_raw
    p.close()
    q = h2b.ParamsKZG.read_downsized(ctx, image, small)
    assert q.write("processed") == want_proc
    with pytest.raises(h2b.H2BError):
        q.write("raw")  # the raw G2 encoding is not in a Processed image
    q.close()


def _mont_small(ctx, v):
    v = np.ascontiguousarray(v, dtype=np.uint64)
    z = np.zeros(len(v), dtype=np.uint64)
    return ctx.field_op(1, 5, np.stack([v, z, z, z], axis=1)) if len(v) else np.zeros((0, 4), dtype=np.uint64)


def _keygen(ctx, h2b, params, k, A, L, sel, bits, b):
    return h2b.keygen(ctx, params, k, A, L, sel, bits, (1 << k) - 9, b["selectors"], b["advice_equalities"],
                      (_mont_small(ctx, b["constants"]), b["constant_index"]), b["lookups"])


def test_gen_srs_creates_reads_and_rejects_bad_files(ctx, h2b, tmp_path, monkeypatch):
    k, A, L, sel, bits = 10, 2, 1, False, 6
    monkeypatch.setenv("PARAMS_DIR", str(tmp_path / "params"))
    path = h2b.srs_path(k)
    assert path == str(tmp_path / "params" / "kzg_bn254_10.srs") and not os.path.exists(path)
    first = h2b.gen_srs(ctx, k)
    ref = h2b.ParamsKZG.setup_seeded(ctx, k)
    assert open(path, "rb").read() == ref.write("processed")
    ref.close()
    second = h2b.gen_srs(ctx, k)
    assert second.g2_processed == first.g2_processed
    b = bo.make_builder(np.random.default_rng(4300), k, A, L, sel, bits, (1 << k) - 9)
    cs1, vk1, bps1 = _keygen(ctx, h2b, first, k, A, L, sel, bits, b)
    cs2, vk2, bps2 = _keygen(ctx, h2b, second, k, A, L, sel, bits, b)
    assert bps1 == bps2
    assert all(np.array_equal(vk1["fixed"][nm], vk2["fixed"][nm]) for nm in vk1["fixed"])
    assert all(np.array_equal(x, y) for x, y in zip(vk1["permutation"], vk2["permutation"]))
    cs1.free(); cs2.free(); second.close()
    # a truncated file and a corrupted point: H2B_ERR_ARG, and the next call on the context succeeds
    good = open(path, "rb").read()
    nonres = next(x for x in range(2, 100) if pow((x ** 3 + 3) % P, (P - 1) // 2, P) != 1)
    for bad in (good[:-1], good[:4 + 32 * 5] + nonres.to_bytes(32, "little") + good[4 + 32 * 6:]):
        open(path, "wb").write(bad)
        with pytest.raises(h2b.H2BError) as ei:
            h2b.gen_srs(ctx, k)
        assert ei.value.code == h2b.H2B_ERR_ARG
        open(path, "wb").write(good)
        h2b.gen_srs(ctx, k).close()
    first.close()


def test_a_proof_on_gen_srs_params_and_keygen_circuit(ctx, h2b, tmp_path):
    k, A, L, sel, bits = 12, 2, 1, True, 8
    params = h2b.gen_srs(ctx, k, str(tmp_path))
    raw = np.frombuffer(params.write("raw"), dtype=np.uint8)
    n = 1 << k
    bases = (raw[4:4 + 64 * n].view(np.uint64).reshape(n, 8), raw[4 + 64 * n:4 + 128 * n].view(np.uint64).reshape(n, 8))
    rng = np.random.default_rng(4400)
    b = bo.make_builder(rng, k, A, L, sel, bits, (1 << k) - 9)
    cs, _, bps = _keygen(ctx, h2b, params, k, A, L, sel, bits, b)
    sess = h2b.ProverSession(ctx, params, cs)
    cells = _mont_small(ctx, b["values"])
    lk = np.ascontiguousarray(b["lookups"] if L else np.zeros(0, dtype=np.uint64))
    rnd = mont(rand_ints(rng, n, R), R)
    sess.keep = {}
    res = sess.prove(cells.ctypes.data, len(cells), rnd.ctypes.data, break_points=np.array(bps, dtype=np.uint64),
                     lookup_index_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))
    assert len(res["commitments"]) == len(sess.keep["committed"])
    for cm, (basis, poly) in zip(res["commitments"], sess.keep["committed"]):
        assert np.array_equal(ctx.g1_normalize(np.asarray(cm).reshape(1, 12))[0], orc.msm_pippenger(poly, bases[basis]))
    left, right = pc.quotient_identity(res, k, cs.bf, A, L, sel)
    assert left == right
    sess.free(); cs.free(); params.close()


def test_cpp_front_end_matches_python(ctx, h2b, tmp_path):
    exe = os.path.join(ROOT, "build", "srs_write_test")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    libdir = os.path.join(ROOT, "halo2-lib_b200")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "cpp", "srs_write_test.cpp"), "-o", exe,
                           f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])
    out = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "all checks passed" in out.stdout
    rd = lambda nm: open(tmp_path / nm, "rb").read()
    p4 = h2b.ParamsKZG.setup_seeded(ctx, 4)
    assert rd("k4_processed.bin") == p4.write("processed") and rd("k4_raw.bin") == p4.write("raw")
    p4.close()
    p12 = h2b.ParamsKZG.setup_seeded(ctx, 12)
    image = p12.write("processed")
    p12.downsize(8)
    assert rd("down_12_8.bin") == p12.write("raw")
    p12.close()
    q = h2b.ParamsKZG.read_downsized(ctx, image, 8)
    assert rd("image_12_8.bin") == q.write("processed")
    q.close()
    p6 = h2b.ParamsKZG.setup_seeded(ctx, 6)
    assert rd("params/kzg_bn254_6.srs") == p6.write("processed")
    p6.close()

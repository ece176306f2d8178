"""CPU tests of gen_srs's params (halo2-base/src/utils/mod.rs:413-443): tests/params_oracle.py's ChaCha20, from_uniform_bytes, Fq2 / G2
and params image against published vectors and against each other; the library's host-only calls h2b_srs_seeded_tau and
h2b_g2_generator_mul against params_oracle; the committed golden image rebuilt from Python integers."""
import ctypes as C
import importlib.util
import json
import os
import random
import numpy as np
from oracle import pyref
import params_oracle as po
from util import mont, limbs_to_ints

R, P = pyref.R, pyref.P
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_chacha20_keystream_matches_rfc7539():
    """RFC 7539 §A.1 test vector #1 (all-zero key, nonce 0, counter 0), also rand_chacha's own `true_values` test"""
    w = po.chacha20_block(bytes(32), 0)
    assert w[:4] == [0xADE0B876, 0x903DF1A0, 0xE56A5D40, 0x28BD8653]
    stream = po.chacha20_fill_bytes(bytes(32), 100)
    assert stream[:64] == b"".join(x.to_bytes(4, "little") for x in w)
    assert stream[64:] == b"".join(x.to_bytes(4, "little") for x in po.chacha20_block(bytes(32), 1))[:36]


def test_from_uniform_bytes_is_the_512_bit_integer_mod_r():
    b = bytes(range(64))
    lo, hi = int.from_bytes(b[:32], "little"), int.from_bytes(b[32:], "little")
    assert po.from_uniform_bytes(b) == (lo + hi * (1 << 256)) % R
    assert po.from_uniform_bytes(bytes([0xFF] * 64)) == ((1 << 512) - 1) % R


def test_g2_generator_is_on_the_twist_and_has_order_r():
    assert po.g2_is_on_curve(po.G2)
    assert po.g2_mul(R, po.G2) is None
    assert po.g2_mul(R - 1, po.G2) == (po.G2[0], po.f2_sub((0, 0), po.G2[1]))


def test_tau_g2_along_two_routes_and_encodings_decode():
    rng = random.Random(11)
    for tau in [po.seeded_tau(), 2, R - 1] + [rng.randrange(1, R) for _ in range(3)]:
        s = po.g2_mul(tau, po.G2)
        assert s == po.g2_add(po.g2_mul(tau - 1, po.G2), po.G2)
        assert po.g2_is_on_curve(s)
        for pt in (s, po.G2, None):
            e = po.g2_compress(pt)
            assert len(e) == 64 and po.g2_decompress(e) == (pt, True)
            assert po.g2_from_raw(po.g2_raw(pt)) == pt
    neg = (po.G2[0], po.f2_sub((0, 0), po.G2[1]))
    assert po.g2_compress(neg)[63] ^ po.g2_compress(po.G2)[63] == 0x40


def _lib_tau(seed: bytes) -> np.ndarray:
    from halo2_lib_b200._capi import lib
    s = np.frombuffer(seed, dtype=np.uint8).copy()
    t = np.zeros(4, dtype=np.uint64)
    assert lib.h2b_srs_seeded_tau(C.c_void_p(s.ctypes.data), C.c_void_p(t.ctypes.data)) == 0
    return t


def _lib_g2(tau_limbs: np.ndarray):
    from halo2_lib_b200._capi import lib
    proc, raw = np.zeros(128, dtype=np.uint8), np.zeros(256, dtype=np.uint8)
    t = np.ascontiguousarray(tau_limbs, dtype=np.uint64)
    assert lib.h2b_g2_generator_mul(C.c_void_p(t.ctypes.data), C.c_void_p(proc.ctypes.data), C.c_void_p(raw.ctypes.data)) == 0
    return proc.tobytes(), raw.tobytes()


def test_library_seeded_tau_and_g2_pair_match_python_integers():
    rng = random.Random(2026)
    for seed in [bytes(32)] + [bytes(rng.randrange(256) for _ in range(32)) for _ in range(20)]:
        tau = po.seeded_tau(seed)
        t = _lib_tau(seed)
        assert np.array_equal(t, mont([tau], R)[0]), seed.hex()
        proc, raw = _lib_g2(t)
        s = po.g2_mul(tau, po.G2)
        assert proc == po.g2_compress(po.G2) + po.g2_compress(s)
        assert raw == po.g2_raw(po.G2) + po.g2_raw(s)
    # a tau that is not below r, and null pointers, are rejected
    from halo2_lib_b200._capi import lib
    bad = np.array([0xFFFFFFFFFFFFFFFF] * 4, dtype=np.uint64)
    assert lib.h2b_g2_generator_mul(C.c_void_p(bad.ctypes.data), None, None) == -1
    assert lib.h2b_srs_seeded_tau(None, None) == -1


def _golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_srs", os.path.join(GOLDEN, "make_golden_srs.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_golden_image_rebuilds_from_python_integers():
    want = json.load(open(os.path.join(GOLDEN, "srs_seeded_k4.json")))
    assert _golden_module().build() == want
    assert int(want["tau"], 16) == po.seeded_tau()
    img = bytes.fromhex(want["processed"])
    n = 1 << 4
    assert len(img) == 4 + 2 * n * 32 + 128 and len(bytes.fromhex(want["raw"])) == 4 + 2 * n * 64 + 256
    # the library's host-only params views read both images
    from halo2_lib_b200._capi import lib
    for key, view, g1, g2 in (("processed", lib.h2b_params_processed_view, 32, 64), ("raw", lib.h2b_params_raw_view, 64, 128)):
        b = np.frombuffer(bytes.fromhex(want[key]), dtype=np.uint8).copy()
        kk, o = C.c_uint32(), [C.c_size_t() for _ in range(4)]
        assert view(C.c_void_p(b.ctypes.data), len(b), C.byref(kk), *[C.byref(x) for x in o]) == 0
        assert kk.value == 4 and [x.value for x in o] == [4, 4 + n * g1, 4 + 2 * n * g1, 4 + 2 * n * g1 + g2]
    # every G1 encoding of the processed image decodes to the raw image's point
    raw = bytes.fromhex(want["raw"])
    for i in range(2 * n):
        pt, ok = pyref.g1_decompress(img[4 + 32 * i:36 + 32 * i])
        assert ok and po.g1_raw(pt) == raw[4 + 64 * i:68 + 64 * i]


def test_params_write_size_query_needs_no_device():
    from halo2_lib_b200._capi import lib
    ln = C.c_size_t(0)
    assert lib.h2b_params_write_processed(None, None, None, 5, None, None, C.byref(ln)) == 0 and ln.value == 4 + 2 * 32 * 32 + 128
    assert lib.h2b_params_write_raw(None, None, None, 5, None, None, C.byref(ln)) == 0 and ln.value == 4 + 2 * 32 * 64 + 256
    assert lib.h2b_params_write_raw(None, None, None, 29, None, None, C.byref(ln)) == -1

"""The C++ host mirror (include/h2b200.hpp) compiles against the C ABI (CPU) and passes its checks on the GPU."""
import os
import subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "host_mirror_test.cpp")
EXE = os.path.join(ROOT, "build", "host_mirror_test")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _build():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    libdir = os.path.join(ROOT, "halo2-lib_b200")
    subprocess.check_call([CXX, "-std=c++17", "-O1", "-Wall", SRC, "-o", EXE, f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])


def test_cpp_mirror_compiles_and_links():
    _build()
    assert os.path.exists(EXE)


@pytest.mark.gpu
def test_cpp_mirror_runs():
    _build()
    out = subprocess.run([EXE], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "all checks passed" in out.stdout


PROVER_HOST_SRC = os.path.join(ROOT, "tests", "cpp", "prover_host_test.cpp")
PROVER_HOST_EXE = os.path.join(ROOT, "build", "prover_host_test")


def test_cpp_prover_host_side_matches_python_integers():
    """the host pieces of include/h2b200_prover.hpp — Blake2b-512, the transcript's challenge (64 bytes mod r), the 254-bit
    Montgomery arithmetic used for rotations and powers of challenges, the normalisation of commitments — against hashlib and
    plain Python integers"""
    import hashlib
    os.makedirs(os.path.dirname(PROVER_HOST_EXE), exist_ok=True)
    libdir = os.path.join(ROOT, "halo2-lib_b200")
    subprocess.check_call([CXX, "-std=c++17", "-O1", "-Wall", PROVER_HOST_SRC, "-o", PROVER_HOST_EXE, f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])
    out = dict(l.split() for l in subprocess.check_output([PROVER_HOST_EXE]).decode().splitlines())
    R = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
    mont_hex = lambda x: (x * (1 << 256) % R).to_bytes(32, "little").hex()
    pat = bytes((i * 7 + 3) & 0xFF for i in range(300))
    assert out["blake_empty"] == hashlib.blake2b(b"", digest_size=64).hexdigest()
    assert out["blake_abc"] == hashlib.blake2b(b"abc", digest_size=64).hexdigest()
    assert out["blake_128"] == hashlib.blake2b(pat[:128], digest_size=64).hexdigest()
    assert out["blake_300"] == hashlib.blake2b(pat, digest_size=64).hexdigest()
    h = hashlib.blake2b(digest_size=64)

    def squeeze():
        d = h.digest()
        h.update(b"\x00")
        return int.from_bytes(d, "little") % R
    h.update(pat[:96]); c1 = squeeze(); h.update(pat[96:296]); c2 = squeeze(); c3 = squeeze()
    assert (out["squeeze1"], out["squeeze2"], out["squeeze3"]) == (mont_hex(c1), mont_hex(c2), mont_hex(c3))
    assert out["mul"] == mont_hex(c1 * c2 % R) and out["add"] == mont_hex((c1 + c2) % R) and out["pow"] == mont_hex(pow(c3, 1234567, R))
    root = pow(7, (R - 1) >> 28, R)
    assert out["omega5"] == mont_hex(pow(root, 1 << 23, R)) and out["omega19"] == mont_hex(pow(root, 1 << 9, R))
    assert out["wide_ff"] == mont_hex(int.from_bytes(b"\xff" * 64, "little") % R)
    # commitments enter the transcript in affine form: the host normalisation of both provers agrees
    import numpy as np
    from halo2_lib_b200.prover import g1_normalize_host
    limbs = lambda h: np.frombuffer(bytes.fromhex(h), dtype=np.uint64)
    pt = np.concatenate([limbs(out["squeeze1"]), limbs(out["squeeze2"]), limbs(out["squeeze3"])])
    assert np.array_equal(g1_normalize_host(pt), limbs(out["normalize"]))
    pt0 = pt.copy(); pt0[8:] = 0
    assert not limbs(out["normalize_identity"]).any() and not g1_normalize_host(pt0).any()
    # a batch with one inversion (the identity in the middle): each point as alone
    pt2 = np.concatenate([limbs(out["squeeze3"]), limbs(out["squeeze1"]), limbs(out["squeeze2"])])
    assert np.array_equal(limbs(out["batch0"]), g1_normalize_host(pt)) and not limbs(out["batch1"]).any()
    assert np.array_equal(limbs(out["batch2"]), g1_normalize_host(pt2))


def test_cpp_prover_mirror_compiles_and_links():
    exe = os.path.join(ROOT, "build", "prover_mirror_test")
    libdir = os.path.join(ROOT, "halo2-lib_b200")
    subprocess.check_call([CXX, "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "cpp", "prover_mirror_test.cpp"), "-o", exe,
                           f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])
    assert os.path.exists(exe)

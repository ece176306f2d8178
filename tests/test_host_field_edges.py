"""The prover's host field arithmetic (HostField<Fr / Fq>, HostFr::from_wide_bytes, HostFr::omega and
g1_normalize_host_batch in include/h2b200_prover.hpp) on the raw-limb families of tests/field_edges.py, against plain
Python integers.  CPU only: tests/cpp/host_field_test.cpp answers one request per line."""
import os
import subprocess
import numpy as np
import pytest
import field_edges as fe

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "host_field_test.cpp")
EXE = os.path.join(ROOT, "build", "host_field_test")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
H = lambda v: f"{v:064x}"
N_PATTERN = 4096


@pytest.fixture(scope="module")
def run():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    libdir = os.path.join(ROOT, "halo2-lib_b200")
    subprocess.check_call([CXX, "-std=c++17", "-O1", "-Wall", SRC, "-o", EXE, f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])

    def ask(lines):
        out = subprocess.run([EXE], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True, timeout=600).stdout
        res = [l.split() for l in out.splitlines()]
        assert len(res) == len(lines)
        return [[int(v, 16) for v in r[1:]] for r in res]
    return ask


def _check(requests, got, want, what):
    bad = [i for i in range(len(want)) if got[i] != want[i]]
    assert not bad, (f"{what}: {len(bad)} of {len(want)} wrong; first: {requests[bad[0]]} -> "
                     f"{' '.join(map(H, got[bad[0]]))}, want {' '.join(map(H, want[bad[0]]))}")


@pytest.mark.parametrize("field", ["Fq", "Fr"])
def test_host_field_mul_add_on_raw_limb_edges(run, field):
    """mul and add of HostField on every ordered pair of the fixed family, on limb-pattern pairs, on pairs close to m,
    and on products and sums aimed at both sides of the final subtraction"""
    m = fe.FIELDS[field][1]
    f = field[1].lower()
    s = fe.samples(field)
    for op, name in ((0, "mul"), (1, "add")):
        tuples = [t for g, ts in s[op].items() if g != "pattern" for t in ts] + s[op]["pattern"][:N_PATTERN]
        req = [f"{name} {f} {H(a)} {H(b)}" for a, b in tuples]
        _check(req, run(req), [[fe.reference(op, m, t)] for t in tuples], f"{field} {name}")


@pytest.mark.parametrize("field", ["Fq", "Fr"])
def test_host_field_pow_inv_from_canonical(run, field):
    m = fe.FIELDS[field][1]
    f = field[1].lower()
    rinv = pow(fe.W, -1, m)
    fixed = fe.fixed_family(m)
    s = fe.samples(field)[3]
    vals = fe.checked(fixed + [t[0] for t in fe.inversion_samples(m) + s["pattern"][:N_PATTERN // 2] + s["near m"][:256]], m)
    exps = [0, 1, 2, 3, 1234567, (1 << 64) - 1, 1 << 63]
    req, want = [], []
    for a in fixed:
        for e in exps:
            req.append(f"pow {f} {H(a)} {e:x}")
            want.append([pow(a * rinv % m, e, m) * fe.W % m])
    for a in vals:
        req.append(f"inv {f} {H(a)}")
        want.append([fe.reference(3, m, (a,))])
        req.append(f"canon {f} {H(a)}")
        want.append([a * fe.W % m])
    _check(req, run(req), want, f"{field} pow / inv / from_canonical")


def test_host_from_wide_bytes(run):
    """the transcript's challenge: 64 bytes -> (lo + hi 2^256) mod r, Montgomery form; each half up to 2^256 - 1 takes up
    to five subtractions before the products"""
    r = fe.R
    rng = np.random.default_rng(64)
    halves = [0, r - 1, r, r + 1, 2 * r, 5 * r, (1 << 256) - 1] + [int.from_bytes(rng.bytes(32), "little") for _ in range(3)]
    req, want = [], []
    for lo in halves:
        for hi in halves:
            d = lo.to_bytes(32, "little") + hi.to_bytes(32, "little")
            req.append(f"wide {d.hex()}")
            want.append([(lo + (hi << 256)) % r * fe.W % r])
    _check(req, run(req), want, "from_wide_bytes")


def test_host_omega_every_k(run):
    r = fe.R
    root = pow(7, (r - 1) >> 28, r)
    req = [f"omega {k}" for k in range(29)]
    want = [[pow(root, 1 << (28 - k), r) * fe.W % r] for k in range(29)]
    got = run(req)
    _check(req, got, want, "omega")
    for k in range(1, 29):  # and each is a primitive 2^k-th root
        w = got[k][0] * pow(fe.W, -1, r) % r
        assert pow(w, 1 << k, r) == 1 and pow(w, 1 << (k - 1), r) == r - 1, k


def test_host_normalize_batch_identity_positions(run):
    """g1_normalize_host_batch (one inversion per batch): identities first, last, everywhere, or alone, and z with raw
    limb patterns"""
    p = fe.P
    rinv = pow(fe.W, -1, p)
    rng = np.random.default_rng(65)
    zs = [z for z in fe.fixed_family(p) if z] + fe.pattern_family(p, 32, 66)
    rnd = lambda: int.from_bytes(rng.bytes(32), "little") % p
    pt = lambda i: (rnd(), rnd(), zs[i % len(zs)])
    ident = (rnd(), rnd(), 0)
    batches = [[ident, pt(0), pt(1)], [pt(2), pt(3), ident], [ident] * 4, [ident], [pt(4)], [],
               [pt(i) for i in range(len(zs))], [ident if i % 3 == 0 else pt(i) for i in range(20)]]

    def norm(x, y, z):
        if z == 0:
            return [0, 0, 0]
        zi = pow(z * rinv % p, -1, p)
        return [x * rinv * zi * zi % p * fe.W % p, y * rinv * zi * zi * zi % p * fe.W % p, fe.W % p]
    req = [f"norm {len(b)} " + " ".join(H(v) for q in b for v in q) for b in batches]
    want = [[v for q in b for v in norm(*q)] for b in batches]
    _check(req, run(req), want, "g1_normalize_host_batch")

"""Plain-integer restatement of the params gen_srs creates (halo2-base/src/utils/mod.rs:413-443:
ParamsKZG::setup(k, ChaCha20Rng::from_seed(seed)) and ParamsKZG::write), on top of oracle/pyref.py's BN254 G1 and Fr: the
ChaCha20 block function and rand_chacha's fill_bytes, Fr::from_uniform_bytes, Fq2 and the G2 twist (affine double-and-add,
compressed and raw encodings) and the params image.  Test infrastructure only, like the other *_oracle modules here."""
from __future__ import annotations
from oracle.pyref import P, R, G1, g1_mul, g1_compress, omega_for, to_mont, from_mont

# rand_chacha 0.3, halo2curves-axiom 0.7.3 and halo2-axiom 0.5.3 are not vendored; the conventions below are
# recalled (DESIGN.md §2) and restated with no regard for speed.
M32 = 0xFFFFFFFF


def chacha20_block(key: bytes, counter: int) -> list[int]:
    """the ChaCha20 block function (RFC 7539 §2.3, 20 rounds) with rand_chacha's layout: 64-bit block counter in words 12-13,
    stream 0 in words 14-15; returns 16 words"""
    rotl = lambda v, s: ((v << s) | (v >> (32 - s))) & M32
    s = [0x61707865, 0x3320646E, 0x79622D32, 0x6B206574] + [int.from_bytes(key[4 * i:4 * i + 4], "little") for i in range(8)]
    s += [counter & M32, counter >> 32, 0, 0]
    x = list(s)

    def qr(a, b, c, d):
        x[a] = (x[a] + x[b]) & M32; x[d] = rotl(x[d] ^ x[a], 16)
        x[c] = (x[c] + x[d]) & M32; x[b] = rotl(x[b] ^ x[c], 12)
        x[a] = (x[a] + x[b]) & M32; x[d] = rotl(x[d] ^ x[a], 8)
        x[c] = (x[c] + x[d]) & M32; x[b] = rotl(x[b] ^ x[c], 7)
    for _ in range(10):
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
    return [(a + b) & M32 for a, b in zip(x, s)]


def chacha20_fill_bytes(seed: bytes, n: int) -> bytes:
    """`ChaCha20Rng::from_seed(seed).fill_bytes(&mut [0; n])` on a fresh generator: the words of blocks 0, 1, .. in order,
    each little-endian"""
    out = b""
    block = 0
    while len(out) < n:
        out += b"".join(w.to_bytes(4, "little") for w in chacha20_block(seed, block))
        block += 1
    return out[:n]


def from_uniform_bytes(b: bytes) -> int:
    """Fr::from_uniform_bytes(64 bytes): (lo + hi 2^256) mod r, i.e. the 512-bit little-endian integer mod r"""
    assert len(b) == 64
    return int.from_bytes(b, "little") % R


def seeded_tau(seed: bytes = bytes(32)) -> int:
    """the tau of ParamsKZG::setup(k, ChaCha20Rng::from_seed(seed)): its first draw, Fr::random"""
    return from_uniform_bytes(chacha20_fill_bytes(seed, 64))


# Fq2 = Fq[u] / (u^2 + 1) as (c0, c1)
def f2_add(a, b):
    return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)


def f2_sub(a, b):
    return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)


def f2_mul(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def f2_inv(a):
    t = pow(a[0] * a[0] + a[1] * a[1], -1, P)
    return (a[0] * t % P, -a[1] * t % P)


def f2_pow(a, e: int):
    acc = (1, 0)
    while e:
        if e & 1:
            acc = f2_mul(acc, a)
        a = f2_mul(a, a)
        e >>= 1
    return acc


def f2_sqrt(a):
    """a square root in Fq2 (p = 3 mod 4: Adj & Rodriguez-Henriquez, Algorithm 9), None for a non-residue"""
    if a == (0, 0):
        return (0, 0)
    a1 = f2_pow(a, (P - 3) // 4)
    alpha = f2_mul(f2_mul(a1, a1), a)
    x0 = f2_mul(a1, a)
    if alpha == (P - 1, 0):
        x = f2_mul((0, 1), x0)
    else:
        x = f2_mul(f2_pow(f2_add((1, 0), alpha), (P - 1) // 2), x0)
    return x if f2_mul(x, x) == a else None


G2_B = f2_mul((3, 0), f2_inv((9, 1)))  # the twist y^2 = x^3 + 3 / (9 + u)
G2 = ((0x1800DEEF121F1E76426A00665E5C4479674322D4F75EDADD46DEBD5CD992F6ED, 0x198E9393920D483A7260BFB731FB5D25F1AA493335A9E71297E485B7AEF312C2),
      (0x12C85EA5DB8C6DEB4AAB71808DCB408FE3D1E7690C43D37B4CE6CC0166FA7DAA, 0x090689D0585FF075EC9E99AD690C3395BC4B313370B38EF355ACDADCD122975B))  # EIP-197


def g2_is_on_curve(pt) -> bool:
    if pt is None:
        return True
    x, y = pt
    return f2_mul(y, y) == f2_add(f2_mul(f2_mul(x, x), x), G2_B)


def g2_add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    (x1, y1), (x2, y2) = a, b
    if x1 == x2:
        if f2_add(y1, y2) == (0, 0):
            return None
        xx = f2_mul(x1, x1)
        lam = f2_mul(f2_add(f2_add(xx, xx), xx), f2_inv(f2_add(y1, y1)))
    else:
        lam = f2_mul(f2_sub(y2, y1), f2_inv(f2_sub(x2, x1)))
    x3 = f2_sub(f2_sub(f2_mul(lam, lam), x1), x2)
    return (x3, f2_sub(f2_mul(lam, f2_sub(x1, x3)), y1))


def g2_mul(k: int, a):
    """affine double-and-add, most significant bit first (k is not reduced: r * g2 must come out as the identity)"""
    acc = None
    for bit in bin(k)[2:] if k > 0 else "":
        acc = g2_add(acc, acc)
        if bit == "1":
            acc = g2_add(acc, a)
    return acc


def _sgn0(y) -> int:
    """sgn0 of an Fq2 element: the parity of c0, or of c1 when c0 = 0"""
    return (y[0] & 1) if y[0] else (y[1] & 1)


def g2_compress(pt) -> bytes:
    """G2Affine::to_bytes (SerdeFormat::Processed): x.c0 | x.c1 canonical little-endian; byte 63 bit 7 = identity, bit 6 =
    sgn0(y)"""
    if pt is None:
        return bytes(63) + bytes([0x80])
    b = bytearray(pt[0][0].to_bytes(32, "little") + pt[0][1].to_bytes(32, "little"))
    b[63] |= _sgn0(pt[1]) << 6
    return bytes(b)


def g2_decompress(b: bytes):
    """inverse of g2_compress; returns (point, ok)"""
    inf, sign = b[63] >> 7, (b[63] >> 6) & 1
    x0 = int.from_bytes(b[:32], "little")
    x1 = int.from_bytes(b[32:63] + bytes([b[63] & 0x3F]), "little")
    if inf:
        return None, (x0 == 0 and x1 == 0 and sign == 0)
    if x0 >= P or x1 >= P:
        return None, False
    y = f2_sqrt(f2_add(f2_mul(f2_mul((x0, x1), (x0, x1)), (x0, x1)), G2_B))
    if y is None:
        return None, False
    if _sgn0(y) != sign:
        y = f2_sub((0, 0), y)
    return ((x0, x1), y), True


def _mont_bytes(v: int, m: int) -> bytes:
    return to_mont(v, m).to_bytes(32, "little")


def g2_raw(pt) -> bytes:
    """SerdeFormat::RawBytes: x.c0 | x.c1 | y.c0 | y.c1, Montgomery limbs; the identity (0, 0)"""
    if pt is None:
        return bytes(128)
    return b"".join(_mont_bytes(v, P) for v in (pt[0][0], pt[0][1], pt[1][0], pt[1][1]))


def g2_from_raw(b: bytes):
    v = [from_mont(int.from_bytes(b[32 * i:32 * i + 32], "little"), P) for i in range(4)]
    return None if not any(v) else ((v[0], v[1]), (v[2], v[3]))


def g1_raw(pt) -> bytes:
    """SerdeFormat::RawBytes G1: x | y, Montgomery limbs; the identity (0, 0)"""
    return bytes(64) if pt is None else _mont_bytes(pt[0], P) + _mont_bytes(pt[1], P)


def lagrange_scalars(tau: int, k: int) -> list[int]:
    """L_i(tau) on the 2^k domain: (tau^n - 1) / n * omega^i / (tau - omega^i)"""
    n = 1 << k
    w = omega_for(k)
    c = (pow(tau, n, R) - 1) * pow(n, -1, R) % R
    return [c * pow(w, i, R) * pow((tau - pow(w, i, R)) % R, -1, R) % R for i in range(n)]


def params_setup(k: int, tau: int):
    """ParamsKZG::setup for a given tau: (g, g_lagrange, g2, s_g2) as affine points"""
    g = [g1_mul(pow(tau, i, R), G1) for i in range(1 << k)]
    gl = [g1_mul(l, G1) for l in lagrange_scalars(tau, k)]
    return g, gl, G2, g2_mul(tau, G2)


def params_image(k: int, g, g_lagrange, g2, s_g2, processed: bool = True) -> bytes:
    """ParamsKZG::write(SerdeFormat::Processed / RawBytes): u32 LE k | g | g_lagrange | g2 | s_g2"""
    p1, p2 = (g1_compress, g2_compress) if processed else (g1_raw, g2_raw)
    return k.to_bytes(4, "little") + b"".join(p1(p) for p in list(g) + list(g_lagrange)) + p2(g2) + p2(s_g2)

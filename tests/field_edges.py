"""Operand families for the field arithmetic, and its reference on plain Python integers.

Every kernel inlines the Montgomery routines of csrc/field.cuh and the prover's host code has its own copy (`HostField` in
include/h2b200_prover.hpp); both work on the raw limbs of a value.  Edge *integers* passed through `mont()` give limbs that
look random, so the families here are built on the raw limbs themselves: small raw values, values just below the modulus,
saturated and cleared limbs, a top limb equal to the modulus's, and bit 31 of a limb set in chosen patterns (where the
squaring's doubled limbs carry into the next limb).

Products are also aimed at the final conditional subtraction (`reduce_once`).  A CIOS product leaves
t = (S + M m) / 2^256 before that subtraction, with S = a b (+ c d for the fused two-product routine) and
M = -S m^-1 mod 2^256; the word-by-word loop builds the same M.  Solving for the second operand so that the result is a
chosen small value δ puts t in [m, m + 2^32) (the subtraction is taken); a result just below m puts t just below m (it
is not).  `unreduced` returns t so that a test can tell which side a sample is on.

Nothing here reuses oracle/: its C code shares the limb-level approach.  Every value handed out is < m: `inv_bgcd` on a
raw value equal to m would never terminate."""
from __future__ import annotations
import functools
import numpy as np

P = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47  # Fq
R = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001  # Fr
FIELDS = {"Fq": (0, P), "Fr": (1, R)}  # name -> (field index of h2b_test_field_op, modulus)
W = 1 << 256  # the Montgomery radix
OPS = {0: "mul", 1: "add", 2: "sub", 3: "inv", 4: "from_mont", 5: "to_mont", 6: "sqr", 7: "a*b+(a+b)(a-b)",
       8: "a*b-b*b", 9: "inv_bgcd", 10: "a*b+c*d"}
ARITY = {0: 2, 1: 2, 2: 2, 3: 1, 4: 1, 5: 1, 6: 1, 7: 2, 8: 2, 9: 1, 10: 4}
PRODUCT_OPS = (0, 4, 5, 6, 7, 8, 10)  # the ops that end in one CIOS reduction and `reduce_once`
TARGETS = lambda m: [1, 2, (1 << 32) - 1, m - 1, m - 2, m - (1 << 32)]  # results aimed at on both sides of the subtraction
LIMB_PATTERNS = [0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF]  # plus a uniform draw as the seventh choice
N_PATTERN = 1 << 18


def limb(m: int, j: int) -> int:
    """32-bit limb j of m (MOD(j) in field.cuh)"""
    return (m >> (32 * j)) & 0xFFFFFFFF


def checked(vals, m: int) -> list[int]:
    vals = [int(v) for v in vals]
    bad = [v for v in vals if not 0 <= v < m]
    if bad:  # a raw m in inv_bgcd loops forever; anything >= m is outside every routine's contract
        raise ValueError(f"operand out of range [0, m): {bad[0]:#x}")
    return vals


# ------------------------------------------------------------------------------------------------ conversions
def to_limbs(vals) -> np.ndarray:
    """ints -> n x 4 uint64 (the [u64;4] little-endian layout)"""
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint64).reshape(-1, 4).copy()


def from_limbs(arr) -> list[int]:
    b = np.ascontiguousarray(arr, dtype=np.uint64).tobytes()
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


# ------------------------------------------------------------------------------------------------ square roots
def sqrt_mod(x: int, m: int) -> int | None:
    """a square root of x mod m, or None when x is not a square (m = 3 mod 4: one power; else Tonelli-Shanks)"""
    x %= m
    if x == 0:
        return 0
    if pow(x, (m - 1) // 2, m) != 1:
        return None
    if m % 4 == 3:
        return pow(x, (m + 1) // 4, m)
    q, s = m - 1, 0
    while q % 2 == 0:
        q, s = q // 2, s + 1
    z = 2
    while pow(z, (m - 1) // 2, m) != m - 1:
        z += 1
    c, t, r = pow(z, q, m), pow(x, q, m), pow(x, (q + 1) // 2, m)
    while t != 1:
        i, t2 = 0, t
        while t2 != 1:
            t2, i = t2 * t2 % m, i + 1
        b = pow(c, 1 << (s - i - 1), m)
        s, c = i, b * b % m
        t, r = t * c % m, r * b % m
    return r


# ------------------------------------------------------------------------------------------------ reference
def neg(x: int, m: int) -> int:
    return (m - x) % m


@functools.lru_cache(maxsize=None)
def consts(m: int) -> tuple[int, int, int]:
    """(R^-1 mod m, R^2 mod m, m^-1 mod 2^256)"""
    return pow(W, -1, m), W * W % m, pow(m, -1, W)


def product_terms(op: int, m: int, ops: tuple) -> list[tuple[int, int]]:
    """the operand pairs whose products one CIOS reduction sums, as the kernel forms them"""
    a = ops[0]
    if op == 0:
        return [(a, ops[1])]
    if op == 4:
        return [(a, 1)]
    if op == 5:
        return [(a, consts(m)[1])]
    if op == 6:
        return [(a, a)]
    if op == 7:
        b = ops[1]
        return [(a, b), ((a + b) % m, (a - b) % m)]
    if op == 8:
        b = ops[1]
        return [(a, b), (neg(b, m), b)]
    if op == 10:
        return [(a, ops[1]), (ops[2], ops[3])]
    raise ValueError(op)


def unreduced(op: int, m: int, ops: tuple) -> int:
    """t, the value before the final conditional subtraction (a + b for add; a CIOS product's (S + M m) / 2^256)"""
    if op == 1:
        return ops[0] + ops[1]
    s = sum(x * y for x, y in product_terms(op, m, ops))
    mm = (-s * consts(m)[2]) % W
    assert (s + mm * m) % W == 0
    return (s + mm * m) // W


def reference(op: int, m: int, ops: tuple) -> int:
    """the raw result limbs of op on raw operand limbs, as an integer < m"""
    a = ops[0]
    if op == 1:
        return (a + ops[1]) % m
    if op == 2:
        return (a - ops[1]) % m
    if op in (3, 9):  # (a R^-1)^-1 R = R^2 / a; inv(0) = 0
        return pow(a, -1, m) * consts(m)[1] % m if a else 0
    return sum(x * y for x, y in product_terms(op, m, ops)) * consts(m)[0] % m


def reference_many(op: int, m: int, tuples: list[tuple]) -> list[int]:
    """`reference` over a list; inversions share one modular inverse (Montgomery's trick) instead of one each"""
    if op not in (3, 9):
        return [reference(op, m, t) for t in tuples]
    vals = [t[0] for t in tuples]
    pref, acc = [], 1
    for v in vals:
        pref.append(acc)
        if v:
            acc = acc * v % m
    inv, out = pow(acc, -1, m), [0] * len(vals)
    r2 = consts(m)[1]
    for i in range(len(vals) - 1, -1, -1):
        if vals[i]:
            out[i] = inv * pref[i] % m * r2 % m
            inv = inv * vals[i] % m
    return out


# ------------------------------------------------------------------------------------------------ families
def fixed_family(m: int) -> list[int]:
    """about 50 raw values: small, just below m, the Montgomery constants, 2^(32j) - 1 and 2^(32j), one saturated limb,
    and prefixes of m (its top limbs with the rest cleared, or with the next limb one lower and the rest saturated)"""
    one = W % m
    v = [0, 1, 2, 3, m - 1, m - 2, m - (1 << 32), m - (1 << 64), (m - 1) // 2, (m + 1) // 2, one, m - one, W * W % m, 1 << 253]
    v += [(1 << (32 * j)) - 1 for j in range(1, 8)] + [1 << (32 * j) for j in range(1, 8)]
    v += [0xFFFFFFFF << (32 * j) for j in range(7)]
    for k in range(1, 8):
        top = (m >> (32 * (8 - k))) << (32 * (8 - k))
        v.append(top)
        j = 7 - k
        v.append(top + ((limb(m, j) - 1) << (32 * j)) + (1 << (32 * j)) - 1)
    return checked(dict.fromkeys(v), m)


def pattern_family(m: int, n: int, seed: int) -> list[int]:
    """n raw values, each 32-bit limb drawn from LIMB_PATTERNS or uniform, the top limb capped at MOD(7).  Where that leaves
    the value >= m, the walk down from limb 6 either keeps the limb equal to m's and goes on, or lowers it by one and
    stops, so the lower limbs stay saturated; about two thirds of the values have the top limb of m."""
    rng = np.random.default_rng(seed)
    pick = rng.integers(0, 7, size=(n, 8))
    uni = rng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint64)
    L = np.where(pick < 6, np.array(LIMB_PATTERNS, dtype=np.uint64)[np.minimum(pick, 5)], uni)
    L[:, 7] = np.minimum(L[:, 7], limb(m, 7))
    keep_equal = rng.random((n, 8)) < 0.5
    out = []
    for i, row in enumerate(L.tolist()):
        if row[7] == limb(m, 7):
            for j in range(6, -1, -1):
                mj = limb(m, j)
                if row[j] < mj:
                    break
                if row[j] > mj and not (keep_equal[i, j] and j > 0):
                    row[j] = mj - 1
                    break
                row[j] = mj
                if j == 0:  # every limb equal to m's: step to m - 1
                    row[0] = mj - 1
        out.append(sum(x << (32 * j) for j, x in enumerate(row)))
    return checked(out, m)


def near_top_family(m: int, n: int, seed: int) -> list[int]:
    """n raw values m - 1 - u with u uniform below 2^(32j), j = 1..7: both factors of a product this close to m reach
    the largest t a product can have (about 1.19 m)"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        bits = 32 * (1 + i % 7)
        u = int.from_bytes(rng.bytes(32), "little") & ((1 << bits) - 1)
        out.append(m - 1 - u)
    return checked(out, m)


def _bits(rng, m):
    return int.from_bytes(rng.bytes(32), "little") % m


# ------------------------------------------------------------------------------------------------ samples per op
def boundary_samples(op: int, m: int, bases: list[int], seed: int) -> list[tuple]:
    """products whose result is each of TARGETS(m): for a given first operand, solve for the other (for op 6 a square
    root of δR, both signs; for op 7 the quadratic in a; for op 10 the fourth operand).  Targets without a solution
    are skipped."""
    rng = np.random.default_rng(seed)
    out = []
    # about half the targets have no square root: squaring aims at more of them (-1 is not a square mod p)
    targets = TARGETS(m) + ([j for j in range(3, 40)] + [m - j for j in range(3, 40)] if op == 6 else [])
    for d in targets:
        dr = d * W % m
        if op == 4:
            out.append((dr,))
        elif op == 5:
            out.append((d * pow(W, -1, m) % m,))
        elif op == 6:
            r = sqrt_mod(dr, m)
            if r is not None:
                out += [(r,), (neg(r, m),)]
        for a in bases:
            if a == 0:
                continue
            if op == 0:
                out.append((a, dr * pow(a, -1, m) % m))
            elif op == 7:  # a^2 + a b - b^2 = δR with b given: a = (-b ± sqrt(5 b^2 + 4 δR)) / 2
                b = a
                r = sqrt_mod(5 * b * b + 4 * dr, m)
                if r is not None:
                    inv2 = pow(2, -1, m)
                    out += [((-b + r) * inv2 % m, b), ((-b - r) * inv2 % m, b)]
            elif op == 8:  # a b - b^2 = δR: a = δR / b + b
                out.append(((dr * pow(a, -1, m) + a) % m, a))
            elif op == 10:  # a b + c d = δR: d = (δR - a b) / c, with c = -x as the group law forms it and c near m
                b, x = _bits(rng, m), bases[int(rng.integers(0, len(bases)))]
                for c in (neg(x, m), m - 1 - (_bits(rng, m) >> 200)):
                    if c:
                        out.append((a, b, c, (dr - a * b) * pow(c, -1, m) % m))
    return out


def add_sub_samples(op: int, m: int, bases: list[int]) -> list[tuple]:
    """add: a + b in {m-1, m, m+1, 2m-2}; sub: a - b in {0, -1, -(m-1)} and m-1; op 8 with b in {0, m-1} (neg of 0 and of m-1)"""
    out = []
    for a in bases:
        if op == 1:
            out += [(a, s - a) for s in (m - 1, m, m + 1, 2 * m - 2) if 0 <= s - a < m]
        elif op == 2:
            out += [(a, a)] + ([(a, a + 1)] if a + 1 < m else [])
        elif op == 8:
            out += [(a, 0), (a, m - 1)]
    if op == 2:
        out += [(0, m - 1), (m - 1, 0), (0, 0)]
    return out


def inversion_samples(m: int) -> list[tuple]:
    """raw 1, raw 2^j (long runs of halvings in inv_bgcd), m - 1 and (m + 1) / 2"""
    return [(v,) for v in checked([1] + [1 << j for j in range(1, m.bit_length())] + [m - 1, (m + 1) // 2], m)]


def _quads(m, rng, pool, n, minus_x):
    """n four-operand samples for op 10 drawn from pool; with minus_x, c = -x for a drawn x (the group law's p - s1)"""
    idx = rng.integers(0, len(pool), size=(n, 4))
    return [(pool[i], pool[j], neg(pool[k], m) if minus_x else pool[k], pool[l]) for i, j, k, l in idx.tolist()]


@functools.lru_cache(maxsize=None)
def samples(field: str, n_pattern: int = N_PATTERN) -> dict:
    """op -> {group name -> list of operand tuples} for one field; every operand < m"""
    which, m = FIELDS[field]
    seed = 0xF1E1D + which
    fixed = fixed_family(m)
    pat_a = pattern_family(m, n_pattern, seed)
    pat_b = pattern_family(m, n_pattern, seed + 100)
    near = near_top_family(m, 4096, seed + 200)
    rng = np.random.default_rng(seed + 300)
    bases = fixed + pat_a[:48] + near[:16]
    out = {}
    for op in OPS:
        g = {}
        if ARITY[op] == 1:
            g["fixed"] = [(a,) for a in fixed]
            g["pattern"] = [(a,) for a in pat_a]
            g["near m"] = [(a,) for a in near]
        elif ARITY[op] == 2:
            g["fixed pairs"] = [(a, b) for a in fixed for b in fixed]
            g["pattern"] = list(zip(pat_a, pat_b))
            g["near m"] = list(zip(near, near[1:] + near[:1]))
        else:
            k = len(fixed)
            g["fixed pairs"] = [(a, b, neg(b, m), fixed[(i + j + 1) % k]) for i, a in enumerate(fixed) for j, b in enumerate(fixed)]
            g["pattern"] = list(zip(pat_a, pat_b, pat_b[1:] + pat_b[:1], pat_a[7:] + pat_a[:7]))
            g["near m"] = _quads(m, rng, near, 4096, False)  # ab + cd close to 2 m^2: the largest t of the fused routine
            g["c = -x"] = _quads(m, rng, fixed + pat_a[:200], 4096, True)
        if op in PRODUCT_OPS:
            g["boundary"] = boundary_samples(op, m, bases, seed + 400 + op)
        if op in (1, 2, 8):
            g["add/sub boundary"] = add_sub_samples(op, m, fixed + pat_a[:64] + near[:16])
        if op in (3, 9):
            g["boundary"] = inversion_samples(m)
        for name, tuples in g.items():
            for t in tuples:
                checked(t, m)
        out[op] = g
    return out


def pack(op: int, tuples: list[tuple]) -> tuple[np.ndarray, np.ndarray | None]:
    """operand tuples -> (a, b) of h2b_test_field_op: op 10 stacks (a, c) and (b, d) as 2n rows each"""
    if ARITY[op] == 1:
        return to_limbs([t[0] for t in tuples]), None
    if ARITY[op] == 2:
        return to_limbs([t[0] for t in tuples]), to_limbs([t[1] for t in tuples])
    return (to_limbs([t[0] for t in tuples] + [t[2] for t in tuples]),
            to_limbs([t[1] for t in tuples] + [t[3] for t in tuples]))


def first_mismatch(op: int, field: str, group: str, tuples: list[tuple], got: list[int], want: list[int]) -> str | None:
    """None when got == want, else a message naming the op, the field and the first failing operands in hex"""
    if got == want:
        return None
    bad = [i for i in range(len(want)) if got[i] != want[i]]
    i = bad[0]
    m = FIELDS[field][1]
    side = ""
    if op in PRODUCT_OPS or op == 1:
        t = unreduced(op, m, tuples[i])
        side = f"; t = {t:#066x} ({'>=' if t >= m else '<'} m)"
    operands = ", ".join(f"{v:#066x}" for v in tuples[i])
    return (f"op {op} ({OPS[op]}) on {field}, {group}: {len(bad)} of {len(want)} wrong; first at #{i}: operands (raw limbs) "
            f"{operands} -> got {got[i]:#066x}, want {want[i]:#066x}{side}")


# ------------------------------------------------------------------------------------------------ curve points
def curve_points(raw_xs: list[int], limit: int) -> list[tuple[int, int]]:
    """affine points (x, y), canonical, whose Montgomery x limbs are the given raw values: x = x_raw R^-1 with x^3 + 3 a
    square mod p; both signs of y.  Up to `limit` points."""
    rinv = pow(W, -1, P)
    pts = []
    for xr in checked(raw_xs, P):
        x = xr * rinv % P
        y = sqrt_mod(x * x * x + 3, P)
        if y is None:
            continue
        pts += [(x, y), (x, neg(y, P))] if y else [(x, 0)]
        if len(pts) >= limit:
            break
    return pts[:limit]

"""oracle/pyref.py — pure-Python big-int restatement of the BN254 arithmetic on the create_proof hot path.

TEST INFRASTRUCTURE ONLY.  Nothing outside `tests/`, `__graft_entry__.smoke()` and
`bench.py`'s cpu_baseline / `--impl reference` legs may import this module.  The product
path (halo2-lib_b200/) never routes through it.

PARITY STATUS: **unpinned by reference goldens.**  The arithmetic restated here lives in
third-party crates that are NOT vendored in the reference tree:
  * halo2curves-axiom 0.7.3 (Cargo.lock:1185-1188): bn256::{Fr,Fq,G1,G1Affine}, msm::best_multiexp
  * halo2-axiom 0.5.3 @5e4f0e5 (Cargo.lock:1063-1065): arithmetic::best_fft,
    poly::EvaluationDomain::{lagrange_to_coeff, coeff_to_extended, extended_to_coeff},
    poly::kzg::commitment::ParamsKZG::{commit, commit_lagrange, setup}
The reference tree holds no golden vector for any of them (SURVEY.md §4, §8c).  What pins this
file instead: (1) the outputs are mathematically unique (group element / field element), so any
correct implementation is bit-identical after canonicalisation; (2) the public BN254 (alt_bn128)
constants and the EIP-196 doubling vector `2·(1,2)` checked in tests/test_oracle_kat.py;
(3) cross-checks between this file (Python ints, textbook formulas) and the independent C
restatement oracle/bn254_oracle.c (Montgomery limbs, Jacobian formulas, Pippenger, radix-2 NTT).

Reference call sites this path is reached from:
  create_proof      halo2-base/src/utils/testing.rs:40-48
  keygen_vk/pk      halo2-base/src/utils/testing.rs:224,227 ; utils/halo2.rs:135
  ParamsKZG::setup  halo2-base/src/utils/mod.rs:439-443
  [u64;4] LE limbs  halo2-base/src/utils/mod.rs:332-377
  assign_witnesses  halo2-base/src/gates/flex_gate/threads/single_phase.rs:273-312
  lookup copy       halo2-base/src/virtual_region/lookups.rs:130-155
"""
from __future__ import annotations

# ---------------------------------------------------------------- constants (SURVEY.md §8c)
P = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47  # Fq
R = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001  # Fr
S = 28  # Fr two-adicity
GENERATOR = 7  # Fr multiplicative generator (halo2curves bn256::Fr::MULTIPLICATIVE_GENERATOR)
ROOT_OF_UNITY = pow(GENERATOR, (R - 1) >> S, R)  # primitive 2^28-th root
ZETA = 0x30644E72E131A029048B6E193FD84104CC37A73FEC2BC5E9B8CA0B2D36636F23  # Fr cube root of unity
B = 3  # y^2 = x^3 + 3
G1 = (1, 2)
MONT_R = 1 << 256


def to_mont(x: int, m: int) -> int:
    return (x * MONT_R) % m


def from_mont(x: int, m: int) -> int:
    return (x * pow(MONT_R, -1, m)) % m


def limbs(x: int) -> list[int]:
    """[u64;4] little-endian limbs (halo2-base/src/utils/mod.rs:332-377 contract)."""
    return [(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)]


def from_limbs(l) -> int:
    return sum(int(v) << (64 * i) for i, v in enumerate(l))


# ---------------------------------------------------------------- G1 (affine, None = identity)
def is_on_curve(pt) -> bool:
    if pt is None:
        return True
    x, y = pt
    return (y * y - x * x * x - B) % P == 0


def g1_add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    x1, y1 = a
    x2, y2 = b
    if x1 == x2:
        if (y1 + y2) % P == 0:
            return None
        lam = (3 * x1 * x1) * pow(2 * y1, -1, P) % P
    else:
        lam = (y2 - y1) * pow(x2 - x1, -1, P) % P
    x3 = (lam * lam - x1 - x2) % P
    y3 = (lam * (x1 - x3) - y1) % P
    return (x3, y3)


def g1_neg(a):
    return None if a is None else (a[0], (-a[1]) % P)


def g1_compress(pt) -> bytes:
    """halo2curves `G1Affine::to_bytes` as `ParamsKZG::write` emits it in SerdeFormat::Processed (reference call sites
    halo2-base/src/utils/mod.rs:401-435; halo2curves-axiom 0.7.3 not vendored — flag positions recalled): 32 bytes, x
    little-endian; last byte bit 7 = identity, bit 6 = parity of y."""
    if pt is None:
        return bytes(31) + bytes([0x80])
    b = bytearray(pt[0].to_bytes(32, "little"))
    b[31] |= (pt[1] & 1) << 6
    return bytes(b)


def g1_decompress(b: bytes):
    """inverse of g1_compress; returns (point, ok).  y = (x^3 + 3)^((p+1)/4) since p = 3 mod 4."""
    inf, odd = b[31] >> 7, (b[31] >> 6) & 1
    x = int.from_bytes(b[:31] + bytes([b[31] & 0x3F]), "little")
    if inf:
        return None, (x == 0 and odd == 0)
    if x >= P:
        return None, False
    rhs = (x * x * x + B) % P
    y = pow(rhs, (P + 1) // 4, P)
    if y * y % P != rhs:
        return None, False
    if (y & 1) != odd:
        y = P - y
    return (x, y), True


def g1_mul(k: int, a):
    k %= R
    acc = None
    while k:
        if k & 1:
            acc = g1_add(acc, a)
        a = g1_add(a, a)
        k >>= 1
    return acc


def msm_naive(scalars, bases):
    """Definition of best_multiexp: sum_i s_i * P_i (halo2curves-axiom 0.7.3 msm::best_multiexp)."""
    acc = None
    for s, b in zip(scalars, bases):
        acc = g1_add(acc, g1_mul(s, b))
    return acc


# ---------------------------------------------------------------- Fr NTT (definitions)
def omega_for(k: int) -> int:
    """EvaluationDomain omega for 2^k rows: ROOT_OF_UNITY^(2^(S-k)) (SURVEY.md App. B)."""
    assert 0 <= k <= S
    return pow(ROOT_OF_UNITY, 1 << (S - k), R)


def dft(a, omega):
    """best_fft's contract: natural in, natural out, out[i] = sum_j a[j] * omega^(i*j)."""
    n = len(a)
    return [sum(a[j] * pow(omega, i * j, R) for j in range(n)) % R for i in range(n)]


def ntt(a, omega):
    """Recursive radix-2 (same output as dft)."""
    n = len(a)
    if n == 1:
        return list(a)
    e = ntt(a[0::2], omega * omega % R)
    o = ntt(a[1::2], omega * omega % R)
    out = [0] * n
    w = 1
    for i in range(n // 2):
        t = w * o[i] % R
        out[i] = (e[i] + t) % R
        out[i + n // 2] = (e[i] - t) % R
        w = w * omega % R
    return out


def lagrange_to_coeff(evals, k):
    n = 1 << k
    assert len(evals) == n
    ninv = pow(n, -1, R)
    return [x * ninv % R for x in ntt(evals, pow(omega_for(k), -1, R))]


def coeff_to_extended(coeffs, k, ext_k):
    """EvaluationDomain::coeff_to_extended: a[i] *= zeta^(i mod 3); zero-pad; FFT(extended_omega)."""
    zp = [1, ZETA, ZETA * ZETA % R]
    a = [c * zp[i % 3] % R for i, c in enumerate(coeffs)] + [0] * ((1 << ext_k) - len(coeffs))
    return ntt(a, omega_for(ext_k))


def extended_to_coeff(ext, k, ext_k, quotient_poly_degree=None):
    """EvaluationDomain::extended_to_coeff: iFFT, scale, a[i] *= zeta^-(i mod 3), truncate."""
    n_ext = 1 << ext_k
    ninv = pow(n_ext, -1, R)
    a = [x * ninv % R for x in ntt(ext, pow(omega_for(ext_k), -1, R))]
    zp = [1, ZETA * ZETA % R, ZETA]
    a = [c * zp[i % 3] % R for i, c in enumerate(a)]
    if quotient_poly_degree is not None:
        a = a[: (1 << k) * quotient_poly_degree]
    return a


# ---------------------------------------------------------------- witness assignment
def assign_witnesses(threads, break_points, num_cols, n_rows):
    """Literal restatement of assign_witnesses
    (halo2-base/src/gates/flex_gate/threads/single_phase.rs:273-312).
    `threads`: list of lists of ints (ctx.advice).  Returns num_cols columns of n_rows ints
    (unassigned rows = 0, as WitnessCollection initialises advice to zero)."""
    cols = [[0] * n_rows for _ in range(num_cols)]
    if num_cols == 0:
        assert sum(len(t) for t in threads) == 0, "Trying to assign threads in a phase with no columns"
        return cols
    bps = iter(break_points)
    bp = next(bps, None)
    gate_index = 0
    row_offset = 0
    for ctx in threads:
        for advice in ctx:
            cols[gate_index][row_offset] = advice
            if bp is not None and bp == row_offset:
                bp = next(bps, None)
                row_offset = 0
                gate_index += 1
                cols[gate_index][row_offset] = advice  # IndexError == Rust panic (out of columns)
            row_offset += 1
    return cols


def break_points_for(threads_lens_and_selectors, max_rows, rotations=4):
    """assign_with_constraints' break-point rule (single_phase.rs:193-263, condition at :229).
    `threads_lens_and_selectors`: list of per-thread selector lists (bools, one per advice cell)."""
    bps = []
    row_offset = 0
    for sel in threads_lens_and_selectors:
        for q in sel:
            if (q and row_offset + rotations > max_rows) or row_offset >= max_rows - 1:
                bps.append(row_offset)
                row_offset = 0
            row_offset += 1
    return bps


def assign_lookups(values, num_lookup_cols, n_rows):
    """LookupAnyManager::assign_raw (halo2-base/src/virtual_region/lookups.rs:130-155):
    j-th looked-up value -> column j mod L, row j div L."""
    cols = [[0] * n_rows for _ in range(num_lookup_cols)]
    for j, v in enumerate(values):
        cols[j % num_lookup_cols][j // num_lookup_cols] = v
    return cols


# ---- quotient h(X) terms and opening arithmetic on plain integers (pins oracle/bn254_oracle.c on small sizes) -------
# halo2-axiom 0.5.3 plonk/evaluation.rs / arithmetic.rs are not vendored; these are the textbook formulas the Rust
# code implements (comments there quote them), written with no regard for speed.
ZETA = pow(pow(7, (R - 1) // 3, R), 2, R)  # Fr::ZETA
DELTA = pow(7, 1 << 28, R)                 # Fr::DELTA = GENERATOR^(2^S)


def eval_polynomial(coeffs, x):
    return sum(c * pow(x, i, R) for i, c in enumerate(coeffs)) % R


def kate_division(a, z):
    """quotient of a(X) by (X - z) by schoolbook long division; remainder dropped"""
    a = list(a)
    q = [0] * (len(a) - 1)
    for i in range(len(a) - 1, 0, -1):
        q[i - 1] = a[i] % R
        a[i - 1] = (a[i - 1] + z * a[i]) % R
    return q


def rotate(col, idx, rot, k, ext_k):
    n = 1 << ext_k
    return col[(idx + rot * (1 << (ext_k - k))) % n]


def permutation_terms(z_sets, columns, sigma, chunk_len, l0, l_last, l_active, beta, gamma, y, blinding_factors, k, ext_k, values):
    n = 1 << ext_k
    w = omega_for(ext_k)
    out = []
    for i in range(n):
        x = ZETA * pow(w, i, R) % R  # the point of the extended coset this row evaluates at
        v = values[i]
        v = (v * y + (1 - z_sets[0][i]) * l0[i]) % R
        zl = z_sets[-1][i]
        v = (v * y + (zl * zl - zl) * l_last[i]) % R
        for s in range(1, len(z_sets)):
            v = (v * y + (z_sets[s][i] - rotate(z_sets[s - 1], i, -(blinding_factors + 1), k, ext_k)) * l0[i]) % R
        for s in range(len(z_sets)):
            left, right = rotate(z_sets[s], i, 1, k, ext_k), z_sets[s][i]
            for c in range(s * chunk_len, min((s + 1) * chunk_len, len(columns))):
                left = left * (columns[c][i] + beta * sigma[c][i] + gamma) % R
                right = right * (columns[c][i] + pow(DELTA, c, R) * beta * x + gamma) % R
            v = (v * y + (left - right) * l_active[i]) % R
        out.append(v)
    return out


def lookup_terms(table_values, z, a, s, l0, l_last, l_active, beta, gamma, y, k, ext_k, values):
    """table_values[i] = (compressed input + beta)(compressed table + gamma) at row i"""
    out = []
    for i in range(1 << ext_k):
        v = values[i]
        v = (v * y + (1 - z[i]) * l0[i]) % R
        v = (v * y + (z[i] * z[i] - z[i]) * l_last[i]) % R
        v = (v * y + (rotate(z, i, 1, k, ext_k) * (a[i] + beta) * (s[i] + gamma) - z[i] * table_values[i]) * l_active[i]) % R
        v = (v * y + (a[i] - s[i]) * l0[i]) % R
        v = (v * y + (a[i] - s[i]) * (a[i] - rotate(a, i, -1, k, ext_k)) * l_active[i]) % R
        out.append(v)
    return out


def graph_row(program, n_calc, result, constants, rotations, fixed, advice, instance, challenges, beta, gamma, theta, y, prev, idx, k,
              ext_k):
    """GraphEvaluator::evaluate for one row on plain integers; program / value-source encoding of include/h2b200.h"""
    inter = []

    def fetch(src):
        kind, index, slot = src & 15, (src >> 4) & 0xFFFF, src >> 20
        if kind == 0:
            return constants[index]
        if kind == 1:
            return inter[index]
        if kind in (2, 3, 4):
            return rotate((fixed, advice, instance)[kind - 2][index], idx, rotations[slot], k, ext_k)
        if kind == 5:
            return challenges[index]
        return {6: beta, 7: gamma, 8: theta, 9: y, 10: prev}[kind]

    pc = 0
    for _ in range(n_calc):
        op = program[pc]
        pc += 1
        if op == 6:
            r, f, np_ = fetch(program[pc]), fetch(program[pc + 1]), program[pc + 2]
            pc += 3
            for _j in range(np_):
                r = (r * f + fetch(program[pc])) % R
                pc += 1
        else:
            a = fetch(program[pc])
            pc += 1
            if op <= 2:
                b = fetch(program[pc])
                pc += 1
                r = (a + b) % R if op == 0 else (a - b) % R if op == 1 else a * b % R
            else:
                r = {3: a * a % R, 4: 2 * a % R, 5: (-a) % R, 7: a}[op]
        inter.append(r)
    assert pc == len(program)
    return fetch(result)


def permute_expression_pair(inputs, table, zcash_order=False):
    """usable rows only, plain integers; returns (A', S') or None for ConstraintSystemFailure.  Left-over table values
    (ascending) fill the repeated rows front to back (PSE / axiom sorted-table walk, the default) or, with zcash_order,
    from the last repeated row backwards (zcash halo2: BTreeMap + pop)."""
    a = sorted(inputs)
    left = {}
    for v in table:
        left[v] = left.get(v, 0) + 1
    s_perm, repeated = [None] * len(a), []
    for row, v in enumerate(a):
        if row == 0 or v != a[row - 1]:
            s_perm[row] = v
            if left.get(v, 0) == 0:
                return None
            left[v] -= 1
        else:
            repeated.append(row)
    leftovers = [v for v in sorted(left) for _ in range(left[v])]
    if len(leftovers) != len(repeated):
        return None
    rows = reversed(repeated) if zcash_order else repeated
    for row, v in zip(rows, leftovers):
        s_perm[row] = v
    return a, s_perm

"""GPU tests of halo2_lib_b200.MockProver (include/h2b200_mock.hpp), MockProver on a halo2-base builder's keygen data: its
reports, break points and q_j / q_lookup columns must equal tests/builder_oracle.py on satisfied builders and with planted
violations, in both witness forms, at k = 8 and 12 for every shape and at the full sizes (k = 19 with one column and the
selector lookup, k = 20 with 11 / 2); at k = 12 it agrees with ProverSession.check on the circuit keygen would build; every
panic of the keygen pass raises H2BError with halo2-base's message and leaves the context usable; the C++ front end gives the
same bytes."""
import os
import subprocess
import numpy as np
import pytest
from oracle import pyref
from util import mont
import builder_oracle as bo

pytestmark = pytest.mark.gpu
R = pyref.R
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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


def _mont_small(ctx, v):
    """canonical values < 2^64 -> Montgomery limbs, on the device"""
    v = np.ascontiguousarray(v, dtype=np.uint64)
    z = np.zeros(len(v), dtype=np.uint64)
    return ctx.field_op(1, 5, np.stack([v, z, z, z], axis=1)) if len(v) else np.zeros((0, 4), dtype=np.uint64)


def _forms(ctx, rng, values, n_rational=300):
    """(evaluated cells, (halo2-base form cells, rational_index, rational_den)): Rational(v d, d) at n_rational cells"""
    cells = _mont_small(ctx, values)
    idx = np.sort(rng.choice(len(values), size=min(n_rational, len(values)), replace=False)).astype(np.uint64)
    d = [int(x) for x in rng.integers(1, 1 << 62, size=len(idx))]
    w = cells.copy()
    w[idx.astype(np.int64)] = mont([int(values[int(i)]) * di % R for i, di in zip(idx, d)], R)
    return cells, (w, idx, mont(d, R))


def _run(mp, b, cells, form=None, max_report=16):
    kw = {} if form is None else {"rational_index": form[1], "rational_den": form[2]}
    return mp.run(cells if form is None else form[0], b["selectors"], b["advice_equalities"],
                  (_mont_small(mp.ctx, b["constants"]), b["constant_index"]), b["lookups"], max_report=max_report, **kw)


def _same(got, want):
    for key in ("gates", "lookups", "equalities", "constants", "equality_cells", "constant_cells", "break_points", "satisfied"):
        assert got[key] == want[key], key


def _nonzero_rows(col):
    return set(np.flatnonzero(col.download().any(axis=1)).tolist())


def _same_columns(mp, want, A):
    one = mont([1], R)[0]
    for j in range(A):
        col = mp.lagr["q%d" % j].download()
        rows = np.flatnonzero(col.any(axis=1))
        assert set(rows.tolist()) == want["q"][j] and (col[rows] == one).all()
    if want["q_lookup"] is not None:
        assert _nonzero_rows(mp.lagr["q_lookup"]) == want["q_lookup"]


@pytest.mark.parametrize("k", [8, 12])
@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_mock_prover_matches_the_oracle(ctx, h2b, k, A, L, sel):
    rng = np.random.default_rng(900 + k + 10 * A + L)
    bits = min(8, k - 2)
    max_rows = (1 << k) - 9
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, contexts=3)
    mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows)
    cells, form = _forms(ctx, rng, b["values"])
    want = bo.run(k, A, L, sel, bits, max_rows, b, b["values"])
    assert want["satisfied"] and (A == 1 or want["break_points"])
    for f in (None, form):
        got = _run(mp, b, cells, f)
        _same(got, want)
        _same_columns(mp, want, A)
    v = bo.plant(rng, b, bits, many=20)
    cells, form = _forms(ctx, rng, v)
    for max_report in (3, 16):
        want = bo.run(k, A, L, sel, bits, max_rows, b, v, max_report=max_report)
        assert not want["satisfied"] and want["equalities"][0] > 3 and want["constants"][0] >= 1
        assert sum(c for c, _ in want["gates"]) >= 1 and (not want["lookups"] or sum(c for c, _ in want["lookups"]) >= 1)
        for f in (None, form):
            _same(_run(mp, b, cells, f, max_report), want)
    mp.free()


@pytest.mark.parametrize("k,A,L,sel,bits", [(19, 1, 0, True, 18), (20, 11, 2, False, 19)])
def test_mock_prover_at_full_size(ctx, h2b, k, A, L, sel, bits):
    """the gates are checked by the oracle at the rows a planted cell reaches (the builder is satisfied elsewhere, as the small
    sizes show over every row); everything else over the whole builder"""
    rng = np.random.default_rng(k)
    max_rows = (1 << k) - 9
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
    mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows)
    v = bo.plant(rng, b, bits, many=40)
    bps = bo.assign_with_constraints(b["contexts"], A, max_rows, record=False)[0]
    rows = {}
    for p in np.flatnonzero(v != b["values"]):
        for q in (int(p), int(p) + 1) if int(p) + 1 < len(v) else (int(p),):  # a break cell also sits at row 0 of the next column
            j, r = bo.raw_cell(bps, q)
            rows.setdefault(j, set()).update(x for x in range(r - 3, r + 1) if x >= 0)
    want = bo.run(k, A, L, sel, bits, max_rows, b, v, gate_rows=rows, record=False)
    assert not want["satisfied"] and want["break_points"] == bps
    cells, form = _forms(ctx, rng, v, 1000)
    for f in (None, form):
        _same(_run(mp, b, cells, f), want)
    _same_columns(mp, want, A)
    mp.free()


def test_errors_carry_halo2_base_messages_and_leave_the_context_usable(ctx, h2b):
    rng = np.random.default_rng(3)
    k, bits = 8, 4
    max_rows = (1 << k) - 9
    b = bo.make_builder(rng, k, 2, 1, False, bits, max_rows)
    cells = _mont_small(ctx, b["values"])
    mp = h2b.MockProver(ctx, k, 2, 1, False, bits, max_rows)
    want = bo.run(k, 2, 1, False, bits, max_rows, b, b["values"])

    def expect(msg, mock=mp, **changes):
        bb = dict(b, **changes)
        with pytest.raises(h2b.H2BError, match=msg):
            _run(mock, bb, cells)
        with pytest.raises(bo.Panic, match=msg):
            bo.run(k, mock.A, mock.L, False, bits, mock.max_rows, dict(bb, contexts=[bb["selectors"]]), b["values"])
        _same(_run(mp, b, cells), want)

    one_col = h2b.MockProver(ctx, k, 1, 1, False, bits, max_rows)
    expect("NOT ENOUGH ADVICE COLUMNS", mock=one_col)
    one_col.free()
    s = np.zeros_like(b["selectors"])
    s[max_rows - 3] = s[max_rows - 4] = 1  # the gate at row max_rows - 3 breaks; the one at max_rows - 4 overlaps it at distance 1
    expect("We do not support overlaps with delta = 1", selectors=s)
    s[max_rows - 4], s[max_rows - 5] = 0, 1
    expect("We do not support overlaps with delta = 2", selectors=s)
    expect("range lookups would be assigned to unusable rows", lookups=np.arange(max_rows + 1, dtype=np.uint64))
    N = len(b["values"])
    e = b["advice_equalities"].copy()
    e[7, 1] = N
    expect("virtual cell not assigned", advice_equalities=e)
    ci = b["constant_index"].copy()
    ci[-1] = N + 5
    expect("virtual cell not assigned", constant_index=ci)
    expect("virtual cell not assigned", lookups=np.concatenate([b["lookups"][:5], [N]]).astype(np.uint64))
    u = (1 << k) - 7
    expect(r"NotEnoughRowsAvailable \{ current_k: 8 \}", constants=np.arange(u + 1, dtype=np.uint64),
           constant_index=np.zeros(u + 1, dtype=np.uint64))
    no_lookup = h2b.MockProver(ctx, k, 2, 0, False, bits, max_rows)
    expect("range lookups require lookup advice columns", mock=no_lookup)
    no_lookup.free()
    with pytest.raises(h2b.H2BError, match="a Rational index is >= the witness length"):
        mp.run(cells, b["selectors"], rational_index=[N], rational_den=mont([3], R))
    _same(_run(mp, b, cells), want)
    mp.free()


# ------------------------------------------------------------------------------------------------ against ProverSession.check
def _keygen_circuit(k, A, L, sel, bits, b, lay):
    """the fixed columns and sigma keygen would build from the oracle's layout: q_j, q_lookup, the table, the constants column
    c (distinct constants in assign_raw order) and sigma with one cycle per class of the union of every equality the keygen
    pass imposes (advice and constant equalities, break copies, lookup-advice copies)"""
    n = 1 << k
    one = mont([1], R)[0]
    fixed = {}
    for j in range(A):
        q = np.zeros((n, 4), dtype=np.uint64)
        q[sorted(lay["q"][j])] = one
        fixed["q%d" % j] = q
    if lay["q_lookup"] is not None:
        ql = np.zeros((n, 4), dtype=np.uint64)
        ql[sorted(lay["q_lookup"])] = one
        fixed["q_lookup"] = ql
    if L or sel:
        t = np.zeros((n, 4), dtype=np.uint64)
        t[: 1 << bits] = mont(list(range(1 << bits)), R)
        fixed["table"] = t
    crow = bo.assign_constants(zip(b["constants"], b["constant_index"]), n - 7, k)
    c = np.zeros((n, 4), dtype=np.uint64)
    for val, r in crow.items():
        c[r] = mont([val], R)[0]
    fixed["c"] = c
    bps = lay["break_points"]
    parent = {}

    def find(x):
        while parent.setdefault(x, x) != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    def union(x, y):
        parent[find(x)] = find(y)
    cell = lambda p: (1 + bo.raw_cell(bps, int(p))[0], bo.raw_cell(bps, int(p))[1])  # permutation column order [c, a0.., l0..]
    for x, y in b["advice_equalities"]:
        union(cell(x), cell(y))
    for val, p in zip(b["constants"], b["constant_index"]):
        union((0, crow[int(val) % R]), cell(p))
    for j, bp in enumerate(bps):
        union((1 + j, bp), (2 + j, 0))
    for i, p in enumerate(b["lookups"] if L else ()):
        union((1 + A + i % L, i // L), cell(p))
    w = pyref.omega_for(k)
    ident = lambda cc, r: pow(pyref.DELTA, cc, R) * pow(w, r, R) % R
    sigma = [[ident(cc, r) for r in range(n)] for cc in range(1 + A + L)]
    cycles = {}
    for x in list(parent):
        cycles.setdefault(find(x), []).append(x)
    for cyc in cycles.values():
        for i, (cc, r) in enumerate(cyc):
            sigma[cc][r] = ident(*cyc[(i + 1) % len(cyc)])
    return fixed, [mont(s, R) for s in sigma]


@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_mock_prover_agrees_with_the_session_check(ctx, h2b, A, L, sel):
    k, bits = 12, 8
    n, max_rows = 1 << k, (1 << k) - 9
    rng = np.random.default_rng(77 + A + L)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
    lay = bo.run(k, A, L, sel, bits, max_rows, b, b["values"])
    fixed, sigma = _keygen_circuit(k, A, L, sel, bits, b, lay)
    cs = h2b.Circuit(ctx, k, fixed, sigma, A=A, L=L, selector_lookup=sel)
    params = h2b.ParamsKZG(ctx, k, g=np.zeros((n, 8), dtype=np.uint64), g_lagrange=np.zeros((n, 8), dtype=np.uint64))
    sess = h2b.ProverSession(ctx, params, cs)
    mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows)
    for v in (b["values"], bo.plant(rng, b, bits)):
        cells = _mont_small(ctx, v)
        lk = cells[b["lookups"].astype(np.int64)] if L else np.zeros((0, 4), dtype=np.uint64)
        chk = sess.check(cells.ctypes.data, len(cells), break_points=lay["break_points"], lookup_ptr=lk.ctypes.data if len(lk) else 0,
                         n_lookup=len(lk))
        got = _run(mp, b, cells)
        assert chk["gates"] == got["gates"] and chk["lookups"] == got["lookups"]
        assert chk["satisfied"] == got["satisfied"]
        assert (sum(c for c, _ in chk["copies"]) > 0) == (got["equalities"][0] + got["constants"][0] > 0)
    mp.free(); sess.free(); cs.free(); params.close()


# ------------------------------------------------------------------------------------------------ C++ front end
def _serialize(r):
    out = [len(r["break_points"])] + r["break_points"]
    for count, rows in r["gates"] + r["lookups"] + [r["equalities"], r["constants"]]:
        out += [count, len(rows)] + rows
    for (c0, r0), (c1, r1) in r["equality_cells"]:
        out += [c0, r0, c1, r1]
    for c0, r0 in r["constant_cells"]:
        out += [c0, r0]
    return np.array(out, dtype=np.uint64).tobytes()


def test_cpp_mock_prover_matches_python(ctx, h2b, tmp_path):
    k, A, L, sel, bits, max_report = 10, 3, 1, False, 6, 8
    max_rows = (1 << k) - 9
    rng = np.random.default_rng(12)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
    v = bo.plant(rng, b, bits, many=12)
    cells, form = _forms(ctx, rng, v)
    d = str(tmp_path)
    consts = _mont_small(ctx, b["constants"])
    files = {"cells": cells, "witness": form[0], "rational_index": form[1], "rational_den": form[2], "selectors": b["selectors"],
             "eq": b["advice_equalities"], "consts": consts, "const_index": b["constant_index"], "lookups": b["lookups"]}
    for name, arr in files.items():
        np.ascontiguousarray(arr).tofile(os.path.join(d, name + ".bin"))
    with open(os.path.join(d, "manifest.txt"), "w") as f:
        f.write(" ".join(str(x) for x in (k, A, L, int(sel), bits, max_rows, len(cells), len(form[1]), len(b["advice_equalities"]),
                                          len(consts), len(b["lookups"]), max_report)))
    exe = os.path.join(ROOT, "build", "mock_prover_test")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    libdir = os.path.join(ROOT, "halo2-lib_b200")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "cpp", "mock_prover_test.cpp"), "-o", exe,
                           f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])
    out = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    mp = h2b.MockProver(ctx, k, A, L, sel, bits, max_rows)
    want = _serialize(_run(mp, b, cells, None, max_report)) + _serialize(_run(mp, b, cells, form, max_report)) * 2
    assert open(os.path.join(d, "report.bin"), "rb").read() == want
    mp.free()

"""GPU tests of the constraint check (ProverSession.check, h2b_check_*_dev, h2b_permutation_decode_dev): its reports must
equal tests/mock_oracle.py exactly — failure counts and rows — on satisfied instances and with planted violations, in both
witness forms, at the small sizes and at the full sizes; a check changes nothing a proof computes."""
import ctypes as C
import numpy as np
import pytest
from oracle import pyref
from util import *
import mock_oracle as mo
from test_gpu_assigned_witness import _setup, halo2_base_form, _prove_eval, _same_proof

pytestmark = pytest.mark.gpu
R = pyref.R
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


def _arr(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _check(sess, inst, V=None, lookup=None, max_report=16):
    V = _arr(inst["virtual"] if V is None else V)
    lk = _arr(inst["lookup"] if lookup is None else lookup)
    return sess.check(V.ctypes.data, len(V), break_points=inst["break_points"], lookup_ptr=lk.ctypes.data if len(lk) else 0,
                      n_lookup=len(lk), max_report=max_report)


def _oracle(k, A, L, sel, inst, fixed, V, lookup, max_report=16):
    fx = {nm: unmont(col, R) for nm, col in fixed.items()}
    cols = mo.assign(k, A, L, unmont(V, R), [int(b) for b in inst["break_points"]], unmont(lookup, R) if len(lookup) else [])
    return mo.verify(k, A, L, sel, fx, [unmont(s, R) for s in inst["sigma"]], cols, max_report)


def _layout(k, A):
    """(virtual index of (gate column j, row r)) under synthetic_circuit's layout"""
    usable = (1 << k) - 20
    G = usable // 4 if A == 1 else (usable - 4) // 4
    return (lambda j, r: r) if A == 1 else (lambda j, r: j * 4 * G + r), G


def _plant(k, A, L, inst, rng):
    """violations at row 0, at the 2048-row tile boundary (k >= 12) and in the last permutation column; returns (V, lookup)"""
    V, lk = _arr(inst["virtual"]).copy(), _arr(inst["lookup"]).copy()
    ix, G = _layout(k, A)
    one = mont([1], R)[0]
    add1 = lambda a, i: a.__setitem__(i, mont([unmont(a[i:i + 1], R)[0] + 1], R)[0])
    add1(V, ix(0, 3))                        # row 0: a gate output cell
    if k >= 12:
        add1(V, ix(A - 1, 2047))             # the last row of the first tile: gate 511's output
        add1(V, ix(A - 1, 2048))             # the first row of the second tile: gate 512's a operand
        b = next(i for i in range(600, 700) if unmont(V[ix(0, 4 * i + 1):ix(0, 4 * i + 1) + 1], R)[0])
        V[ix(0, 4 * b + 2)] = one if not V[ix(0, 4 * b + 2)].any() else 0  # a bit cell past the boundary: gate + copies
    if L:                                    # the last permutation column: a lookup-advice cell (a copy and maybe the lookup)
        t = L - 1
        lk[5 * L + t] = mont([1 << 40], R)[0]
    else:                                    # the last permutation column is the last gate column: one of its bit cells
        i = next(i for i in range(3, 40) if unmont(V[ix(A - 1, 4 * i + 1):ix(A - 1, 4 * i + 1) + 1], R)[0])
        r = ix(A - 1, 4 * i + 2)
        V[r] = one if not V[r].any() else 0
    return V, lk


@pytest.mark.parametrize("k", [8, 12])
@pytest.mark.parametrize("A,L,sel", SHAPES)
def test_check_matches_the_mock_prover(ctx, h2b, k, A, L, sel):
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 7100 + k + 10 * A + L, A, L, sel)
    got = _check(sess, inst)
    want = _oracle(k, A, L, sel, inst, inst["fixed"], _arr(inst["virtual"]), _arr(inst["lookup"]))
    assert want["satisfied"] and got == want
    V, lk = _plant(k, A, L, inst, rng)
    got = _check(sess, inst, V, lk)
    want = _oracle(k, A, L, sel, inst, inst["fixed"], V, lk)
    assert not want["satisfied"] and got == want
    assert got["gates"][0][0] >= 1 and got["copies"][-1][0] >= 1
    if k >= 12:
        assert 2044 in got["gates"][A - 1][1] and 2048 in got["gates"][A - 1][1]
    sess.free(); cs.free(); params.close()


@pytest.mark.parametrize("A,L,sel", [(1, 0, True), (2, 1, True)])
def test_rows_past_the_usable_ones_read_as_zero(ctx, h2b, A, L, sel):
    """a gate at row u - 1 reads rows >= u: they count as 0, whether they hold a previous proof's blinding rows or witness
    cells the walk placed there"""
    k = 8
    rng, params, cs0, sess0, inst, bases = _setup(ctx, h2b, k, 7300 + A, A, L, sel)
    sess0.free(); cs0.free()
    n, u = 1 << k, (1 << k) - 7
    fixed = {nm: _arr(c).copy() for nm, c in inst["fixed"].items()}
    fixed["q%d" % (A - 1)][u - 1] = mont([1], R)[0]
    cs = h2b.Circuit(ctx, k, fixed, inst["sigma"], A=A, L=L, selector_lookup=sel)
    sess = h2b.ProverSession(ctx, params, cs)
    ix, G = _layout(k, A)
    rnd = mont(rand_ints(rng, n, R), R)
    _prove_eval(sess, inst, rnd)  # leaves blinding scalars in rows >= u of every advice column
    V = _arr(inst["virtual"])
    last = ix(A - 1, 0)
    for cell_u1 in (0, 5):
        W = np.zeros((last + n, 4), dtype=np.uint64)
        W[:len(V)] = V
        W[last + u:] = mont(list(range(11, 11 + n - u)), R)  # junk placed at rows >= u of the last gate column
        W[last + u - 1] = mont([cell_u1], R)[0]
        got = _check(sess, inst, W)
        want = _oracle(k, A, L, sel, inst, fixed, W, _arr(inst["lookup"]))
        assert got == want
        assert got["gates"][A - 1] == ((1, [u - 1]) if cell_u1 else (0, []))
    sess.free(); cs.free(); params.close()


@pytest.mark.parametrize("k,A,L,sel", [(9, 1, 0, True), (9, 2, 1, True), (10, 3, 2, False)])
def test_both_witness_forms_give_identical_reports(ctx, h2b, k, A, L, sel):
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 7500 + k + A, A, L, sel)
    form = halo2_base_form(inst, k, rng)
    values, idx, den, lk_idx = (np.ascontiguousarray(a) for a in form)

    def check_form(vals, lki=lk_idx):
        return sess.check(vals.ctypes.data, len(vals), break_points=inst["break_points"], rational_index_ptr=idx.ctypes.data,
                          rational_den_ptr=den.ctypes.data, n_rational=len(idx), lookup_index_ptr=lki.ctypes.data if len(lki) else 0,
                          n_lookup=len(lki))
    assert check_form(values) == _check(sess, inst)
    # the same violation in both forms: a Rational cell (gate output) and a plain cell (a bit cell) changed
    V = _arr(inst["virtual"]).copy()
    vals = values.copy()
    j = int(idx[np.nonzero(idx % 4 == 3)[0][0]])
    pos = int(np.nonzero(idx == j)[0][0])
    new = unmont(V[j:j + 1], R)[0] + 3
    V[j] = mont([new], R)[0]
    vals[j] = mont([new * unmont(den[pos:pos + 1], R)[0]], R)[0] if den[pos].any() else mont([new], R)[0]
    b = next(i for i in range(2, 4 * 50, 4) if i not in set(int(x) for x in idx))
    V[b] = vals[b] = mont([7], R)[0]
    got = check_form(vals)
    assert not got["satisfied"] and got == _check(sess, inst, V)
    # a bad index: H2BError, and the session still checks
    bad = idx.copy(); bad[-1] = len(values)
    with pytest.raises(h2b.H2BError):
        sess.check(values.ctypes.data, len(values), break_points=inst["break_points"], rational_index_ptr=bad.ctypes.data,
                   rational_den_ptr=den.ctypes.data, n_rational=len(bad), lookup_index_ptr=lk_idx.ctypes.data if len(lk_idx) else 0,
                   n_lookup=len(lk_idx))
    assert check_form(values)["satisfied"]
    sess.free(); cs.free(); params.close()


def test_more_failures_than_max_report(ctx, h2b):
    k, A, L, sel = 12, 1, 0, True
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 7700, A, L, sel)
    V = _arr(inst["virtual"]).copy()
    rows = sorted(rng.choice(np.arange(3, 4 * 1000, 4), size=300, replace=False).tolist())
    for r in rows:
        V[r] = mont([unmont(V[r:r + 1], R)[0] + 1], R)[0]
    a = _check(sess, inst, V, max_report=7)
    b = _check(sess, inst, V, max_report=7)
    assert a["gates"] == [(300, [r - 3 for r in rows[:7]])] and a == b
    assert a == _oracle(k, A, L, sel, inst, inst["fixed"], V, _arr(inst["lookup"]), max_report=7)
    # the raw report bytes of two runs are identical
    raw = []
    for _ in range(2):
        _check(sess, inst, V, max_report=7)
        raw.append(sess.check_report.download().tobytes())
    assert raw[0] == raw[1]
    sess.free(); cs.free(); params.close()


def _decode(ctx, h2b, k, sigma, max_report=4):
    import torch
    npc, n = len(sigma), 1 << k
    d_sig = [torch.from_numpy(_arr(s).view(np.int64)).cuda() for s in sigma]
    d_map = torch.full((npc * n,), -1, dtype=torch.int32, device="cuda")
    d_rep = torch.full((npc * (max_report + 1),), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ptrs = (C.c_void_p * npc)(*[t.data_ptr() for t in d_sig])
    ctx.check(h2b.lib.h2b_permutation_decode_dev(ctx.h, ptrs, npc, k, C.c_void_p(d_map.data_ptr()), max_report, C.c_void_p(d_rep.data_ptr())))
    ctx.synchronize()
    return d_map.cpu().numpy().view(np.uint32).reshape(npc, n), d_rep.cpu().numpy().view(np.uint64).reshape(npc, max_report + 1)


def test_sigma_decode(ctx, h2b):
    k, A, L = 9, 2, 1
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 7900, A, L, True)
    n, npc = 1 << k, 1 + A + L
    w = pyref.omega_for(k)
    ident = [mont([pow(pyref.DELTA, c, R) * pow(w, r, R) % R for r in range(n)], R) for c in range(npc)]
    m, rep = _decode(ctx, h2b, k, ident)
    assert np.array_equal(m, (np.arange(npc, dtype=np.uint32)[:, None] << k) | np.arange(n, dtype=np.uint32)[None, :])
    assert not rep.any()
    m, rep = _decode(ctx, h2b, k, inst["sigma"])
    targets, bad = mo.decode_sigma(k, [unmont(s, R) for s in inst["sigma"]])
    assert not bad and not rep.any()
    want = np.zeros((npc, n), dtype=np.uint32)
    for (c, r), (c2, r2) in targets.items():
        want[c, r] = (c2 << k) | r2
    assert np.array_equal(m, want)
    # random field elements in the last column: reported as malformed, each row in place
    sig = [_arr(s).copy() for s in inst["sigma"]]
    bad_rows = [3, 200, 201]
    sig[-1][bad_rows] = mont(rand_ints(rng, 3, R), R)
    m, rep = _decode(ctx, h2b, k, sig)
    assert rep[-1, 0] == 3 and rep[-1, 1:4].tolist() == bad_rows and not rep[:-1].any()
    assert all(m[-1, r] == ((npc - 1) << k) | r for r in bad_rows)
    # a circuit with such a sigma raises on its first check, naming the first malformed cell
    cs2 = h2b.Circuit(ctx, k, inst["fixed"], sig, A=A, L=L, selector_lookup=True)
    sess2 = h2b.ProverSession(ctx, params, cs2)
    with pytest.raises(h2b.H2BError) as e:
        _check(sess2, inst)
    assert "column %d" % (npc - 1) in str(e.value) and "row 3" in str(e.value)
    sess2.free(); cs2.free(); sess.free(); cs.free(); params.close()


@pytest.mark.parametrize("A,L,sel", [(1, 0, True), (3, 2, True)])
def test_check_leaves_proofs_unchanged(ctx, h2b, A, L, sel):
    k = 9
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 8100 + A, A, L, sel)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    V, lk = _plant(k, A, L, inst, rng)
    first = _check(sess, inst, V, lk)
    after_check = _prove_eval(sess, inst, rnd)
    sess2 = h2b.ProverSession(ctx, params, cs)
    _same_proof(after_check, _prove_eval(sess2, inst, rnd))
    assert _check(sess, inst, V, lk) == first  # a proof in between changes nothing either
    sess2.free(); sess.free(); cs.free(); params.close()


def test_argument_errors_leave_the_session_usable(ctx, h2b):
    import torch
    k, A, L, sel = 8, 1, 0, True
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 8300, A, L, sel)
    lib, vp, n = h2b.lib, C.c_void_p, 1 << k
    buf = torch.zeros((4 * n * 4,), dtype=torch.int64, device="cuda")
    p = buf.data_ptr()
    col = vp(cs.lagr["table"].ptr)
    g = h2b.GraphEvaluator()  # the vertical gate q (a0 + a1 a2 - a3) on fixed slot 0 / advice slot 0
    a = lambda r: ("advice", 0, r)
    res = g.add_expression(("product", ("fixed", 0, 0), ("sum", ("sum", a(0), ("product", a(1), a(2))), ("negated", a(3)))))
    smap = cs.sigma_map
    bg = h2b.BoundGraph(g, res, fixed=[cs.lagr["q0"].ptr], advice=[sess.lagr["a0"].ptr])
    bad_bg = h2b.BoundGraph(g, res, fixed=[cs.lagr["q0"].ptr], advice=[sess.lagr["a0"].ptr])
    bad_bg.struct.n_calculations = 65
    two = (C.c_void_p * 2)(cs.lagr["c"].ptr, sess.lagr["a0"].ptr)
    nul = (C.c_void_p * 2)(cs.lagr["c"].ptr, None)
    calls = [
        lambda: lib.h2b_check_graph_dev(ctx.h, None, k, n, 4, vp(p)),
        lambda: lib.h2b_check_graph_dev(ctx.h, C.byref(bg.struct), k, n, 4, None),
        lambda: lib.h2b_check_graph_dev(ctx.h, C.byref(bg.struct), k, n + 1, 4, vp(p)),
        lambda: lib.h2b_check_graph_dev(ctx.h, C.byref(bg.struct), k, n, 0, vp(p)),
        lambda: lib.h2b_check_graph_dev(ctx.h, C.byref(bg.struct), k, n, h2b.CHECK_MAX_REPORT + 1, vp(p)),
        lambda: lib.h2b_check_graph_dev(ctx.h, C.byref(bg.struct), 29, n, 4, vp(p)),
        lambda: lib.h2b_check_graph_dev(ctx.h, C.byref(bad_bg.struct), k, n, 4, vp(p)),
        lambda: lib.h2b_check_lookup_dev(ctx.h, None, col, k, n, 4, vp(p)),
        lambda: lib.h2b_check_lookup_dev(ctx.h, col, col, k, n + 1, 4, vp(p)),
        lambda: lib.h2b_check_lookup_dev(ctx.h, col, col, 0, 1, 4, vp(p)),
        lambda: lib.h2b_permutation_decode_dev(ctx.h, two, 0, k, vp(p), 4, vp(p)),
        lambda: lib.h2b_permutation_decode_dev(ctx.h, nul, 2, k, vp(p), 4, vp(p)),
        lambda: lib.h2b_permutation_decode_dev(ctx.h, two, 2, 32, vp(p), 4, vp(p)),
        lambda: lib.h2b_permutation_decode_dev(ctx.h, two, 2, k, None, 4, vp(p)),
        lambda: lib.h2b_check_copies_dev(ctx.h, two, vp(smap.ptr), 2, k, 0, vp(p)),
        lambda: lib.h2b_check_copies_dev(ctx.h, two, None, 2, k, 4, vp(p)),
        lambda: lib.h2b_check_copies_dev(ctx.h, two, vp(smap.ptr), 0, k, 4, vp(p)),
        lambda: lib.h2b_check_copies_dev(ctx.h, two, vp(smap.ptr), 1 << 10, 24, 4, vp(p)),
    ]
    for i, f in enumerate(calls):
        assert f() == h2b.H2B_ERR_ARG, i
        assert lib.h2b_last_error(ctx.h)
    with pytest.raises(ValueError):
        _check(sess, inst, max_report=0)
    assert _check(sess, inst)["satisfied"]
    sess.free(); cs.free(); params.close()


class _Limbs:
    """a column of Montgomery limbs read as canonical integers on access (the full-size oracle reads few rows)"""

    def __init__(self, arr):
        self.a = arr

    def __getitem__(self, r):
        return unmont(self.a[r:r + 1], R)[0]


@pytest.mark.parametrize("k,A,L,sel", [(19, 1, 0, True), (20, 11, 2, True)])
def test_full_size_against_the_mock_prover(ctx, h2b, k, A, L, sel):
    """k = 19 (the ECDSA shape) and k = 20 (11 gate, 2 lookup-advice columns): satisfied, then a handful of planted violations.
    A Python walk over every cell is too slow here, so mock_oracle checks only the cells the planted violations can reach
    (the gate rows that read a changed cell, its lookup row, the cell and the cell whose sigma names it), with the sigma dict
    holding those cells; the device must report exactly those failures over the whole circuit."""
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 8500 + A, A, L, sel)
    n, u, npc = 1 << k, (1 << k) - 7, 1 + A + L
    assert _check(sess, inst)["satisfied"]
    V, lk = _arr(inst["virtual"]).copy(), _arr(inst["lookup"]).copy()
    cols = [c.copy() for c in inst["cols"]]
    ix, G = _layout(k, A)
    changed = []  # (permutation column, row)

    def put(j, r, v):
        """gate column j, row r (a cell of the virtual column) := v"""
        V[ix(j, r)] = cols[j][r] = mont([v], R)[0]
        changed.append((1 + j, r))
    val = lambda j, r: unmont(cols[j][r:r + 1], R)[0]
    put(0, 3, val(0, 3) + 1)                                  # row 0: a gate output
    put(A - 1, 4 * (G - 1) + 3, val(A - 1, 4 * (G - 1) + 3) + 5)  # the last gate
    put(A - 1, 2048, val(A - 1, 2048) + 1)                    # a tile boundary
    if L == 0:                                                # a looked-up cell outside the table, its gate kept
        i = 1000
        put(0, 4 * i + 1, 1 << 40)
        put(0, 4 * i + 3, (val(0, 4 * i) + (1 << 40) * val(0, 4 * i + 2)) % R)
    else:                                                     # lookup-advice cells: one outside the table, one copy broken
        for i, v in ((7, 1 << 40), (2 * 1000 + 1, 3)):
            t, r = i % L, i // L
            lk[i] = cols[A + t][r] = mont([v], R)[0]
            changed.append((1 + A + t, r))
    got = _check(sess, inst, V, lk, max_report=64)
    # the cells the changes reach
    w = pyref.omega_for(k)
    only = {"gates": {}, "lookups": {}, "copies": {}}
    targets = set()
    for c, r in changed:
        if c <= A:
            only["gates"].setdefault(c - 1, set()).update(x for x in range(r - 3, r + 1) if 0 <= x < u)
            if L == 0 and c == 1:
                only["lookups"].setdefault(0, set()).add(r)
        else:
            only["lookups"].setdefault(c - 1 - A, set()).add(r)
        ident = mont([pow(pyref.DELTA, c, R) * pow(w, r, R) % R], R)[0]
        hits = [(c2, int(r2)) for c2 in range(npc) for r2 in np.nonzero((_arr(inst["sigma"][c2]) == ident).all(axis=1))[0]]
        assert len(hits) == 1
        for cc, rr in [(c, r), hits[0]]:
            only["copies"].setdefault(cc, set()).add(rr)
            targets.add((cc, rr))
    only["targets"] = targets
    fixed = {nm: _Limbs(_arr(a)) for nm, a in inst["fixed"].items()}
    fixed["table"] = unmont(_arr(inst["fixed"]["table"])[: 1 << 8], R) + [0] * (n - (1 << 8))
    want = mo.verify(k, A, L, sel, fixed, [_Limbs(_arr(s)) for s in inst["sigma"]], [_Limbs(c) for c in cols], 64, only=only)
    assert not want["satisfied"] and got == want
    sess.free(); cs.free(); params.close()


def test_cpp_check_matches_python(ctx, h2b, tmp_path):
    """tests/cpp/prover_check_test.cpp runs ProverSession::check of include/h2b200_prover.hpp on a (9, 3, 2) instance with planted
    violations, in both witness forms: the same reports as halo2-lib_b200/prover.py"""
    import os
    import subprocess
    import test_cpp_mirror as tcm
    k, A, L, sel = 9, 3, 2, True
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 8700, A, L, sel)
    V, lk = _plant(k, A, L, inst, rng)
    form = halo2_base_form(dict(inst, virtual=V), k, rng)  # the looked-up cells by index: the original lookup cells
    values, idx, den, lk_idx = (np.ascontiguousarray(a) for a in form)
    max_report = 5
    want_eval = _check(sess, inst, V, lk, max_report)
    want_form = _check(sess, inst, V, None, max_report)
    assert not want_eval["satisfied"] and not want_form["satisfied"] and want_eval != want_form
    d = str(tmp_path)
    w = lambda name, arr: np.ascontiguousarray(arr, dtype=np.uint64).tofile(os.path.join(d, name))
    for nm in cs.fixed_names:
        w("fixed_%s.bin" % nm, inst["fixed"][nm])
    for i, sg in enumerate(inst["sigma"]):
        w("sigma_%d.bin" % i, sg)
    w("eval.bin", V); w("lookup.bin", lk); w("witness.bin", values); w("breaks.bin", inst["break_points"])
    w("rational_index.bin", idx); w("rational_den.bin", den); w("lookup_index.bin", lk_idx)
    with open(os.path.join(d, "manifest.txt"), "w") as f:
        f.write("%d %d %d %d %d %d %d %d %d %d %d\n" % (k, A, L, 1 if sel else 0, len(V), len(lk), len(values), len(inst["break_points"]),
                                                        len(idx), len(lk_idx), max_report))
    exe = os.path.join(d, "prover_check_test")
    libdir = os.path.join(tcm.ROOT, "halo2-lib_b200")
    subprocess.check_call([tcm.CXX, "-std=c++17", "-O1", "-Wall", os.path.join(tcm.ROOT, "tests", "cpp", "prover_check_test.cpp"), "-o", exe,
                           f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])
    out = subprocess.run([exe, d], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    raw = np.fromfile(os.path.join(d, "report.bin"), dtype=np.uint64).tolist()
    items = A + L + 1 + A + L
    pos = 0
    for want in (want_eval, want_form, want_form):  # evaluated form, halo2-base form, halo2-base form after a rejected index
        got = []
        for _ in range(items):
            cnt, nr = raw[pos], raw[pos + 1]
            got.append((cnt, raw[pos + 2: pos + 2 + nr]))
            pos += 2 + nr
        assert {"gates": got[:A], "lookups": got[A:A + L], "copies": got[A + L:], "satisfied": False} == want
    assert pos == len(raw)
    sess.free(); cs.free(); params.close()

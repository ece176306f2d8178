"""GPU tests of the resident prover fed with halo2-base's own witness form: the virtual column with n in place of every
Rational(n, d) cell, the (index, d) pairs of those cells, and the looked-up cells as virtual-column indices
(h2b_apply_rational_dev, h2b_assign_lookups_indexed_dev, ProverSession.prove's rational_* / lookup_index_ptr arguments).
The evaluated-witness proof of the same instance is the yardstick: both forms must give the same bytes."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from oracle import pyref, oracle as orc
from util import *
import prover_check as pc
import assigned_oracle as ao

pytestmark = pytest.mark.gpu
R = pyref.R


@pytest.fixture(scope="module")
def h2b():
    import halo2_lib_b200 as h
    return h


@pytest.fixture(scope="module")
def ctx(h2b):
    c = h2b.Context(0)
    yield c
    c.close()


def _setup(ctx, h2b, k, seed, A=1, L=0, sel=True):
    rng = np.random.default_rng(seed)
    n = 1 << k
    g = affine_to_limbs([pyref.G1])[0]
    bases_m = ctx.g1_fixed_base_mul(g, mont([3 + 5 * i for i in range(n)], R))
    bases_l = ctx.g1_fixed_base_mul(g, mont([7 + 11 * i for i in range(n)], R))
    params = h2b.ParamsKZG(ctx, k, g=bases_m, g_lagrange=bases_l)
    inst = h2b.synthetic_circuit(ctx, k, rng, A=A, L=L, selector_lookup=sel)
    cs = h2b.Circuit(ctx, k, inst["fixed"], inst["sigma"], A=A, L=L, selector_lookup=sel)
    sess = h2b.ProverSession(ctx, params, cs)
    return rng, params, cs, sess, inst, (bases_m, bases_l)


def _rand_mont(rng, m):
    """m random Montgomery elements below r (top limb < 2^61)"""
    a = rng.integers(0, 1 << 63, size=(m, 4), dtype=np.int64).astype(np.uint64)
    a[:, 3] &= np.uint64((1 << 61) - 1)
    return a


def halo2_base_form(inst, k, rng, frac=0.10, n_zero_den=8):
    """the instance as one walk over ctx.advice yields it: about `frac` of the cells Rational(v d, d) with random d, some
    zero-valued bit cells Rational(n, 0), and the looked-up cells replaced by their virtual-column indices"""
    V = np.ascontiguousarray(inst["virtual"])
    N, A = len(V), inst["A"]
    G = (N // (4 * A)) if A > 1 else ((1 << k) - 20) // 4     # gates per column (synthetic_circuit's layout)
    col_len = 4 * G if A > 1 else N                           # cells of one gate column in the virtual column
    idx = np.sort(rng.choice(N, size=max(1, int(frac * N)), replace=False)).astype(np.uint64)
    den = _rand_mont(rng, len(idx))
    values = V.copy()
    values[idx] = orc.f_mul(orc.FR, V[idx], den)
    # bit cells (row 4i + 2) holding 0 that are not Rational yet: Rational(n, 0) -> 0
    is_rat = np.zeros(N, dtype=bool); is_rat[idx] = True
    bit_rows = np.array([j * col_len + 4 * i + 2 for j in range(A) for i in range(G)])
    zeros = bit_rows[(~V[bit_rows].any(axis=1)) & (~is_rat[bit_rows])][:n_zero_den]
    if len(zeros):
        values[zeros] = _rand_mont(rng, len(zeros))
        idx = np.concatenate([idx, zeros.astype(np.uint64)])
        den = np.concatenate([den, np.zeros((len(zeros), 4), dtype=np.uint64)])
        order = np.argsort(idx, kind="stable")
        idx, den = np.ascontiguousarray(idx[order]), np.ascontiguousarray(den[order])
    # lookup cell i is the copy of cell (j, 4 i' + 1), in synthetic_circuit's order
    n_lk = len(inst["lookup"])
    per_col = n_lk // A if A else 0
    lk_idx = np.array([j * col_len + 4 * i + 1 for j in range(A) for i in range(per_col)], dtype=np.uint64)
    assert len(lk_idx) == n_lk
    if n_lk:
        assert np.array_equal(V[lk_idx], inst["lookup"])
    return values, idx, den, lk_idx


def _prove_eval(sess, inst, rnd, seed=5):
    v = np.ascontiguousarray(inst["virtual"])
    lk = np.ascontiguousarray(inst["lookup"])
    return sess.prove(v.ctypes.data, len(v), rnd.ctypes.data, seed=seed, break_points=inst["break_points"],
                      lookup_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))


def _prove_form(sess, inst, rnd, form, seed=5):
    values, idx, den, lk_idx = (np.ascontiguousarray(a) for a in form)
    return sess.prove(values.ctypes.data, len(values), rnd.ctypes.data, seed=seed, break_points=inst["break_points"],
                      rational_index_ptr=idx.ctypes.data if len(idx) else 0, rational_den_ptr=den.ctypes.data if len(idx) else 0,
                      n_rational=len(idx), lookup_index_ptr=lk_idx.ctypes.data if len(lk_idx) else 0, n_lookup=len(lk_idx))


def _same_proof(a, b):
    assert a["challenges"] == b["challenges"]
    assert [np.asarray(c).tobytes() for c in a["commitments"]] == [np.asarray(c).tobytes() for c in b["commitments"]]
    assert list(a["evals"]) == list(b["evals"])
    assert [np.asarray(v).tobytes() for v in a["evals"].values()] == [np.asarray(v).tobytes() for v in b["evals"].values()]


@pytest.mark.parametrize("k,A,L,sel", [(8, 1, 0, True), (8, 1, 0, False), (9, 2, 1, True), (10, 3, 2, True), (9, 8, 2, True)])
def test_same_proof_from_both_witness_forms(ctx, h2b, k, A, L, sel):
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 5100 + k + 10 * A, A, L, sel)
    n = 1 << k
    rnd = mont(rand_ints(rng, n, R), R)
    form = halo2_base_form(inst, k, rng)
    N, nR, nL = len(form[0]), len(form[1]), len(form[3])
    assert (~form[2].any(axis=1)).sum() > 0  # some d = 0 cells
    want = _prove_eval(sess, inst, rnd)
    got = _prove_form(sess, inst, rnd, form)
    _same_proof(got, want)
    left, right = pc.quotient_identity(got, k, cs.bf, A, L, sel)
    assert left == right
    # PCIe: the witness, 40 B per Rational cell, 8 B per looked-up cell, the random polynomial and the blinding rows
    blind_bytes = want["h2d_bytes"] - 32 * (N + len(inst["lookup"]) + n)
    assert got["h2d_bytes"] == 32 * N + 40 * nR + 8 * nL + 32 * n + blind_bytes
    # the same session again, the buffers reused: still the same proof
    _same_proof(_prove_form(sess, inst, rnd, form), want)
    sess.free(); cs.free(); params.close()


@pytest.mark.parametrize("k,A,L,sel", [(5, 1, 0, True), (6, 3, 2, True)])
def test_resident_prover_from_assigned_witness_matches_the_oracle_prover(ctx, h2b, k, A, L, sel):
    """oracle/prover_ref.py proves the same bytes from the same halo2-base form, turned into its evaluated inputs with plain
    integers (Rational cells n / d, d = 0 -> 0; looked-up cells gathered by index)"""
    from oracle import prover_ref
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 5700 + k + 10 * A, A, L, sel)
    n = 1 << k
    rnd = mont(rand_ints(rng, n, R), R)
    form = halo2_base_form(inst, k, rng, frac=0.2, n_zero_den=3)
    values, idx, den, lk_idx = form
    sess.blind_log = []
    res = _prove_form(sess, inst, rnd, form)
    it = iter([unmont(b, R) for b in sess.blind_log])
    sess.blind_log = None
    aff = lambda B: [None if (x == 0 and y == 0) else (x, y) for x, y in zip(unmont(B[:, :4], pyref.P), unmont(B[:, 4:], pyref.P))]
    virtual, lookup_cells = ao.evaluated_inputs(unmont(values, R), list(zip([int(i) for i in idx], unmont(den, R))), [int(i) for i in lk_idx])
    want = prover_ref.create_proof(k, A, L, sel, {nm: unmont(inst["fixed"][nm], R) for nm in cs.fixed_names},
                                   [unmont(sg, R) for sg in inst["sigma"]], virtual, [int(b) for b in inst["break_points"]],
                                   lookup_cells, unmont(rnd, R), lambda rows: next(it), aff(bases[0]), aff(bases[1]))
    assert next(it, None) is None
    assert res["challenges"] == want["challenges"]
    assert [np.asarray(c, dtype=np.uint64).tobytes() for c in res["commitments"]] == want["commitments"]
    assert [np.asarray(v, dtype=np.uint64).tobytes() for v in res["evals"].values()] == [prover_ref.fr_bytes(v) for _, _, v in want["evals"]]
    sess.free(); cs.free(); params.close()


def test_broken_inputs_fail_and_the_session_recovers(ctx, h2b):
    k, A, L, sel = 9, 2, 1, True
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 5900, A, L, sel)
    n = 1 << k
    rnd = mont(rand_ints(rng, n, R), R)
    form = halo2_base_form(inst, k, rng)
    values, idx, den, lk_idx = form
    want = _prove_eval(sess, inst, rnd)
    N = len(values)
    # a Rational cell whose value breaks a gate: the quotient identity fails
    j = int(idx[np.nonzero(idx % 4 == 3)[0][0]])  # an a3 cell (the gate's output)
    pos = int(np.nonzero(idx == j)[0][0])
    v_bad = values.copy()
    v_bad[j] = orc.f_mul(orc.FR, orc.f_add(orc.FR, inst["virtual"][j:j + 1], mont([1], R)), den[pos:pos + 1])[0]
    res = _prove_form(sess, inst, rnd, (v_bad, idx, den, lk_idx))
    l2, r2 = pc.quotient_identity(res, k, cs.bf, A, L, sel)
    assert l2 != r2
    _same_proof(_prove_form(sess, inst, rnd, form), want)
    # a lookup index at a cell whose value is not in the table (an a0 cell: 62-bit values): ConstraintSystemFailure
    lk_bad = lk_idx.copy(); lk_bad[3] = 0
    with pytest.raises(h2b.H2BError) as e:
        _prove_form(sess, inst, rnd, (values, idx, den, lk_bad))
    assert e.value.code == -5 and "ConstraintSystemFailure" in str(e.value)
    _same_proof(_prove_form(sess, inst, rnd, form), want)
    # indices out of range, and Rational indices that do not strictly increase: H2BError, no proof
    bads = []
    i_oor = idx.copy(); i_oor[-1] = N; bads.append((values, i_oor, den, lk_idx))
    i_rep = idx.copy(); i_rep[5] = i_rep[4]; bads.append((values, i_rep, den, lk_idx))
    i_dec = idx.copy(); i_dec[5], i_dec[6] = idx[6], idx[5]; bads.append((values, i_dec, den, lk_idx))
    l_oor = lk_idx.copy(); l_oor[-1] = N + 1000; bads.append((values, idx, den, l_oor))
    for bad in bads:
        with pytest.raises(h2b.H2BError):
            _prove_form(sess, inst, rnd, bad)
        _same_proof(_prove_form(sess, inst, rnd, form), want)
    with pytest.raises(ValueError):  # values and indices for the looked-up cells at once
        v = np.ascontiguousarray(values)
        sess.prove(v.ctypes.data, N, rnd.ctypes.data, break_points=inst["break_points"], lookup_ptr=inst["lookup"].ctypes.data,
                   lookup_index_ptr=lk_idx.ctypes.data, n_lookup=len(lk_idx))
    sess.free(); cs.free(); params.close()


def test_lookup_gather_against_the_c_restatement(ctx, h2b):
    """h2b_assign_lookups_indexed_dev alone: repeated cells, the last cell, n_lookup not divisible by L, the rows past the
    assigned ones zero, the layout rule, and the verdict word"""
    import torch
    k, L, N = 7, 3, 500
    rng = np.random.default_rng(11)
    vals = _rand_mont(rng, N)
    lk = rng.integers(0, N, size=3 * 100 + 2).astype(np.uint64)
    lk[:4] = 17; lk[-1] = N - 1
    rc, _, want = ao.assigned_witness(vals, np.zeros(0, dtype=np.uint64), np.zeros((0, 4), dtype=np.uint64), lk, k, L)
    assert rc == 0
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()
    d_vals, d_lk = dev(vals), dev(lk)
    d_cols = torch.full((L << k, 4), -1, dtype=torch.int64, device="cuda")
    d_st = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    h2b.assign_lookups_indexed_dev(ctx, d_vals.data_ptr(), N, d_lk.data_ptr(), len(lk), k, L, d_cols.data_ptr(), d_st.data_ptr())
    ctx.synchronize()
    assert np.array_equal(d_cols.cpu().numpy().view(np.uint64).reshape(L, 1 << k, 4), want)
    assert int(d_st.cpu().numpy().view(np.uint32)[0]) == 0
    lk[7] = N
    d_lk = dev(lk); torch.cuda.synchronize()
    h2b.assign_lookups_indexed_dev(ctx, d_vals.data_ptr(), N, d_lk.data_ptr(), len(lk), k, L, d_cols.data_ptr(), d_st.data_ptr())
    ctx.synchronize()
    assert int(d_st.cpu().numpy().view(np.uint32)[0]) == 1
    with pytest.raises(h2b.LayoutError):  # ceil(n_lookup / L) > 2^k
        h2b.assign_lookups_indexed_dev(ctx, d_vals.data_ptr(), N, d_lk.data_ptr(), L * (1 << k) + 1, k, L, d_cols.data_ptr(), d_st.data_ptr())


@pytest.mark.parametrize("R_", [(1 << 19) + 1, (1 << 21) + 3])
def test_apply_rational_at_sizes_with_many_elements_per_thread(ctx, h2b, R_):
    """the batch inversion's second code path (E >= 3 elements per thread), with the denominators of one CTA's whole range
    zero, against the C restatement (tests/cpp/assigned_witness_oracle.c)"""
    import torch
    import test_gpu_large_sizes as tls
    rng = np.random.default_rng(R_)
    N = R_ + R_ // 3
    E = tls._elements_per_thread(R_, torch.cuda.get_device_properties(0).multi_processor_count)
    assert E >= 3
    vals = _rand_mont(rng, N)
    idx = np.sort(rng.choice(N, size=R_, replace=False)).astype(np.uint64)
    den = _rand_mont(rng, R_)
    den[256 * E: 2 * 256 * E] = 0          # CTA 1's whole range
    den[-1] = 0
    rc, want, _ = ao.assigned_witness(vals, idx, den, np.zeros(0, dtype=np.uint64), 0, 0)
    assert rc == 0
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()
    d_vals, d_idx, d_den = dev(vals), dev(idx), dev(den)
    d_st = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    h2b.apply_rational_dev(ctx, d_vals.data_ptr(), N, d_idx.data_ptr(), d_den.data_ptr(), R_, d_st.data_ptr())
    ctx.synchronize()
    assert int(d_st.cpu().numpy().view(np.uint32)[0]) == 0
    assert np.array_equal(d_vals.cpu().numpy().view(np.uint64).reshape(N, 4), want)
    # a repeated index is reported (bit 1), an index == N too (bit 0)
    idx[10] = idx[9]; idx[-1] = N
    d_idx = dev(idx); torch.cuda.synchronize()
    h2b.apply_rational_dev(ctx, d_vals.data_ptr(), N, d_idx.data_ptr(), d_den.data_ptr(), R_, d_st.data_ptr())
    ctx.synchronize()
    assert int(d_st.cpu().numpy().view(np.uint32)[0]) == 3


def test_resident_proof_k20_from_assigned_witness(ctx, h2b):
    """k = 20, 11 gate columns and 2 lookup columns, about 1 % Rational cells: the same bytes as the evaluated witness"""
    k, A, L = 20, 11, 2
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 6100, A, L, True)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    form = halo2_base_form(inst, k, rng, frac=0.01)
    want = _prove_eval(sess, inst, rnd)
    got = _prove_form(sess, inst, rnd, form)
    _same_proof(got, want)
    sess.free(); cs.free(); params.close()


def test_cpp_prover_from_assigned_witness_matches_python(ctx, h2b, tmp_path):
    """tests/cpp/prover_assigned_test.cpp proves a (9, 7, 2) instance from the halo2-base form through
    include/h2b200_prover.hpp: the same bytes as halo2-lib_b200/prover.py, and the same bytes up"""
    k, A, L, sel = 9, 7, 2, True
    rng, params, cs, sess, inst, bases = _setup(ctx, h2b, k, 6300, A, L, sel)
    n = 1 << k
    rnd = mont(rand_ints(rng, n, R), R)
    form = halo2_base_form(inst, k, rng)
    values, idx, den, lk_idx = form
    sess.blind_log = []
    res = _prove_form(sess, inst, rnd, form)
    blind = np.concatenate(sess.blind_log)
    sess.blind_log = None
    d = str(tmp_path)
    w = lambda name, arr: np.ascontiguousarray(arr, dtype=np.uint64).tofile(os.path.join(d, name))
    for nm in cs.fixed_names:
        w("fixed_%s.bin" % nm, inst["fixed"][nm])
    for i, sg in enumerate(inst["sigma"]):
        w("sigma_%d.bin" % i, sg)
    w("witness.bin", values); w("breaks.bin", inst["break_points"]); w("rational_index.bin", idx); w("rational_den.bin", den)
    w("lookup_index.bin", lk_idx); w("random.bin", rnd); w("blind.bin", blind); w("bases_m.bin", bases[0]); w("bases_l.bin", bases[1])
    with open(os.path.join(d, "manifest.txt"), "w") as f:
        f.write("%d %d %d %d %d %d %d %d %d\n" % (k, A, L, 1 if sel else 0, len(values), len(inst["break_points"]), len(idx), len(lk_idx), len(blind)))
    import test_cpp_mirror as tcm
    exe = os.path.join(str(tmp_path), "prover_assigned_test")
    libdir = os.path.join(tcm.ROOT, "halo2-lib_b200")
    subprocess.check_call([tcm.CXX, "-std=c++17", "-O1", "-Wall", os.path.join(tcm.ROOT, "tests", "cpp", "prover_assigned_test.cpp"), "-o", exe,
                           f"-L{libdir}", "-lh2b200", f"-Wl,-rpath,{libdir}"])
    out = subprocess.run([exe, d], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    raw = np.fromfile(os.path.join(d, "proof.bin"), dtype=np.uint64)
    nc = int(raw[0])
    cms = raw[1:1 + 12 * nc].reshape(nc, 12)
    ne = int(raw[1 + 12 * nc])
    evs = raw[2 + 12 * nc: 2 + 12 * nc + 4 * ne].reshape(ne, 4)
    chal = raw[2 + 12 * nc + 4 * ne:].reshape(5, 4)
    assert nc == len(res["commitments"]) and np.array_equal(cms, np.stack(res["commitments"]))
    assert ne == len(res["evals"]) and np.array_equal(evs, np.stack(list(res["evals"].values())))
    assert [pc.fr(c) for c in chal] == [res["challenges"][c] for c in ("theta", "beta", "gamma", "y", "x")]
    assert "h2d_bytes %d" % res["h2d_bytes"] in out.stdout
    sess.free(); cs.free(); params.close()

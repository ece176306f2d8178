"""GPU tests of halo2's selector compression (Circuit / keygen with compress_selectors, DESIGN.md §4.13): the conflict kernel
against a numpy restatement in both its forms, gen_proof's bytes against tests/selectors_oracle.py at k = 8 for every shape kind,
the committed golden proof, oracle-verified proofs on a keygen'd circuit at k = 12, the ECDSA shape's columns as the legacy ones
renamed, `check` on compressed and legacy circuits, and a legacy session's bytes beside a compressed one."""
import ctypes as C
import numpy as np
import pytest
from oracle import pyref
from util import mont, unmont, rand_ints
import halo2_proof_oracle as hp
import params_oracle as po
import selectors_oracle as so
import test_gpu_constants as tgc
import test_gpu_halo2_proof as tgh
import test_oracle_halo2_proof as toh

pytestmark = pytest.mark.gpu
R = pyref.R
TAU = po.seeded_tau()
VK_REPR = 0x5E1EC7
ONE = mont([1], R)[0]
params_for, point = tgh.params_for, tgh.point
h2b, ctx, _close_params = tgh.h2b, tgh.ctx, tgh._close_params


def _want_conflicts(bits):
    b = bits.astype(np.int64)
    return ((b @ b.T) > 0).astype(np.uint8)


@pytest.mark.parametrize("k,S", [(10, 12), (11, 292), (20, 12), (23, 12)])
def test_conflict_kernel(ctx, h2b, k, S):
    import torch
    from halo2_lib_b200._capi import lib
    n = 1 << k
    rng = np.random.default_rng(k + S)
    bits = np.zeros((S, n), dtype=bool)
    for i in range(S):  # staggered blocks, some pairs disjoint, one all-zero column, sparse random extra rows
        if i == 3:
            continue
        start = (i * n) // S
        bits[i, start:start + max(1, n // (2 * S))] = True
        if i % 2:
            bits[i, rng.integers(0, n, size=3)] = True
    want = _want_conflicts(bits)
    got = np.zeros((S, S), dtype=np.uint8)
    one = torch.from_numpy(ONE.view(np.int64).copy()).cuda()
    cols = []
    for i in range(S):
        c = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
        c[torch.from_numpy(bits[i]).cuda()] = one
        cols.append(c)
    ptrs = (C.c_void_p * S)(*[c.data_ptr() for c in cols])
    torch.cuda.synchronize()
    ctx.check(lib.h2b_selector_conflicts_dev(ctx.h, ptrs, S, k, got.ctypes.data))
    assert np.array_equal(got, want)
    if n * S <= 1 << 20:  # the host-pointer form through the staging path
        host = [c.cpu().numpy().view(np.uint64) for c in cols]
        hp_ = (C.c_void_p * S)(*[h.ctypes.data for h in host])
        got2 = np.zeros((S, S), dtype=np.uint8)
        ctx.check(lib.h2b_selector_conflicts(ctx.h, hp_, S, k, got2.ctypes.data))
        assert np.array_equal(got2, want)
    del cols


def test_conflict_kernel_rejects_values_other_than_0_and_1(ctx, h2b):
    from halo2_lib_b200._capi import lib
    k, S = 10, 3
    cols = [np.zeros((1 << k, 4), dtype=np.uint64) for _ in range(S)]
    cols[0][5] = ONE
    cols[2][77] = mont([2], R)[0]
    ptrs = (C.c_void_p * S)(*[c.ctypes.data for c in cols])
    out = np.zeros((S, S), dtype=np.uint8)
    with pytest.raises(h2b.H2BError, match="selector column 2 holds a value other than 0 or 1 at row 77"):
        ctx.check(lib.h2b_selector_conflicts(ctx.h, ptrs, S, k, out.ctypes.data))
    cols[2][77] = ONE  # the context stays usable
    ctx.check(lib.h2b_selector_conflicts(ctx.h, ptrs, S, k, out.ctypes.data))


def _circuit(ctx, h2b, k, inst, A, L, sel, F, I, compress):
    return h2b.Circuit(ctx, k, {nm: mont(v, R) for nm, v in inst["fixed"].items()}, [mont(sg, R) for sg in inst["sigma"]], A=A, L=L,
                       selector_lookup=sel, I=I, F=F, compress_selectors=compress)


def _gen_proof(ctx, h2b, k, cs, inst, rnd, blind):
    sess = h2b.ProverSession(ctx, params_for(ctx, h2b, k), cs)
    sess.blind_source = blind
    v, lk, rp = mont(inst["virtual"], R), mont(inst["lookup"], R), mont(rnd, R)
    proof = sess.gen_proof(v.ctypes.data, len(v), rp.ctypes.data, VK_REPR, instances=[mont(p, R) for p in inst["public"]],
                           break_points=np.array(inst["break_points"], dtype=np.uint64), lookup_ptr=lk.ctypes.data if len(lk) else 0,
                           n_lookup=len(lk))
    sess.free()
    return proof


@pytest.mark.parametrize("A,L,sel", toh.SHAPE_KINDS)
def test_gen_proof_is_the_oracles_bytes(ctx, h2b, A, L, sel):
    import random
    k, F, I = 6, 2, 1
    seed = 300 + 10 * A + L + 3 * F + I + k
    inst = toh.instance(k, A, L, sel, 3, F, I, seed)
    _, lay = so.compress(k, A, L, sel, F, inst["fixed"])
    cs = _circuit(ctx, h2b, k, inst, A, L, sel, F, I, True)
    assert cs.fixed_names == lay["columns"] and cs.fixed_queries == lay["queries"]
    assert cs.selectors == {nm: tuple(v) for nm, v in lay["selectors"].items()}
    r1 = random.Random(seed)
    rnd = [r1.randrange(R) for _ in range(1 << k)]
    got = _gen_proof(ctx, h2b, k, cs, inst, rnd, lambda rows: mont([r1.randrange(R) for _ in range(rows)], R))
    r2 = random.Random(seed)
    g, gl = toh.params(k)
    want = so.create_proof(k, A, L, sel, F, inst["fixed"], inst["sigma"], inst["virtual"], inst["break_points"], inst["lookup"],
                           [r2.randrange(R) for _ in range(1 << k)], lambda rows: [r2.randrange(R) for _ in range(rows)], g, gl,
                           inst["public"], VK_REPR)
    assert got == want
    cs.free()


def test_gen_proof_reproduces_the_committed_golden_proof(ctx, h2b):
    import json, os
    from golden import make_golden_compressed_proof as g
    want = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "halo2_proof_compressed_k5.json")))
    inst, rnd, rr = g.inputs()
    cs = _circuit(ctx, h2b, g.K, inst, g.A, g.L, g.SEL, g.F, g.I, True)
    assert cs.fixed_names == want["fixed_columns"] and cs.fixed_queries == want["fixed_queries"]
    sess = h2b.ProverSession(ctx, params_for(ctx, h2b, g.K), cs)
    sess.blind_source = lambda rows: mont([rr.randrange(R) for _ in range(rows)], R)
    v, lk, rp = mont(inst["virtual"], R), mont(inst["lookup"], R), mont(rnd, R)
    proof = sess.gen_proof(v.ctypes.data, len(v), rp.ctypes.data, g.VK_REPR, instances=[mont(p, R) for p in inst["public"]],
                           break_points=np.array(inst["break_points"], dtype=np.uint64), lookup_ptr=lk.ctypes.data, n_lookup=len(lk))
    assert proof == bytes.fromhex(want["proof"])
    sess.free(); cs.free()


def _keygen(ctx, h2b, k, A, L, sel, bits, F, I, seed, compress, fill=0.6):
    rng = np.random.default_rng(seed)
    max_rows = (1 << k) - 9
    b = tgc._builder(rng, k, A, L, sel, bits, max_rows, F, fill=fill, extra=False)
    inst = tgc._instances(rng, b, I, 5)
    cs, vk, bps = h2b.keygen(ctx, params_for(ctx, h2b, k), k, A, L, sel, bits, max_rows, b["selectors"], b["advice_equalities"],
                             tgc._consts(ctx, b), b["lookups"], F=F, I=I, instances=inst if I else None, compress_selectors=compress)
    public = tgc._public(ctx, b, inst) if I else None
    return dict(b=b, cs=cs, vk=vk, bps=bps, public=public)


def _session_inputs(ctx, r, L):
    cells = tgc._mont_small(ctx, r["b"]["values"])
    lk = np.ascontiguousarray(r["b"]["lookups"] if L else np.zeros(0, dtype=np.uint64))
    kw = dict(break_points=np.array(r["bps"], dtype=np.uint64), lookup_index_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))
    return cells, lk, kw


@pytest.mark.parametrize("k,A,L,sel,F,bits", [(12, 3, 2, False, 2, 8)])
def test_oracle_verifies_keygen_proofs(ctx, h2b, k, A, L, sel, F, bits):
    I = 1
    r = _keygen(ctx, h2b, k, A, L, sel, bits, F, I, 90 + k, True)
    cs = r["cs"]
    lay = {"columns": cs.fixed_names, "queries": cs.fixed_queries, "selectors": cs.selectors}
    cells, lk, kw = _session_inputs(ctx, r, L)
    rng = np.random.default_rng(k)
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    sess = h2b.ProverSession(ctx, params_for(ctx, h2b, k), cs)
    proof = sess.gen_proof(cells.ctypes.data, len(cells), rnd.ctypes.data, VK_REPR, instances=r["public"], seed=1, **kw)
    vkp = {"fixed": {nm: point(c) for nm, c in r["vk"]["fixed"].items()}, "permutation": [point(c) for c in r["vk"]["permutation"]]}
    assert list(vkp["fixed"]) == cs.fixed_names
    public = [unmont(p, R) for p in r["public"]]
    verify = lambda pf, lay_=lay: so.verify_proof(pf, k, A, L, sel, F, lay_, vkp, public, VK_REPR, pyref.G1, TAU)
    assert verify(proof)
    s = so.shape(k, A, L, sel, F, I, lay)
    first_eval = 32 * (len(s["adv"]) + 2 * s["n_lookups"] + s["n_sets"] + s["n_lookups"] + 1 + s["degree"] - 1)
    h1 = first_eval + 32 * len(hp.evaluation_order(s))
    assert len(proof) == h1 + 64
    fixed_eval = first_eval + 32 * hp.evaluation_order(s).index(("s0", 0))
    for what, at in {"advice commitment": 3, "evaluation": first_eval + 5, "combination column evaluation": fixed_eval + 1,
                     "h_x commitment": h1 + 1, "W'": h1 + 33}.items():
        bad = bytearray(proof)
        bad[at] ^= 1
        assert not verify(bytes(bad)), what
    assert not verify(proof, dict(lay, queries=list(cs.fixed_names)))
    sess.free(); cs.free()


def test_ecdsa_shape_is_the_legacy_columns_renamed(ctx, h2b):
    """the selector lookup shape (1 / 0, degree 5): s0 = q_lookup, s1 = q0 with the same values and commitments"""
    k, A, L, sel, F, bits = 19, 1, 0, True, 1, 18
    new = _keygen(ctx, h2b, k, A, L, sel, bits, F, 0, 7, True)
    old = _keygen(ctx, h2b, k, A, L, sel, bits, F, 0, 7, False)
    cn, co_ = new["cs"], old["cs"]
    assert cn.fixed_names == ["table", "c", "s0", "s1"] and cn.fixed_queries == ["c", "table", "s0", "s1"]
    assert cn.selectors == {"q_lookup": ("s0", 1, 1), "q0": ("s1", 1, 1)}
    for a, b in (("s0", "q_lookup"), ("s1", "q0"), ("table", "table"), ("c", "c")):
        assert np.array_equal(cn.lagr[a].download(), co_.lagr[b].download())
        assert np.array_equal(new["vk"]["fixed"][a], old["vk"]["fixed"][b])
    assert all(np.array_equal(x, y) for x, y in zip(new["vk"]["permutation"], old["vk"]["permutation"]))
    cn.free(); co_.free()


def test_check_reports_equal_on_compressed_and_legacy(ctx, h2b):
    """a broken gate cell in a column whose selector shares a combination column: the same reports on both layouts"""
    k, A, L, sel, F, bits = 10, 4, 1, False, 1, 6
    reports = []
    for compress in (False, True):
        r = _keygen(ctx, h2b, k, A, L, sel, bits, F, 0, 33, compress, fill=0.4)
        cs = r["cs"]
        cells, lk, kw = _session_inputs(ctx, r, L)
        gate = np.flatnonzero(np.asarray(r["b"]["selectors"]))
        cells = cells.copy()
        for p in gate[[0, len(gate) // 2, len(gate) - 1]]:
            cells[p + 3] = mont([12345], R)[0]
        sess = h2b.ProverSession(ctx, params_for(ctx, h2b, k), cs)
        res = sess.check(cells.ctypes.data, len(cells), **kw)
        reports.append(res)
        sess.free(); cs.free()
    assert not reports[0]["satisfied"] and reports[0] == reports[1]


def test_legacy_session_unchanged_beside_a_compressed_one(ctx, h2b):
    k, A, L, sel, F, bits = 10, 2, 1, False, 1, 6
    out = []
    for compress in (False, True, False):
        r = _keygen(ctx, h2b, k, A, L, sel, bits, F, 0, 21, compress)
        cells, lk, kw = _session_inputs(ctx, r, L)
        rnd = mont(rand_ints(np.random.default_rng(2), 1 << k, R), R)
        sess = h2b.ProverSession(ctx, params_for(ctx, h2b, k), r["cs"])
        out.append(sess.prove(cells.ctypes.data, len(cells), rnd.ctypes.data, seed=3, **kw))
        sess.free(); r["cs"].free()
    a, b = out[0], out[2]
    assert all(np.array_equal(x, y) for x, y in zip(a["commitments"], b["commitments"])) and a["challenges"] == b["challenges"]
    assert all(np.array_equal(a["evals"][q], b["evals"][q]) for q in a["evals"])

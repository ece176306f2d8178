"""CPU: halo2's proof bytes on plain Python integers (tests/halo2_proof_oracle.py) — the personalized transcript against
hashlib and the committed SRS image, the shared phases against constants_oracle.create_proof, oracle proofs that the oracle's
verify_proof accepts for every shape kind, and rejections of changed bytes, a different vk_repr and a changed public value."""
import hashlib
import json
import os
import random
import numpy as np
import pytest
from oracle import pyref
import builder_oracle as bo
import constants_oracle as co
import halo2_proof_oracle as hp
import params_oracle as po
import test_oracle_constants as toc

R = pyref.R
HERE = os.path.dirname(os.path.abspath(__file__))
TAU = po.seeded_tau()
_params = {}


def params(k):
    if k not in _params:
        g, gl, _, _ = po.params_setup(k, TAU)
        _params[k] = (g, gl)
    return _params[k]


def test_transcript_is_personalized_blake2b():
    tr = hp.Blake2bWrite()
    pt = pyref.g1_mul(5, pyref.G1)
    tr.write_point(pt)
    tr.write_scalar(R - 1)
    tr.common_scalar(7)
    c = tr.squeeze()
    ref = hashlib.blake2b(digest_size=64, person=b"Halo2-Transcript")
    ref.update(b"\x01" + pt[0].to_bytes(32, "little") + pt[1].to_bytes(32, "little"))
    ref.update(b"\x02" + (R - 1).to_bytes(32, "little") + b"\x02" + (7).to_bytes(32, "little") + b"\x00")
    assert c == int.from_bytes(ref.digest(), "little") % R
    assert tr.finalize() == pyref.g1_compress(pt) + (R - 1).to_bytes(32, "little")
    plain = hashlib.blake2b(ref.digest(), digest_size=64).digest()  # an unpersonalized hash differs
    assert plain != ref.digest()
    with pytest.raises(ValueError):
        tr.write_point(None)


def test_point_encoding_is_the_processed_srs_image():
    """write_point's bytes for the bases of the committed gen_srs(4) image are that image's 32-byte encodings"""
    d = json.load(open(os.path.join(HERE, "golden", "srs_seeded_k4.json")))
    k = int(d["k"])
    assert int(d["tau"], 16) == TAU
    img = bytes.fromhex(d["processed"])
    g, gl = params(k)
    tr = hp.Blake2bWrite()
    for p in g + gl:
        tr.write_point(p)
    assert tr.finalize() == img[4:4 + 64 * (1 << k)]
    rd = hp.Blake2bRead(tr.finalize())
    assert [rd.read_point() for _ in range(2 << k)] == g + gl
    assert rd.squeeze() == tr.squeeze()


def instance(k, A, L, sel, bits, F, I, seed):
    """a satisfied keygen-form builder (test_oracle_constants._keygen_instance) with I instance columns of 5 cells each"""
    n, max_rows = 1 << k, (1 << k) - 9
    rng = np.random.default_rng(seed)
    b = bo.make_builder(rng, k, A, L, sel, bits, max_rows, fill=0.6)
    if F == 0:
        b = dict(b, constants=np.zeros(0, dtype=np.uint64), constant_index=np.zeros(0, dtype=np.uint64))
    inst = toc._keygen_instance(k, A, L, sel, bits, F, seed)
    idx = [rng.choice(len(b["selectors"]), size=5).astype(np.uint64) for _ in range(I)]
    pairs, _, _ = co.copy_sequence(k, A, L, max_rows, b, F, idx)
    inst["sigma"] = toc._sigma(k, F + A + L + I, pairs)
    inst["public"] = [[int(b["values"][int(p)]) % R for p in ix] for ix in idx]
    return inst


def prove(k, A, L, sel, F, inst, seed, vk_repr):
    rng = random.Random(seed)
    g, gl = params(k)
    blind = lambda rows: [rng.randrange(R) for _ in range(rows)]
    return hp.create_proof(k, A, L, sel, F, inst["fixed"], inst["sigma"], inst["virtual"], inst["break_points"], inst["lookup"],
                           [rng.randrange(R) for _ in range(1 << k)], blind, g, gl, inst["public"], vk_repr)


def vk_of(k, A, L, sel, F, inst):
    s = hp.shape(k, A, L, sel, F, len(inst["public"]))
    _, gl = params(k)
    return {"fixed": {nm: pyref.msm_naive(inst["fixed"][nm], gl) for nm in s["fixed"]},
            "permutation": [pyref.msm_naive(col, gl) for col in inst["sigma"]]}


def verify(proof, k, A, L, sel, F, inst, vk, vk_repr, public=None):
    g, _ = params(k)
    return hp.verify_proof(proof, k, A, L, sel, F, vk, inst["public"] if public is None else public, vk_repr, g[0], TAU)


def test_phases_are_the_oracle_provers():
    """through the library's own transcript the shared phases give constants_oracle.create_proof's commitments and challenges"""
    from oracle.prover_ref import Transcript, g1_bytes
    k, A, L, sel, F = 5, 2, 1, False, 2
    inst = instance(k, A, L, sel, 3, F, 1, 41)

    class Legacy(Transcript):
        def write_point(self, pt):
            self.absorb(g1_bytes(pt))

        def common_scalar(self, v):
            self.absorb(hp.fr_bytes(v))
    draws = lambda: random.Random(5)
    args = (inst["fixed"], inst["sigma"], inst["virtual"], inst["break_points"], inst["lookup"], [3 + i for i in range(1 << k)])
    bases = (params(k)[0], params(k)[1])
    r1, r2 = draws(), draws()
    ph = hp.phases(hp.shape(k, A, L, sel, F, 1), *args, lambda rows: [r1.randrange(R) for _ in range(rows)], *bases, inst["public"], Legacy())
    want = co.create_proof(k, A, L, sel, F, *args, lambda rows: [r2.randrange(R) for _ in range(rows)], *bases, instances=inst["public"])
    assert [g1_bytes(p) for p in ph["commitments"]] == want["commitments"][:len(ph["commitments"])]
    assert ph["challenges"] == want["challenges"]


SHAPE_KINDS = [(1, 0, True), (2, 1, False), (2, 0, False)]  # selector lookup, lookup advice, no lookup


@pytest.mark.parametrize("k,F,I", [(5, 1, 0), (5, 0, 1), (5, 2, 1), (6, 2, 1)])
@pytest.mark.parametrize("A,L,sel", SHAPE_KINDS)
def test_oracle_proofs_verify(A, L, sel, F, I, k):
    seed = 300 + 10 * A + L + 3 * F + I + k
    inst = instance(k, A, L, sel, 3, F, I, seed)
    proof = prove(k, A, L, sel, F, inst, seed, 12345)
    s = hp.shape(k, A, L, sel, F, I)
    n_points = len(s["adv"]) + 2 * s["n_lookups"] + s["n_sets"] + s["n_lookups"] + 1 + s["degree"] - 1 + 2
    assert len(proof) == 32 * (n_points + len(hp.evaluation_order(s)))
    assert verify(proof, k, A, L, sel, F, inst, vk_of(k, A, L, sel, F, inst), 12345)


def mutations(k, A, L, sel, F, I):
    """byte offsets of: the first advice commitment, the first evaluation, h_x's commitment, W'"""
    s = hp.shape(k, A, L, sel, F, I)
    n_pts = len(s["adv"]) + 2 * s["n_lookups"] + s["n_sets"] + s["n_lookups"] + 1 + s["degree"] - 1
    first_eval = 32 * n_pts
    h1 = first_eval + 32 * len(hp.evaluation_order(s))
    return {"advice commitment": 3, "evaluation": first_eval + 5, "h_x commitment": h1 + 1, "W'": h1 + 32 + 1}


def swapped_openings(proof: bytes) -> bytes:
    """h_x's commitment and W' exchanged: two valid points, so only SHPLONK's equation can reject"""
    return proof[:-64] + proof[-32:] + proof[-64:-32]


def test_rejections():
    k, A, L, sel, F, I = 5, 2, 1, False, 2, 1
    inst = instance(k, A, L, sel, 3, F, I, 77)
    vk = vk_of(k, A, L, sel, F, inst)
    proof = prove(k, A, L, sel, F, inst, 77, 99)
    assert verify(proof, k, A, L, sel, F, inst, vk, 99)
    for what, at in mutations(k, A, L, sel, F, I).items():
        bad = bytearray(proof)
        bad[at] ^= 1
        assert not verify(bytes(bad), k, A, L, sel, F, inst, vk, 99), what
    assert not verify(proof, k, A, L, sel, F, inst, vk, 100)
    public = [list(c) for c in inst["public"]]
    public[0][0] = (public[0][0] + 1) % R
    assert not verify(proof, k, A, L, sel, F, inst, vk, 99, public)
    assert not verify(proof + bytes(32), k, A, L, sel, F, inst, vk, 99)
    assert not verify(swapped_openings(proof), k, A, L, sel, F, inst, vk, 99)


def test_oracle_reproduces_the_committed_golden_proof():
    """tests/golden/halo2_proof_k5.json (tests/golden/make_golden_halo2_proof.py): the frozen bytes of the oracle, which its
    verifier accepts"""
    from golden import make_golden_halo2_proof as g
    want = json.load(open(os.path.join(HERE, "golden", "halo2_proof_k5.json")))
    assert g.proof() == want
    inst, _, _ = g.inputs()
    assert verify(bytes.fromhex(want["proof"]), g.K, g.A, g.L, g.SEL, g.F, inst, vk_of(g.K, g.A, g.L, g.SEL, g.F, inst), g.VK_REPR)

"""Generates tests/golden/halo2_proof_compressed_k5.json: ONE tiny proof in halo2's bytes with halo2's selector compression
(keygen_vk's layout) from the integer restatement tests/selectors_oracle.py (pure Python integers): 3 gate-advice + 1
lookup-advice column (degree 4), 1 constants column, 1 instance column, k = 5, params of gen_srs's tau.  The builder is
tests/test_oracle_halo2_proof.instance; its q0 and q1 are active on disjoint rows and share the column s0 with roots 1 and 2,
while q2 (active beside them) stays alone in s1: both roots of a pair reach h.
Run: python tests/golden/make_golden_compressed_proof.py"""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import selectors_oracle as so
import test_oracle_halo2_proof as t

K, A, L, SEL, F, I, BITS, SEED = 5, 3, 1, False, 1, 1, 3, 5151
VK_REPR = 0x0A1B2C3D4E5F60718293A4B5C6D7E8F90011223344556677


def inputs():
    """the instance, and the random polynomial and blinding stream of random.Random(SEED + 1)"""
    inst = t.instance(K, A, L, SEL, BITS, F, I, SEED)
    rr = random.Random(SEED + 1)
    rnd = [rr.randrange(t.R) for _ in range(1 << K)]
    return inst, rnd, rr


def proof() -> dict:
    inst, rnd, rr = inputs()
    g, gl = t.params(K)
    blind = lambda rows: [rr.randrange(t.R) for _ in range(rows)]
    pf = so.create_proof(K, A, L, SEL, F, inst["fixed"], inst["sigma"], inst["virtual"], inst["break_points"], inst["lookup"], rnd, blind,
                         g, gl, inst["public"], VK_REPR)
    _, lay = so.compress(K, A, L, SEL, F, inst["fixed"])
    return {"shape": {"k": K, "gate_advice": A, "lookup_advice": L, "selector_lookup": SEL, "constants": F, "instance": I,
                      "lookup_bits": BITS, "seed": SEED,
                      "note": "instance: tests/test_oracle_halo2_proof.instance; random polynomial "
                              "then blinding rows: random.Random(seed + 1); params: ParamsKZG::setup(k, ChaCha20Rng::from_seed([0; 32]))"},
            "combinations": lay["combinations"], "fixed_columns": lay["columns"], "fixed_queries": lay["queries"],
            "vk_repr": hex(VK_REPR), "proof": pf.hex()}


if __name__ == "__main__":
    json.dump(proof(), open(os.path.join(HERE, "halo2_proof_compressed_k5.json"), "w"), indent=1)
    print("wrote halo2_proof_compressed_k5.json")

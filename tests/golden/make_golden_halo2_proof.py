"""Generates tests/golden/halo2_proof_k5.json: ONE tiny proof in halo2's bytes (Blake2bWrite + ProverSHPLONK) from the integer
restatement tests/halo2_proof_oracle.py (pure Python integers), on the seeded keygen-form builder of
tests/test_oracle_halo2_proof.instance — 2 gate-advice + 1 lookup-advice column, 2 constants columns, 1 instance column, k = 5 —
with params of gen_srs's tau (ParamsKZG::setup with ChaCha20Rng::from_seed([0; 32])).  A restatement golden: it freezes today's
answer so that later rounds compare the oracle (tests/test_oracle_halo2_proof.py) and the resident CUDA prover
(tests/test_gpu_halo2_proof.py, both front ends) with a FIXED file.
Run: python tests/golden/make_golden_halo2_proof.py"""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import test_oracle_halo2_proof as t

K, A, L, SEL, F, I, BITS, SEED = 5, 2, 1, False, 2, 1, 3, 4343
VK_REPR = 0x0F1E2D3C4B5A69788796A5B4C3D2E1F00112233445566778899AABBCCDDEEFF


def inputs():
    """the instance, and the random polynomial and blinding stream of random.Random(SEED + 1): random polynomial first, then
    the blinding rows in the order the prover asks for them"""
    inst = t.instance(K, A, L, SEL, BITS, F, I, SEED)
    rr = random.Random(SEED + 1)
    rnd = [rr.randrange(t.R) for _ in range(1 << K)]
    return inst, rnd, rr


def proof() -> dict:
    inst, rnd, rr = inputs()
    g, gl = t.params(K)
    blind = lambda rows: [rr.randrange(t.R) for _ in range(rows)]
    pf = t.hp.create_proof(K, A, L, SEL, F, inst["fixed"], inst["sigma"], inst["virtual"], inst["break_points"], inst["lookup"], rnd, blind,
                           g, gl, inst["public"], VK_REPR)
    return {"shape": {"k": K, "gate_advice": A, "lookup_advice": L, "selector_lookup": SEL, "constants": F, "instance": I,
                      "lookup_bits": BITS, "seed": SEED,
                      "note": "instance: tests/test_oracle_halo2_proof.instance; random polynomial then blinding rows: "
                              "random.Random(seed + 1); params: ParamsKZG::setup(k, ChaCha20Rng::from_seed([0; 32]))"},
            "vk_repr": hex(VK_REPR), "proof": pf.hex()}


if __name__ == "__main__":
    json.dump(proof(), open(os.path.join(HERE, "halo2_proof_k5.json"), "w"), indent=1)
    print("wrote halo2_proof_k5.json")

"""Generates tests/golden/srs_seeded_k4.json with tests/params_oracle.py (Python integers only): the params `gen_srs(4)` creates —
tau of ParamsKZG::setup(4, ChaCha20Rng::from_seed([0; 32])) and the whole ParamsKZG::write image in SerdeFormat::Processed and
SerdeFormat::RawBytes.  Run: python tests/golden/make_golden_srs.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import params_oracle as p

PATH = os.path.join(HERE, "srs_seeded_k4.json")


def build(k: int = 4, seed: bytes = bytes(32)) -> dict:
    tau = p.seeded_tau(seed)
    g, gl, g2, s_g2 = p.params_setup(k, tau)
    return {
        "note": "gen_srs(k): ParamsKZG::setup(k, ChaCha20Rng::from_seed(seed)) written with ParamsKZG::write; tau canonical; images hex",
        "k": k, "seed": seed.hex(), "tau": hex(tau),
        "processed": p.params_image(k, g, gl, g2, s_g2, processed=True).hex(),
        "raw": p.params_image(k, g, gl, g2, s_g2, processed=False).hex(),
    }


if __name__ == "__main__":
    json.dump(build(), open(PATH, "w"), indent=1)
    print("wrote", PATH)

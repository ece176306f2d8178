"""Wall clock of halo2_lib_b200.keygen on synthetic halo2-base builders at the fp_mul bench shape (k = 16, 8 gate / 2 lookup
columns), ECDSA (k = 19, 1 gate column, selector lookup) and the MSM circuit (k = 20, 11 / 2), split into its phases (copies:
uploads, fixed columns, the copy list and its sorts; forest: spanning forest and walk; sigma: sigma values; pk: the proving key's
coefficient and extended forms; vk: the commitments), and beside it the sequential permutation Assembly of the C restatement
(tests/cpp/keygen_oracle.c) on one host core over the same copy list, labelled "port".  Every run must give the same sigma map.
Usage (on the GPU box): python tools/prof_keygen.py [--reps 10] [--warmup 2]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import halo2_lib_b200 as h
import builder_oracle as bo
import keygen_oracle as ko
from oracle import pyref
from util import mont, affine_to_limbs

SHAPES = [(16, 8, 2, False, 15), (19, 1, 0, True, 18), (20, 11, 2, False, 19)]
PHASES = ("copies", "forest", "sigma", "pk", "vk")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    card = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    power = q.stdout.strip() or "unknown"
    ctx = h.Context(0)
    for k, A, L, sel, bits in SHAPES:
        rng = np.random.default_rng(k)
        n, max_rows = 1 << k, (1 << k) - 9
        b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
        g = affine_to_limbs([pyref.G1])[0]
        bases = ctx.g1_fixed_base_mul(g, mont(list(range(3, 3 + n)), pyref.R))
        params = h.ParamsKZG(ctx, k, g=bases, g_lagrange=bases)
        zc = np.zeros(len(b["constants"]), dtype=np.uint64)
        consts = ctx.field_op(1, 5, np.stack([b["constants"], zc, zc, zc], axis=1))
        first = None
        total, phases = [], {p: [] for p in PHASES}
        for rep in range(args.warmup + args.reps):
            t = {}
            t0 = time.perf_counter()
            cs, vk, bps = h.keygen(ctx, params, k, A, L, sel, bits, max_rows, b["selectors"], b["advice_equalities"],
                                   (consts, b["constant_index"]), b["lookups"], timings=t)
            ms = 1e3 * (time.perf_counter() - t0)
            m = cs.sigma_map.download()
            first = m if first is None else first
            assert np.array_equal(m, first)
            cs.free()
            if rep >= args.warmup:
                total.append(ms)
                for p in PHASES:
                    phases[p].append(t[p])
        params.close()
        pairs = ko.copy_sequence(k, A, L, max_rows, b)[0]
        V = (1 + A + L) << k
        port = []
        for _ in range(3):
            t0 = time.perf_counter()
            ko.assembly_c(V, pairs)
            port.append(1e3 * (time.perf_counter() - t0))
        med = lambda v: round(float(np.median(v)), 3)
        print(json.dumps({"k": k, "A": A, "L": L, "selector_lookup": sel, "cells": len(b["selectors"]), "copies": len(pairs),
                          "keygen_ms_median": med(total), "keygen_ms_min": round(min(total), 3), "keygen_ms_max": round(max(total), 3),
                          **{p + "_ms_median": med(phases[p]) for p in PHASES}, "port_assembly_ms_median": med(port),
                          "reps": args.reps, "card": card, "power_limit": power}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

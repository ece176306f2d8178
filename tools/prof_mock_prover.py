"""Wall clock of MockProver.run on a halo2-base builder in its keygen form (no SRS, sigma or proving key) at the fp_mul bench shape
(k = 16, 8 gate / 2 lookup columns), ECDSA (k = 19, 1 gate column, selector lookup) and the MSM circuit (k = 20, 11 / 2), and
beside it what ProverSession.check needs first for the same shape: building the Circuit (every fixed and sigma column in its
three forms) and the ProverSession.  A run includes the uploads of the builder from pageable host memory and ends with its
reports on the host.  Every run must report the satisfied builder as satisfied.
Usage (on the GPU box): python tools/prof_mock_prover.py [--reps 10] [--warmup 2]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import halo2_lib_b200 as h
import builder_oracle as bo

SHAPES = [(16, 8, 2, False, 15), (19, 1, 0, True, 18), (20, 11, 2, False, 19)]


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
        z = np.zeros(len(b["values"]), dtype=np.uint64)
        cells = ctx.field_op(1, 5, np.stack([b["values"], z, z, z], axis=1))
        zc = np.zeros(len(b["constants"]), dtype=np.uint64)
        consts = ctx.field_op(1, 5, np.stack([b["constants"], zc, zc, zc], axis=1))
        mp = h.MockProver(ctx, k, A, L, sel, bits, max_rows)
        run = lambda: mp.run(cells, b["selectors"], b["advice_equalities"], (consts, b["constant_index"]), b["lookups"])
        for _ in range(args.warmup):
            assert run()["satisfied"]
        times = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            r = run()  # ends with the report download: the device is done
            times.append(1e3 * (time.perf_counter() - t0))
            assert r["satisfied"]
        mp.free()
        # what the existing check needs before its first call, for a circuit of the same shape (contents do not change the cost)
        inst = h.synthetic_circuit(ctx, k, rng, A=A, L=L, selector_lookup=sel)
        params = h.ParamsKZG(ctx, k, g=np.zeros((n, 8), dtype=np.uint64), g_lagrange=np.zeros((n, 8), dtype=np.uint64))
        build = []
        for _ in range(3):
            t0 = time.perf_counter()
            cs = h.Circuit(ctx, k, inst["fixed"], inst["sigma"], A=A, L=L, selector_lookup=sel)
            sess = h.ProverSession(ctx, params, cs)
            ctx.synchronize()
            build.append(1e3 * (time.perf_counter() - t0))
            sess.free(); cs.free()
        params.close()
        print(json.dumps({"k": k, "A": A, "L": L, "selector_lookup": sel, "lookup_bits": bits, "cells": len(cells),
                          "advice_equalities": len(b["advice_equalities"]), "constant_equalities": len(consts), "lookups": len(b["lookups"]),
                          "mock_run_ms_median": round(float(np.median(times)), 3), "mock_run_ms_min": round(min(times), 3),
                          "mock_run_ms_max": round(max(times), 3), "circuit_and_session_build_ms_median": round(float(np.median(build)), 3),
                          "reps": args.reps, "card": card, "power_limit": power}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

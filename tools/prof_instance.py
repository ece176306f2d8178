"""Resident proof time with and without public inputs: a keygen circuit of a synthetic halo2-base builder with I = 0 and with one
instance column of 16 public cells, proved by a ProverSession, at the fp_mul bench shape (k = 16, 8 gate / 2 lookup columns:
11 -> 12 permutation columns in chunks of 2) and ECDSA (k = 19, 1 gate column, selector lookup: 2 -> 3 in chunks of 3).  Both
circuits are timed alternately in one process; each time is one proof ended by its last download (the host synchronises).
Prints the median of --reps proofs after --warmup, the card and its power limit, one JSON line per shape.
Usage (on the GPU box): python tools/prof_instance.py [--reps 10] [--warmup 3]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import halo2_lib_b200 as h
import builder_oracle as bo
from oracle import pyref
from util import mont, affine_to_limbs

SHAPES = [(16, 8, 2, False, 15), (19, 1, 0, True, 18)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
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
        small = lambda v: ctx.field_op(1, 5, np.stack([np.ascontiguousarray(v, dtype=np.uint64)] + [np.zeros(len(v), dtype=np.uint64)] * 3, axis=1))
        consts = (small(b["constants"]), b["constant_index"])
        cells = small(b["values"])
        idx = rng.choice(len(b["values"]), size=16, replace=False).astype(np.uint64)
        public = [small(b["values"][idx.astype(np.int64)])]
        rnd = mont(list(range(1, n + 1)), pyref.R)
        lk = np.ascontiguousarray(b["lookups"] if L else np.zeros(0, dtype=np.uint64))
        runs = {}
        for I in (0, 1):
            kw = dict(I=1, instances=[idx]) if I else {}
            cs, _, bps = h.keygen(ctx, params, k, A, L, sel, bits, max_rows, b["selectors"], b["advice_equalities"], consts, b["lookups"], **kw)
            sess = h.ProverSession(ctx, params, cs)
            pk = dict(break_points=np.array(bps, dtype=np.uint64), lookup_index_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk),
                      instances=public if I else None)
            runs[I] = (cs, sess, pk, [])
        for rep in range(args.warmup + args.reps):
            for I, (cs, sess, pk, times) in runs.items():
                t0 = time.perf_counter()
                sess.prove(cells.ctypes.data, len(cells), rnd.ctypes.data, seed=rep, **pk)
                if rep >= args.warmup:
                    times.append((time.perf_counter() - t0) * 1e3)
        med = {I: float(np.median(r[3])) for I, r in runs.items()}
        print(json.dumps({"k": k, "A": A, "L": L, "selector_lookup": sel, "perm_cols": [len(runs[I][0].perm_cols) for I in (0, 1)],
                          "proof_ms_I0": round(med[0], 2), "proof_ms_I1_16_public": round(med[1], 2),
                          "overhead_ms": round(med[1] - med[0], 2), "reps": args.reps, "card": card, "power_limit": power}), flush=True)
        for cs, sess, _, _ in runs.values():
            sess.free(); cs.free()
        params.close()
    ctx.close()


if __name__ == "__main__":
    main()

"""Keygen and resident proof time with several constants columns: one synthetic halo2-base builder per shape, keygen'd and proved
with F = 1, 2 and 7 constants columns, at k = 17 (8 gate / 2 lookup columns, chunks of 2) and k = 19 (ECDSA: 1 gate column,
selector lookup, chunks of 3).  The three F are timed alternately in one process; a keygen time is one `keygen` call (it ends
synchronised), a proof time one proof ended by its last download.  Prints the median of --reps runs after --warmup, the card
and its power limit, one JSON line per shape.
Usage (on the GPU box): python tools/prof_constants.py [--reps 10] [--warmup 3]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import halo2_lib_b200 as h
import builder_oracle as bo
from oracle import pyref
from util import mont, affine_to_limbs

SHAPES = [(17, 8, 2, False, 16), (19, 1, 0, True, 18)]
FS = (1, 2, 7)


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
        rnd = mont(list(range(1, n + 1)), pyref.R)
        lk = np.ascontiguousarray(b["lookups"] if L else np.zeros(0, dtype=np.uint64))
        kg_args = (ctx, params, k, A, L, sel, bits, max_rows, b["selectors"], b["advice_equalities"], consts, b["lookups"])
        runs = {}
        for F in FS:
            cs, _, bps = h.keygen(*kg_args, F=F)
            sess = h.ProverSession(ctx, params, cs)
            pk = dict(break_points=np.array(bps, dtype=np.uint64), lookup_index_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))
            runs[F] = (cs, sess, pk, [], [])
        for rep in range(args.warmup + args.reps):
            for F, (cs, sess, pk, kg_times, proof_times) in runs.items():
                t0 = time.perf_counter()
                h.keygen(*kg_args, F=F)[0].free()
                t1 = time.perf_counter()
                sess.prove(cells.ctypes.data, len(cells), rnd.ctypes.data, seed=rep, **pk)
                t2 = time.perf_counter()
                if rep >= args.warmup:
                    kg_times.append((t1 - t0) * 1e3)
                    proof_times.append((t2 - t1) * 1e3)
        out = {"k": k, "A": A, "L": L, "selector_lookup": sel, "distinct_constants": len(set(b["constants"].tolist()))}
        for F, (cs, sess, _, kg_times, proof_times) in runs.items():
            out["F%d" % F] = {"perm_cols": len(cs.perm_cols), "n_sets": cs.n_sets, "keygen_ms": round(float(np.median(kg_times)), 2),
                              "proof_ms": round(float(np.median(proof_times)), 2)}
        out.update({"reps": args.reps, "card": card, "power_limit": power})
        print(json.dumps(out), flush=True)
        for cs, sess, _, _, _ in runs.values():
            sess.free(); cs.free()
        params.close()
    ctx.close()


if __name__ == "__main__":
    main()

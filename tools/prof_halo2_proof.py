"""Wall clock of halo2's proof bytes (`ProverSession.gen_proof`) beside the library's own proof (`prove`) on one session, and of
the multi-point division against sequential kate_division.  One synthetic halo2-base builder per shape, keygen'd once: fp_mul at
k = 16 (8 gate / 2 lookup columns) and ECDSA at k = 19 (1 gate column, selector lookup); `prove` and `gen_proof` alternate in one
process, each timed to its last download.  The division: h2b_kate_division_multi_dev against m chained h2b_kate_division_dev on
2^19 coefficients, m = 1..4, CUDA events.  Prints the median of --reps runs after --warmup, the card and its power limit, one
JSON line per shape.
Usage (on the GPU box): python tools/prof_halo2_proof.py [--reps 10] [--warmup 3]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import halo2_lib_b200 as h
from halo2_lib_b200._capi import lib
import builder_oracle as bo
from oracle import pyref
from util import mont

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
    small = lambda v: ctx.field_op(1, 5, np.stack([np.ascontiguousarray(v, dtype=np.uint64)] + [np.zeros(len(v), dtype=np.uint64)] * 3, axis=1))
    for k, A, L, sel, bits in SHAPES:
        rng = np.random.default_rng(k)
        n, max_rows = 1 << k, (1 << k) - 9
        b = bo.make_builder(rng, k, A, L, sel, bits, max_rows)
        params = h.ParamsKZG.setup_seeded(ctx, k)
        cs, _, bps = h.keygen(ctx, params, k, A, L, sel, bits, max_rows, b["selectors"], b["advice_equalities"],
                              (small(b["constants"]), b["constant_index"]), b["lookups"])
        sess = h.ProverSession(ctx, params, cs)
        cells = small(b["values"])
        rnd = mont(list(range(1, n + 1)), pyref.R)
        lk = np.ascontiguousarray(b["lookups"] if L else np.zeros(0, dtype=np.uint64))
        pk = dict(break_points=np.array(bps, dtype=np.uint64), lookup_index_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))
        t_prove, t_gen, size = [], [], 0
        for rep in range(args.warmup + args.reps):
            t0 = time.perf_counter()
            sess.prove(cells.ctypes.data, len(cells), rnd.ctypes.data, seed=rep, **pk)
            t1 = time.perf_counter()
            size = len(sess.gen_proof(cells.ctypes.data, len(cells), rnd.ctypes.data, 12345, seed=rep, **pk))
            t2 = time.perf_counter()
            if rep >= args.warmup:
                t_prove.append((t1 - t0) * 1e3)
                t_gen.append((t2 - t1) * 1e3)
        print(json.dumps({"k": k, "A": A, "L": L, "selector_lookup": sel, "prove_ms": round(float(np.median(t_prove)), 2),
                          "gen_proof_ms": round(float(np.median(t_gen)), 2), "proof_bytes": size, "card": card, "power_limit": power}))
        sess.free(); cs.free(); params.close()
    # the division at 2^19, on torch's stream so that the events bracket the library's launches
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    n = 1 << 19
    a = torch.randint(0, 1 << 60, (n, 4), dtype=torch.int64, device="cuda")
    q = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
    t = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
    vp = lambda x: C.c_void_p(x)
    out = {"n": n, "card": card, "power_limit": power}
    for m in (1, 2, 3, 4):
        zs = [pyref.R - 5 - j for j in range(m)]
        ws = []
        for j in range(m):
            d = 1
            for i in range(m):
                if i != j:
                    d = d * (zs[j] - zs[i]) % pyref.R
            ws.append(pow(d, -1, pyref.R))
        pts, wts = mont(zs, pyref.R), mont(ws, pyref.R)

        def multi():
            ctx.check(lib.h2b_kate_division_multi_dev(ctx.h, vp(a.data_ptr()), n, vp(pts.ctypes.data), m, vp(wts.ctypes.data), vp(q.data_ptr())))

        def chained():
            src, dst = a, q
            for j in range(m):
                ctx.check(lib.h2b_kate_division_dev(ctx.h, vp(src.data_ptr()), n, vp(pts[j].ctypes.data), vp(dst.data_ptr())))
                src, dst = dst, (t if dst is q else q)
        times = {"multi": [], "chained": []}
        for rep in range(args.warmup + args.reps):
            for name, fn in (("multi", multi), ("chained", chained)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); fn(); e1.record()
                torch.cuda.synchronize()
                if rep >= args.warmup:
                    times[name].append(e0.elapsed_time(e1))
        out["m%d" % m] = {k2: round(float(np.median(v)), 4) for k2, v in times.items()}
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

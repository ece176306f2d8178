"""Cost of halo2's selector compression (DESIGN.md §4.13): keygen and gen_proof on the compressed and the legacy layout of one
builder, alternated on one card, and the conflict kernel alone (CUDA events).  Prints the card name and power limit first.
Run: python tools/prof_selectors.py"""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import halo2_lib_b200 as h2b  # noqa: E402
from halo2_lib_b200._capi import lib  # noqa: E402
from oracle import pyref  # noqa: E402
from util import mont, rand_ints  # noqa: E402
import test_gpu_constants as tgc  # noqa: E402

R = pyref.R
REPS, WARM = 10, 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def shape_run(ctx, k, A, L, sel, bits, F, fill, seed):
    params = h2b.ParamsKZG.setup_seeded(ctx, k)
    rng = np.random.default_rng(seed)
    max_rows = (1 << k) - 9
    b = tgc._builder(rng, k, A, L, sel, bits, max_rows, F, fill=fill, extra=False)
    consts = tgc._consts(ctx, b)
    cells = tgc._mont_small(ctx, b["values"])
    lk = np.ascontiguousarray(b["lookups"] if L else np.zeros(0, dtype=np.uint64))
    rnd = mont(rand_ints(rng, 1 << k, R), R)
    kg, pf, info = {False: [], True: []}, {False: [], True: []}, {}
    for it in range(WARM + REPS):
        for compress in (False, True):
            t0 = time.perf_counter()
            cs, vk, bps = h2b.keygen(ctx, params, k, A, L, sel, bits, max_rows, b["selectors"], b["advice_equalities"], consts, b["lookups"],
                                     F=F, compress_selectors=compress)
            t1 = time.perf_counter()
            sess = h2b.ProverSession(ctx, params, cs)
            kw = dict(break_points=np.array(bps, dtype=np.uint64), lookup_index_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))
            t2 = time.perf_counter()
            sess.gen_proof(cells.ctypes.data, len(cells), rnd.ctypes.data, 1, seed=1, **kw)
            t3 = time.perf_counter()
            if it >= WARM:
                kg[compress].append(1e3 * (t1 - t0))
                pf[compress].append(1e3 * (t3 - t2))
            info[compress] = (len(cs.fixed_names), sorted({c for c, _, _ in cs.selectors.values()}),
                              max(ln for _, _, ln in cs.selectors.values()))
            sess.free()
            cs.free()
    params.close()
    med = lambda v: float(np.median(v))
    for compress in (False, True):
        nf, cols, mx = info[compress]
        print("k=%d A=%d L=%d sel=%d F=%d fill=%.2f %-10s keygen %.1f ms  gen_proof %.2f ms  fixed columns %d  longest combination %d"
              % (k, A, L, sel, F, fill, "compressed" if compress else "legacy", med(kg[compress]), med(pf[compress]), nf, mx))


def kernel(ctx, k, S):
    n = 1 << k
    one = torch.from_numpy(mont([1], R)[0].view(np.int64).copy()).cuda()
    cols = []
    for i in range(S):
        c = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
        c[(i * n) // S:(i * n) // S + n // (2 * S)] = one
        cols.append(c)
    ptrs = (C.c_void_p * S)(*[c.data_ptr() for c in cols])
    out = np.zeros((S, S), dtype=np.uint8)
    times = []
    for it in range(WARM + REPS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        ctx.check(lib.h2b_selector_conflicts_dev(ctx.h, ptrs, S, k, out.ctypes.data))
        e1.record()
        torch.cuda.synchronize()
        if it >= WARM:
            times.append(e0.elapsed_time(e1))
    print("conflict kernel k=%d S=%d: %.3f ms (call, CUDA events on the default stream around it)" % (k, S, float(np.median(times))))


def main():
    print("card:", card())
    ctx = h2b.Context(0)
    kernel(ctx, 20, 12)
    kernel(ctx, 11, 292)
    shape_run(ctx, 16, 8, 2, False, 8, 1, 0.6, 5)   # fp_mul shape
    shape_run(ctx, 16, 8, 2, False, 8, 1, 0.2, 5)   # fewer gates per column: more disjoint selectors
    shape_run(ctx, 19, 1, 0, True, 18, 1, 0.6, 7)   # ECDSA shape
    ctx.close()


if __name__ == "__main__":
    main()

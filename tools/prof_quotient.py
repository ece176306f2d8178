"""Device timings of the "next-row" kernels (SURVEY.md §8(f) ranks 1, 2, 4) at the ECDSA shape (k = 19, extended 2^21),
resident inputs, CUDA events on the launching stream; algorithmic bytes per call and the HBM fraction beside them, and
the CPU oracle timed on the same inputs.  Usage (on the GPU box): python tools/prof_quotient.py [k]"""
import os, sys, time, ctypes as C
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import halo2_lib_b200 as h
from halo2_lib_b200 import evaluation as ev
from halo2_lib_b200._capi import lib
from oracle import oracle as orc

k = int(sys.argv[1]) if len(sys.argv) > 1 else 19
QUICK = "--quick" in sys.argv  # one repetition, no CPU leg: the target of an `ncu --set full` capture
ext_k, n, bf = k + 2, 1 << k, 5
ne = 1 << ext_k
dev = torch.device("cuda", 0)
ctx = h.Context(0)
stream = torch.cuda.Stream(device=dev); torch.cuda.set_stream(stream); ctx.set_stream(stream.cuda_stream)
rng = np.random.default_rng(5)
peak = 3350.0  # GB/s: H100 SXM data-sheet HBM3 bandwidth

def rnd(m):
    x = rng.integers(0, 1 << 62, size=(m, 4), dtype=np.int64).astype(np.uint64); x[:, 3] &= np.uint64((1 << 60) - 1); return x
host = [rnd(ne) for _ in range(10)]
d = [torch.from_numpy(x.view(np.int64)).to(dev) for x in host]
ch = rnd(4)
vp = C.c_void_p
acc = torch.from_numpy(rnd(ne).view(np.int64)).to(dev)

def timeit(label, fn, bytes_alg, cpu=None, reps=10):
    if QUICK:
        reps, cpu = 1, None
    fn(); torch.cuda.synchronize()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    tot = 0.0
    for _ in range(reps):
        flush.fill_(1)  # 256 MB > L2: every rep starts cold
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream); fn(); b.record(stream); torch.cuda.synchronize()
        tot += a.elapsed_time(b)
    ms = tot / reps
    gbs = bytes_alg / ms / 1e6
    line = f"{label:44s} {ms*1e3:9.1f} us   {bytes_alg/1e6:8.1f} MB algorithmic   {gbs:7.0f} GB/s = {gbs/peak:5.1%} of {peak:.0f}"
    if cpu:
        t0 = time.perf_counter(); cpu(); line += f"   | CPU oracle {1e3*(time.perf_counter()-t0):9.1f} ms"
    print(line, flush=True)

kw = dict(beta=ch[0], gamma=ch[1], theta=ch[2], y=ch[3])
g = ev.GraphEvaluator()
adv = [("advice", 0, r) for r in range(4)]
gate = g.add_gates([("product", ("fixed", 0, 0), ("sum", ("sum", adv[0], ("product", adv[1], adv[2])), ("negated", adv[3])))])
bd = ev.BoundGraph(g, gate, fixed=[d[0].data_ptr()], advice=[d[1].data_ptr()], **kw)
bh = ev.BoundGraph(g, gate, fixed=[host[0]], advice=[host[1]], **kw)
acc_h = rnd(ne)
timeit(f"quotient_graph (flex gate) 2^{ext_k} rows", lambda: ctx.check(lib.h2b_quotient_graph_dev(ctx.h, C.byref(bd.struct), k, ext_k, vp(acc.data_ptr()))),
       32 * ne * 4, cpu=lambda: orc.quotient_graph(bh.struct, k, ext_k, acc_h))
timeit(f"flex_gate_fold (dedicated) 2^{ext_k} rows", lambda: ctx.check(lib.h2b_flex_gate_fold_dev(ctx.h, vp(d[0].data_ptr()), vp(d[1].data_ptr()), vp(ch[3].ctypes.data), k, ext_k, vp(acc.data_ptr()))),
       32 * ne * 4, cpu=lambda: orc.flex_gate_fold(host[0], host[1], ch[3], k, ext_k, acc_h))
# ECDSA shape: 3 permutation columns (advice, constants, instance), chunk = degree - 2 = 3 -> one set
tz = (C.c_void_p * 1)(d[2].data_ptr()); tc = (C.c_void_p * 3)(d[1].data_ptr(), d[3].data_ptr(), d[4].data_ptr())
ts = (C.c_void_p * 3)(d[5].data_ptr(), d[6].data_ptr(), d[7].data_ptr())
timeit(f"permutation_fold 3 cols / 1 set 2^{ext_k} rows",
       lambda: ctx.check(lib.h2b_permutation_fold_dev(ctx.h, tz, 1, tc, ts, 3, 3, vp(d[8].data_ptr()), vp(d[9].data_ptr()), vp(d[0].data_ptr()),
                                                      vp(ch[0].ctypes.data), vp(ch[1].ctypes.data), vp(ch[3].ctypes.data), bf, k, ext_k, vp(acc.data_ptr()))),
       32 * ne * (1 + 3 + 3 + 3 + 2), cpu=lambda: orc.permutation_fold([host[2]], [host[1], host[3], host[4]], [host[5], host[6], host[7]], 3, host[8], host[9], host[0], ch[0], ch[1], ch[3], bf, k, ext_k, acc_h))
g2 = ev.GraphEvaluator()
lk = g2.add_lookup([("product", ("fixed", 0, 0), ("advice", 0, 0))], [("fixed", 1, 0)])
bl = ev.BoundGraph(g2, lk, fixed=[d[0].data_ptr(), d[3].data_ptr()], advice=[d[1].data_ptr()], **kw)
blh = ev.BoundGraph(g2, lk, fixed=[host[0], host[3]], advice=[host[1]], **kw)
timeit(f"lookup_fold (q*a in table) 2^{ext_k} rows",
       lambda: ctx.check(lib.h2b_lookup_fold_dev(ctx.h, C.byref(bl.struct), vp(d[2].data_ptr()), vp(d[4].data_ptr()), vp(d[5].data_ptr()), vp(d[8].data_ptr()),
                                                 vp(d[9].data_ptr()), vp(d[6].data_ptr()), k, ext_k, vp(acc.data_ptr()))),
       32 * ne * (3 + 3 + 3 + 2), cpu=lambda: orc.lookup_fold(blh.struct, host[2], host[4], host[5], host[8], host[9], host[6], k, ext_k, acc_h))
# opening arithmetic on 2^k coefficients
q = torch.empty((n, 4), dtype=torch.int64, device=dev)
out = np.empty(4, dtype=np.uint64)
timeit(f"kate_division 2^{k} coefficients", lambda: ctx.check(lib.h2b_kate_division_dev(ctx.h, vp(d[0].data_ptr()), n, vp(ch[0].ctypes.data), vp(q.data_ptr()))),
       32 * n * 2, cpu=lambda: orc.kate_division(host[0][:n], ch[0]))
timeit(f"eval_polynomial 2^{k} coefficients (+32 B D2H)", lambda: ctx.check(lib.h2b_eval_polynomial_dev(ctx.h, vp(d[0].data_ptr()), n, vp(ch[0].ctypes.data), vp(out.ctypes.data))),
       32 * n, cpu=lambda: orc.eval_polynomial(host[0][:n], ch[0]))
pt = (C.c_void_p * 4)(*[d[i].data_ptr() for i in range(4)])
sc = rnd(4)
timeit(f"poly_lincomb 4 x 2^{k}", lambda: ctx.check(lib.h2b_poly_lincomb_dev(ctx.h, pt, vp(sc.ctypes.data), 4, n, vp(q.data_ptr()))),
       32 * n * 5, cpu=lambda: orc.poly_lincomb([x[:n] for x in host[:4]], sc))
f = d[0][:n]
z = torch.empty((n, 4), dtype=torch.int64, device=dev)
timeit(f"grand_product 2^{k}", lambda: ctx.check(lib.h2b_grand_product_fr_dev(ctx.h, vp(f.data_ptr()), vp(ch[0].ctypes.data), n, vp(z.data_ptr()))),
       32 * n * 2, cpu=lambda: orc.grand_product(host[0][:n], ch[0]))
inv = d[1][:n].clone()
timeit(f"batch_invert 2^{k}", lambda: ctx.check(lib.h2b_batch_invert_fr_dev(ctx.h, vp(inv.data_ptr()), n)), 32 * n * 2, cpu=lambda: orc.batch_invert(host[1][:n]))

# lookup permutation: a range-check column (values < 2^16 drawn from a 2^16-entry table padded with zeros), 2^k rows
bfq = 5
u = n - (bfq + 1)
tab = np.zeros(n, dtype=np.uint64); tab[:1 << 16] = np.arange(1 << 16, dtype=np.uint64)
inp = rng.integers(0, 1 << 16, size=n).astype(np.uint64)
def to_m(v):
    x = np.zeros((n, 4), dtype=np.uint64); x[:, 0] = v
    return ctx.field_op(1, 5, x)
Tm, Am = to_m(tab), to_m(inp)
dT, dA = torch.from_numpy(Tm.view(np.int64)).to(dev), torch.from_numpy(Am.view(np.int64)).to(dev)
dPA, dPT = torch.zeros_like(dA), torch.zeros_like(dT)
timeit(f"permute_expression_pair 2^{k} rows (16-bit range table)",
       lambda: ctx.check(lib.h2b_permute_expression_pair_dev(ctx.h, vp(dA.data_ptr()), vp(dT.data_ptr()), k, bfq, vp(dPA.data_ptr()), vp(dPT.data_ptr()))),
       32 * u * 4, cpu=lambda: orc.permute_expression_pair(Am, Tm, k, bfq), reps=3)
# the same with full-width values (a theta-compressed multi-column lookup): all 32 byte positions take part in the sort
Tw = host[3][:n].copy()
Aw = Tw[rng.integers(0, u, size=n)]
dTw, dAw = torch.from_numpy(Tw.view(np.int64)).to(dev), torch.from_numpy(Aw.view(np.int64)).to(dev)
timeit(f"permute_expression_pair 2^{k} rows (254-bit values)",
       lambda: ctx.check(lib.h2b_permute_expression_pair_dev(ctx.h, vp(dAw.data_ptr()), vp(dTw.data_ptr()), k, bfq, vp(dPA.data_ptr()), vp(dPT.data_ptr()))),
       32 * u * 4, reps=3)
# keygen side: G1 FFT of 2^16 points (once per SRS; 2^19 is 8 x the points and 19/16 x the stages)
if not QUICK:
    kk = 16
    gb = np.array([0xd35d438dc58f0d9d, 0x0a78eb28f5c70b3d, 0x666ea36f7879462c, 0x0e0a77c19a07df2f,
                   0xa6ba871b8b1e1b3a, 0x14f1d651eb8e167b, 0xccdd46def0f28c58, 0x1c14ef83340fbe5e], dtype=np.uint64)
    dg = torch.empty((1 << kk, 8), dtype=torch.int64, device=dev); dgl = torch.empty_like(dg)
    ctx.check(lib.h2b_srs_setup_dev(ctx.h, vp(ch[0].ctypes.data), vp(gb.ctypes.data), kk, vp(dg.data_ptr()), None))
    timeit(f"g_to_lagrange 2^{kk} points (G1 FFT)", lambda: ctx.check(lib.h2b_g_to_lagrange_dev(ctx.h, vp(dg.data_ptr()), kk, vp(dgl.data_ptr()))),
           64 * (1 << kk) * 2, reps=2)

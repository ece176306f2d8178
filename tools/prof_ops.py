"""Per-kernel device-time breakdown of one MSM / NTT on the GPU via the library's own event hooks
(h2b_profile_*; CUB's sort kernels are not instrumented, their time is the remainder to the op total).
Usage (on the GPU box): python tools/prof_ops.py [k]"""
import os, sys, ctypes as C
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import halo2_lib_b200 as h
from halo2_lib_b200._capi import lib
import bench

k = int(sys.argv[1]) if len(sys.argv) > 1 else 19
n = 1 << k
dev = torch.device("cuda", 0)
ctx = h.Context(0)
stream = torch.cuda.Stream(device=dev); torch.cuda.set_stream(stream); ctx.set_stream(stream.cuda_stream)
rng = np.random.default_rng(1)
gbase = np.array([0xd35d438dc58f0d9d, 0x0a78eb28f5c70b3d, 0x666ea36f7879462c, 0x0e0a77c19a07df2f,
                  0xa6ba871b8b1e1b3a, 0x14f1d651eb8e167b, 0xccdd46def0f28c58, 0x1c14ef83340fbe5e], dtype=np.uint64)
sc = np.zeros((n, 4), dtype=np.uint64); sc[:, 0] = 3 + 5 * np.arange(n, dtype=np.uint64)
d_sc = torch.from_numpy(ctx.field_op(1, 5, sc).view(np.int64)).to(dev)
d_pts = torch.empty((n, 8), dtype=torch.int64, device=dev)
ctx.check(lib.h2b_g1_fixed_base_mul_dev(ctx.h, C.c_void_p(gbase.ctypes.data), C.c_void_p(d_sc.data_ptr()), n, C.c_void_p(d_pts.data_ptr())))
params = h.ParamsKZG(ctx, k, g=d_pts.data_ptr(), device_ptrs=True)
cols = {"uniform": torch.from_numpy(bench.uniform_residues(rng, n).view(np.int64)).to(dev),
        "witness": torch.from_numpy(ctx.field_op(1, 5, bench.witness_like(rng, n)).view(np.int64)).to(dev)}
out = torch.zeros(12, dtype=torch.int64, device=dev)
KERNELS = ["k_sort_count", "k_sort_partition", "k_sort_fine<0>", "k_scan", "k_sort_fine<1>", "k_accumulate", "k_collect_big", "k_collect<", "k_rowcol_sums", "k_weighted_final", "k_ntt_pass"]

def run(label, fn, reps=5):
    fn(); torch.cuda.synchronize()
    ctx.profile_reset(); ctx.profile_enable("*")
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(reps): fn()
    b.record(stream); torch.cuda.synchronize()
    ctx.profile_enable(None)
    tot = a.elapsed_time(b) / reps
    print(f"== {label}: {tot*1e3:.1f} us per op (with event overhead)")
    acc = 0
    for kn in ["k_sort_count", "k_sort_partition", "k_sort_fine<0>", "k_scan", "k_sort_fine<1>", "k_accumulate", "k_collect_big", "k_collect", "k_rowcol_sums", "k_rowcol_weights", "k_weighted_final", "k_ntt_pass"]:
        ms, cnt = ctx.profile_read(kn)
        if kn == "k_collect":
            ms2, cnt2 = ctx.profile_read("k_collect_big"); ms -= ms2; cnt -= cnt2
        if cnt:
            print(f"   {kn:20s} {cnt//reps:3d} launches  {ms/reps*1e3:9.1f} us")
            acc += ms / reps
    print(f"   {'(uninstrumented: sort, memset, gaps)':20s}      {(tot-acc)*1e3:9.1f} us")

for name, col in cols.items():
    run(f"MSM 2^{k} {name}", lambda: params.commit_dev(0, col.data_ptr(), n, out.data_ptr()))
# a prover phase of 4 commitments: every MSM on its own lane (msm.batch_group = 1) against one shared pipeline (= 4)
four = [torch.from_numpy(bench.uniform_residues(rng, n).view(np.int64)).to(dev) for _ in range(4)]
out4 = torch.zeros((4, 12), dtype=torch.int64, device=dev)
for grp in (1, 4):
    ctx.set_option("msm.batch_group", grp)
    run(f"4 x MSM 2^{k} uniform, msm.batch_group = {grp}", lambda: params.commit_batch_dev(0, [c.data_ptr() for c in four], n, out4.data_ptr()))
ctx.set_option("msm.batch_group", 0)
poly = cols["uniform"].clone()
ext = torch.empty((4 * n, 4), dtype=torch.int64, device=dev)
run(f"iNTT 2^{k}", lambda: ctx.check(lib.h2b_lagrange_to_coeff_dev(ctx.h, C.c_void_p(poly.data_ptr()), k)))
run(f"coeff_to_extended 2^{k+2}", lambda: ctx.check(lib.h2b_coeff_to_extended_dev(ctx.h, C.c_void_p(poly.data_ptr()), n, k + 2, C.c_void_p(ext.data_ptr()))))

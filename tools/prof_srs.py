"""Wall clock of creating, writing and downsizing halo2-lib's params on the device (gen_srs, ParamsKZG::write,
Params::downsize) at k = 16, 19, 20 and 23: the median of --reps runs of
  setup     ParamsKZG.setup_seeded(k) (seeded tau, g and g_lagrange on the device, the G2 pair on the host)
  compress  h2b_g1_compress_dev on both bases, device time of k_g1_compress (CUDA events), and its bytes (64 read + 32 written
            per point) per second against the HBM peak of the card
  write     ParamsKZG.write in SerdeFormat::Processed and RawBytes, including the download into host memory
and at k = 23 downsize(23 -> 19) from the resident bases and from a Processed image (ParamsKZG.read_downsized).
Usage (on the GPU box): python tools/prof_srs.py [--reps 10] [--hbm-peak-tbs 3.35]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
import halo2_lib_b200 as h
from halo2_lib_b200._capi import lib


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return 1e3 * (time.perf_counter() - t0), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ks", type=str, default="16,19,20,23")
    ap.add_argument("--hbm-peak-tbs", type=float, default=3.35, help="HBM peak of the card in TB/s (H100 SXM5 80 GB: 3.35)")
    args = ap.parse_args()
    card = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    power = q.stdout.strip() or "unknown"
    ctx = h.Context(0)
    med = lambda v: round(float(np.median(v)), 3)
    for k in [int(x) for x in args.ks.split(",")]:
        n = 1 << k
        enc = h.Poly(ctx, 2 * n)
        t = {x: [] for x in ("setup", "compress", "write_processed", "write_raw", "downsize_resident", "downsize_image")}
        image = None
        for _ in range(args.reps + 1):  # the first run warms up (workspaces, twiddle plans) and is not counted
            ms, params = timed(lambda: (h.ParamsKZG.setup_seeded(ctx, k), ctx.synchronize())[0])
            rec = {"setup": ms}
            ctx.profile_enable("k_g1_compress")
            ctx.profile_reset()
            for base in (params._g, params._gl):
                ctx.check(lib.h2b_g1_compress_dev(ctx.h, C.c_void_p(base.ptr), n, C.c_void_p(enc.ptr + 32 * n * (base is params._gl))))
            rec["compress"] = ctx.profile_read("k_g1_compress")[0]
            ctx.profile_enable(None)
            rec["write_processed"], image = timed(lambda: params.write("processed"))
            rec["write_raw"], _ = timed(lambda: params.write("raw"))
            if k == 23:
                rec["downsize_resident"], _ = timed(lambda: (params.downsize(19), ctx.synchronize()))
            params.close()
            if k == 23:
                ms, q19 = timed(lambda: (h.ParamsKZG.read_downsized(ctx, image, 19), ctx.synchronize())[0])
                rec["downsize_image"] = ms
                q19.close()
            if _ == 0:
                continue
            for x, v in rec.items():
                t[x].append(v)
        enc.free()
        gbs = 2 * n * 96 / (med(t["compress"]) * 1e-3) / 1e9
        out = {"k": k, "setup_ms": med(t["setup"]), "compress_ms": med(t["compress"]), "compress_GBps": round(gbs, 1),
               "compress_frac_hbm_peak": round(gbs / (args.hbm_peak_tbs * 1e3), 3), "write_processed_ms": med(t["write_processed"]),
               "write_raw_ms": med(t["write_raw"]), "reps": args.reps, "card": card, "power_limit": power}
        if k == 23:
            out.update(downsize_23_19_resident_ms=med(t["downsize_resident"]), downsize_23_19_image_ms=med(t["downsize_image"]))
        print(json.dumps(out), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

"""Wall clock of ProverSession.check (the MockProver-style constraint check) against ProverSession.prove on the same session,
alternating: the fp_mul bench (k = 16, 8 gate / 2 lookup columns), ECDSA (k = 19, 1 gate column, selector lookup) and the
MSM circuit (k = 20, 11 / 2).  The first check of a circuit also decodes its sigma columns; that one-off cost is reported
apart ("first_check_ms").  Every check must report the satisfied instance as satisfied.
Usage (on the GPU box): python tools/prof_check.py [--reps 10] [--warmup 2]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import halo2_lib_b200 as h
from oracle import pyref
from util import affine_to_limbs, mont, rand_ints

SHAPES = [(16, 8, 2, False), (19, 1, 0, True), (20, 11, 2, False)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    card = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    power = q.stdout.strip() or "unknown"
    ctx = h.Context(0)
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).pin_memory()
    for k, A, L, sel in SHAPES:
        rng = np.random.default_rng(k)
        n = 1 << k
        g = affine_to_limbs([pyref.G1])[0]
        bases = ctx.g1_fixed_base_mul(g, mont([3 + 5 * i for i in range(n)], pyref.R))
        params = h.ParamsKZG(ctx, k, g=bases, g_lagrange=bases)
        inst = h.synthetic_circuit(ctx, k, rng, A=A, L=L, selector_lookup=sel)
        cs = h.Circuit(ctx, k, inst["fixed"], inst["sigma"], A=A, L=L, selector_lookup=sel)
        sess = h.ProverSession(ctx, params, cs)
        rnd = pin(mont(rand_ints(rng, n, pyref.R), pyref.R))
        v, lk = pin(inst["virtual"]), pin(inst["lookup"]) if len(inst["lookup"]) else None
        bp, n_lk = inst["break_points"], len(inst["lookup"])
        lk_ptr = lk.data_ptr() if lk is not None else 0
        runs = {
            "check": lambda: sess.check(v.data_ptr(), len(inst["virtual"]), break_points=bp, lookup_ptr=lk_ptr, n_lookup=n_lk),
            "prove": lambda: sess.prove(v.data_ptr(), len(inst["virtual"]), rnd.data_ptr(), break_points=bp, lookup_ptr=lk_ptr, n_lookup=n_lk),
        }
        t0 = time.perf_counter()
        first = runs["check"]()  # decodes sigma once for the circuit
        first_ms = 1e3 * (time.perf_counter() - t0)
        assert first["satisfied"], first
        for _ in range(args.warmup):
            for fn in runs.values():
                fn()
        times = {name: [] for name in runs}
        for _ in range(args.reps):  # alternating, so that drift on a shared host hits both alike
            for name, fn in runs.items():
                t0 = time.perf_counter()
                r = fn()  # both end with a download: the device is done
                times[name].append(1e3 * (time.perf_counter() - t0))
                if name == "check":
                    assert r["satisfied"]
        med = {name: float(np.median(t)) for name, t in times.items()}
        print(json.dumps({"k": k, "A": A, "L": L, "selector_lookup": sel, "check_ms_median": round(med["check"], 3),
                          "prove_ms_median": round(med["prove"], 3), "check_over_prove": round(med["check"] / med["prove"], 4),
                          "first_check_ms": round(first_ms, 3), "check_ms_min": round(min(times["check"]), 3),
                          "check_ms_max": round(max(times["check"]), 3), "reps": args.reps, "card": card, "power_limit": power}), flush=True)
        sess.free(); cs.free(); params.close()
    ctx.close()


if __name__ == "__main__":
    main()

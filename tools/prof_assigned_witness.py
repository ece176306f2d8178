"""Wall clock of ProverSession.prove in its two witness forms, alternating on one session: the evaluated witness (every
cell a field element, looked-up cells uploaded as values) and halo2-base's own form (Rational cells as (index, d) pairs
inverted on the device, looked-up cells as virtual-column indices).  Shapes: the fp_mul bench (k = 16, 8 gate / 2 lookup
columns), ECDSA (k = 19, 1 gate column, selector lookup) and the MSM circuit (k = 20, 11 / 2), at Rational fractions of
0, 1 % and 10 %.  Both forms must give the same proof bytes; that is checked on the first proof of each pair.
Usage (on the GPU box): python tools/prof_assigned_witness.py [--reps 10] [--warmup 2]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import halo2_lib_b200 as h
from oracle import pyref
from util import affine_to_limbs, mont, rand_ints
from test_gpu_assigned_witness import halo2_base_form

SHAPES = [(16, 8, 2, False), (19, 1, 0, True), (20, 11, 2, False)]
FRACS = [0.0, 0.01, 0.10]


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
        v_eval, lk_eval = pin(inst["virtual"]), pin(inst["lookup"]) if len(inst["lookup"]) else None
        bp = inst["break_points"]
        for frac in FRACS:
            values, idx, den, lk_idx = halo2_base_form(inst, k, rng, frac=frac, n_zero_den=0 if frac == 0 else 8)
            if frac == 0:
                values, idx, den = inst["virtual"], idx[:0], den[:0]
            hv, hi, hd, hl = pin(values), pin(idx), pin(den), pin(lk_idx)
            forms = {
                "evaluated": lambda: sess.prove(v_eval.data_ptr(), len(values), rnd.data_ptr(), break_points=bp,
                                                lookup_ptr=lk_eval.data_ptr() if lk_eval is not None else 0, n_lookup=len(inst["lookup"])),
                "halo2-base": lambda: sess.prove(hv.data_ptr(), len(values), rnd.data_ptr(), break_points=bp,
                                                 rational_index_ptr=hi.data_ptr() if len(idx) else 0,
                                                 rational_den_ptr=hd.data_ptr() if len(idx) else 0, n_rational=len(idx),
                                                 lookup_index_ptr=hl.data_ptr() if len(lk_idx) else 0, n_lookup=len(lk_idx)),
            }
            first = {name: fn() for name, fn in forms.items()}
            same = all(np.array_equal(a, b) for a, b in zip(first["evaluated"]["commitments"], first["halo2-base"]["commitments"]))
            for _ in range(args.warmup):
                for fn in forms.values():
                    fn()
            times = {name: [] for name in forms}
            for _ in range(args.reps):  # alternating, so that drift on a shared host hits both forms alike
                for name, fn in forms.items():
                    t0 = time.perf_counter()
                    fn()  # ends with the download of the last commitment: the device is done
                    times[name].append(1e3 * (time.perf_counter() - t0))
            for name in forms:
                t = np.array(times[name])
                print(json.dumps({"k": k, "A": A, "L": L, "rational_fraction": frac, "R": int(len(idx)), "n_lookup": int(len(lk_idx)),
                                  "form": name, "ms_per_proof_median": round(float(np.median(t)), 3),
                                  "ms_min": round(float(t.min()), 3), "ms_max": round(float(t.max()), 3),
                                  "h2d_bytes": int(first[name]["h2d_bytes"]), "same_proof_bytes": bool(same),
                                  "card": card, "power_limit": power}), flush=True)
        sess.free(); cs.free(); params.close()
    ctx.close()


if __name__ == "__main__":
    main()

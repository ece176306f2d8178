"""Timeline of ONE resident bench step (kernel, stream, ready -> finished, microseconds after the step's first event)
from the library's own event hooks (h2b_profile_dump) on both contexts of the rig.  `ready` is when the stream reached
the launch, so a kernel that waits for SM slots behind another stream's kernel shows as a long interval.
Usage (GPU box): python tools/timeline.py [--config 3] [--k K] [--out timeline.csv]"""
import argparse, os, sys, ctypes as C, collections
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench

ap = argparse.ArgumentParser()
ap.add_argument("--config", type=int, default=3)
ap.add_argument("--k", type=int, default=None)
ap.add_argument("--out", default="timeline.csv")
ap.add_argument("--prover", action="store_true", help="one resident PROOF (ProverSession.prove) instead of the schedule step")
a = ap.parse_args()
args = argparse.Namespace(gpus=1, inject_fault=None)
rig = bench.Rig(args)
torch = rig.torch
from halo2_lib_b200._capi import lib
wl = bench.Workload(rig, bench.Schedule(a.config, a.k), want_e2e=False)
step = wl.step_resident
if a.prover:
    wl.setup_prover()
    step = wl.step_e2e_prover
for _ in range(3):
    step()
torch.cuda.synchronize()
for c in (rig.ctx, rig.ctx_ntt):
    c.profile_reset(); c.profile_enable("*")
origin = torch.cuda.Event(enable_timing=True)
end = torch.cuda.Event(enable_timing=True)
origin.record(rig.stream)
step()
end.record(rig.stream)
torch.cuda.synchronize()
if os.path.exists(a.out):
    os.remove(a.out)
for c in (rig.ctx, rig.ctx_ntt):
    c.profile_enable(None)
    c.check(lib.h2b_profile_dump(c.h, C.c_void_p(origin.cuda_event), a.out.encode()))
rows = []
for line in open(a.out):
    name, stream, s, e = line.strip().rsplit(",", 3)
    rows.append((float(s), float(e), name, stream))
rows.sort()
streams = {s: i for i, s in enumerate(dict.fromkeys(r[3] for r in rows))}
print(f"step {origin.elapsed_time(end)*1e3:.0f} us with per-launch events (they add ~5 us per launch), {len(rows)} launches, {len(streams)} streams")
busy = collections.defaultdict(float)
for s, e, name, st in rows:
    busy[name] += e - s
for name, t in sorted(busy.items(), key=lambda kv: -kv[1]):
    print(f"  {name:24s} {t:9.0f} us ready->finished, {sum(1 for r in rows if r[2] == name):3d} launches")
print("stream start_us end_us dur_us kernel")
for s, e, name, st in rows:
    print(f"{streams[st]:2d} {s:9.1f} {e:9.1f} {e - s:8.1f} {name}")

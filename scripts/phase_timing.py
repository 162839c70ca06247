"""Prints the per-phase clock budget of one fused launch (M3TB_TIMING=1)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import importlib, os, sys
import numpy as np
os.environ["M3TB_TIMING"] = "1"
pkg = importlib.import_module("3dobjecttracking_b200")
capi = importlib.import_module("3dobjecttracking_b200.capi")
name = sys.argv[1] if len(sys.argv) > 1 else "c2"
wl = pkg.synth.make_workload(name, n_divides=4)
ctx = capi.context_from_workload(wl)
ctx.start_modalities(0)
for _ in range(3):
    ctx.set_poses(wl.start_body2world)
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
ctx.synchronize()
for body in (0, wl.n_bodies // 2):
    c = ctx.phase_clocks(body, 256)
    c = c[c > 0]
    d = np.diff(c)
    print(f"{name} body {body}: total {c[-1]-c[0]} cycles; prologue {d[0]}")
    per = d[1:].reshape(-1, 3 + 2 * 5)
    u = ["acc", "bar", "sum", "solve", "bar2"]
    labels = ["views", "region", "depth"] + [x + "0" for x in u] + [x + "1" for x in u]
    print("   " + " ".join(f"{l:>7}" for l in labels))
    for row in per:
        print("   " + " ".join(f"{v:7d}" for v in row))
    print("   " + " ".join(f"{v:7d}" for v in per.sum(0)), " <- sum")

"""Runs three frames of the c4 workload through the library M3TB_LIB names (default: the in-tree build) and dumps the poses
and the per-line / per-point state: variants that claim to be bit-exact must produce identical files."""
import os, sys, importlib
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
pkg = importlib.import_module("3dobjecttracking_b200")
capi = importlib.import_module("3dobjecttracking_b200.capi")
wl = pkg.synth.make_workload(sys.argv[2] if len(sys.argv) > 2 else "c4", n_divides=4)
ctx = capi.context_from_workload(wl)
ctx.start_modalities(0)
out = []
ctx.set_poses(wl.start_body2world)
for it in range(3):
    ctx.tracking_step(it, wl.n_corr_iterations, wl.n_update_iterations)
    out.append(ctx.get_poses().copy())
lines = ctx.get_region_lines(0, 1024) if wl.region else None
np.savez(sys.argv[1], poses=np.stack(out), lines=np.frombuffer(lines.tobytes(), np.uint8) if lines is not None else np.zeros(1, np.uint8))

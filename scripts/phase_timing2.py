"""Per-phase clock budget of one fused k_track2 launch (M3TB_TIMING=1): warp 0 (lines + solve) and, for bodies
with both modalities, the first point warp."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import importlib
import numpy as np
os.environ["M3TB_TIMING"] = "1"
pkg = importlib.import_module("3dobjecttracking_b200")
capi = importlib.import_module("3dobjecttracking_b200.capi")
name = sys.argv[1] if len(sys.argv) > 1 else "c4"
wl = pkg.synth.make_workload(name, n_divides=4)
ctx = capi.context_from_workload(wl)
ctx.start_modalities(0)
for _ in range(3):
    ctx.set_poses(wl.start_body2world)
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
ctx.synchronize()
nc, nu = wl.n_corr_iterations, wl.n_update_iterations
# makespan view: per-body duration of the launch (first to last stamp of warp 0) against the body's depth
tot, first, last = [], [], []
for b in range(wl.n_bodies):
    c = ctx.phase_clocks(b, 256)
    a = c[:112][c[:112] > 0]
    tot.append(int(a[-1] - a[0])); first.append(int(a[0])); last.append(int(a[-1]))
tot = np.array(tot)
w2c = np.asarray(wl.color_world2camera, np.float64)
z = np.array([w2c[2, :3] @ wl.gt_body2world[b][:, 3] + w2c[2, 3] for b in range(wl.n_bodies)])
order = np.argsort(tot)
print(f"{name}: per-body cycles min {tot.min()} median {int(np.median(tot))} max {tot.max()}; corr(total, z) = {np.corrcoef(tot, z)[0,1]:.2f}")
print("   slowest bodies: " + ", ".join(f"{b}: {tot[b]} (z {z[b]:.3f})" for b in order[-6:]))
print("   fastest bodies: " + ", ".join(f"{b}: {tot[b]} (z {z[b]:.3f})" for b in order[:4]))
slow = int(order[-1])
both = bool(wl.region and wl.depth)
for body in (0, slow):
    c = ctx.phase_clocks(body, 256)
    a = c[:112][c[:112] > 0]
    d = np.diff(a)
    print(f"{name} body {body}: warp 0 total {a[-1]-a[0]} cycles; prologue {d[0]}")
    det = {k: int(c[k] - a[0]) for k in (120, 121, 122, 124, 125, 126, 118, 119) if c[k] > 0}
    print("   prologue detail (cycles after the first stamp): parameters in shared memory %s, staging + mbarriers %s, pose products %s; "
          "tile thread: start %s, tiles sized %s, TMA issued %s; first iteration: before the LUT / tile waits %s, after %s"
          % tuple(det.get(k, "-") for k in (120, 121, 122, 124, 125, 126, 118, 119)))
    per_corr = 2 * (1 if both else (int(bool(wl.region)) + int(bool(wl.depth)))) + 5 * nu
    rows = d[1:1 + nc * per_corr].reshape(nc, per_corr)
    labels = (["view", "lines"] if wl.region else []) + (["view_d", "points"] if (wl.depth and not both) else [])
    for u in range(nu):
        labels += [f"acc{u}", f"bar{u}", f"sum{u}", f"solve{u}", f"bar2_{u}"]
    print("   " + " ".join(f"{l:>7}" for l in labels))
    for row in rows:
        print("   " + " ".join(f"{v:7d}" for v in row))
    print("   " + " ".join(f"{v:7d}" for v in rows.sum(0)), " <- sum")
    if both:
        b = c[128:][c[128:] > 0]
        e = np.diff(b)
        per = 2 + 3 * nu  # view, points; per update: accumulate + reduce, all warps arrived, released
        rows = e[1:1 + nc * per].reshape(nc, per)
        labels = ["view_d", "points"]
        for u in range(nu):
            labels += [f"acc{u}", f"wait{u}", f"rel{u}"]
        print(f"   point warp: total {b[-1]-b[0]}, start offset vs warp 0 {b[0]-a[0]}; prologue {e[0]}")
        print("   " + " ".join(f"{l:>7}" for l in labels))
        for row in rows:
            print("   " + " ".join(f"{v:7d}" for v in row))
        print("   " + " ".join(f"{v:7d}" for v in rows.sum(0)), " <- sum")

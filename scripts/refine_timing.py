"""Cost of a pose refinement (m3tb_refine_poses, Refiner::RefinePoses) at the benchmark's shape: 128 bodies of the c4
workload (region + depth, one 640x480 colour / depth pair each). Times, with CUDA events around K refinements (three
windows per measurement, alternating), a refinement of 1 body and of all 128 bodies, 7 correspondence x 2 update iterations (the Refiner's defaults), and
counts the kernel launches of one refinement. For comparison, the same 7 x 2 iterations of all bodies as the
start_modalities + corr_iteration composition. Prints one JSON line with the card's name and power limit.

    python scripts/refine_timing.py [K]"""
import importlib
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

pkg = importlib.import_module("3dobjecttracking_b200")
capi = importlib.import_module("3dobjecttracking_b200.capi")

K = int(sys.argv[1]) if len(sys.argv) > 1 else 200
REPEATS = 3  # timed windows per measurement, alternating between the measurements: their spread is reported
N_BODIES, N_CORR, N_UPDATE = 128, 7, 2


def gpu_info():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def time_ms(ctx, fn):
    """Mean milliseconds of fn() over K calls, CUDA events on the context's stream (after 3 warm-up calls)."""
    for _ in range(3):
        fn()
    ctx.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(STREAM)
    for _ in range(K):
        fn()
    end.record(STREAM)
    end.synchronize()
    return start.elapsed_time(end) / K


STREAM = torch.cuda.Stream()
wl = pkg.synth.make_workload("c4", n_bodies=N_BODIES, n_divides=2, seed=0)
ctx = capi.context_from_workload(wl, stream=STREAM.cuda_stream)
ctx.start_modalities(0)
ctx.synchronize()
out = dict(bodies=N_BODIES, n_corr_iterations=N_CORR, n_update_iterations=N_UPDATE, K=K, gpu=gpu_info())


def composition():
    for corr in range(N_CORR):
        ctx.start_modalities(0)
        ctx.corr_iteration(0, corr, N_UPDATE)


cases = {"one_body": lambda: ctx.refine_poses([17], (), N_CORR, N_UPDATE),
         "all_bodies": lambda: ctx.refine_poses(range(N_BODIES), (), N_CORR, N_UPDATE),
         "composition_all_bodies": composition}
for name, fn in cases.items():
    n0 = ctx.launch_count
    fn()
    out[name + "_launches"] = ctx.launch_count - n0
times = {name: [] for name in cases}
for _ in range(REPEATS):
    for name, fn in cases.items():
        ctx.set_poses(wl.start_body2world)
        times[name].append(round(time_ms(ctx, fn), 4))
for name, t in times.items():
    out[name + "_ms"] = sorted(t)[len(t) // 2]
    out[name + "_ms_windows"] = t
ctx.close()
print(json.dumps(out))

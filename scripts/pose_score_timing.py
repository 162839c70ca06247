"""m3tb_score_poses and m3tb_calculate_diameters against the CPU restatement built with -O3 -march=native -fopenmp
(tests/pose_score_oracle.cpp, brute-force nearest neighbours, OpenMP over bodies).

Shapes: 1, 128 and 1024 bodies sharing one model; 1000 evaluation vertices (set_n_vertices_evaluation(1000) of
evaluate_{ycb,rtb,opt}_dataset.cpp); full sets of 2,000, 20,000 and 100,000 vertices.
Device: CUDA events around back-to-back calls with device ground truth and device outputs (the two launches and the
call's host work), in REPS windows after a warm-up; the median window and the range are reported.
CPU: one call over 1 body and one over CPU_BODIES bodies per full set, each repeated REPS times after a warm-up call
(which also starts the OpenMP threads); the median and the range are reported. The CPU time of n bodies is the
CPU_BODIES median per body times n: an extrapolation (OpenMP parallelises over bodies, so it scales linearly once the
bodies outnumber the cores), not a measurement.
Diameters: one call for one model, device against the OpenMP all-pairs loop (100,000 vertices on the CPU are not run:
1e10 pairs). The equality checks use the strict build: the native one contracts products into FMAs. Also reports the
fp32 operations each call needs and the rate they imply. Prints the card name and power limit, then one JSON line per
case; the rows are also written as a JSON list to the path given as the first argument, if any."""
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

capi = importlib.import_module("3dobjecttracking_b200.capi")
import pose_score_oracle as pso  # noqa: E402
from scipy.spatial.transform import Rotation  # noqa: E402

CPU_BODIES = int(os.environ.get("CPU_BODIES", "64"))
REPS = int(os.environ.get("REPS", "5"))
N_EVAL = 1000
FLOPS_PER_PAIR = 9  # 3 subtractions, 3 products, 2 sums, 1 comparison


def poses(n, rng):
    out = np.zeros((n, 3, 4), np.float32)
    out[:, :, :3] = Rotation.from_rotvec(rng.normal(0, 0.5, (n, 3))).as_matrix()
    out[:, :, 3] = rng.normal(0, 0.3, (n, 3))
    return out


def timed(ctx, call, n):
    """ms per call over n back-to-back calls on a stream of our own, in REPS windows after a warm-up: (median, min,
    max) of the windows."""
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    for _ in range(3):
        call()
    ctx.synchronize()
    windows = []
    for _ in range(REPS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(n):
            call()
        e1.record(stream)
        e1.synchronize()
        windows.append(e0.elapsed_time(e1) / n)
    return float(np.median(windows)), min(windows), max(windows)


def cpu_timed(call):
    """ms of one call, REPS times after a warm-up call: (median, min, max)."""
    call()
    t = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        call()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t)), min(t), max(t)


def r(x, d=3):
    return [round(v, d) for v in x]


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip())
    print("cpu cores:", os.cpu_count())
    rows = []
    rng = np.random.default_rng(0)
    native = pso.native()
    for n_full in (2000, 20000, 100000):
        v = (rng.standard_normal((n_full, 3)) * 0.1).astype(np.float32)
        reduced = pso.reduce_vertices(v, N_EVAL)
        gt_cpu = poses(CPU_BODIES, rng)
        est_cpu = gt_cpu.copy()
        est_cpu[:, :, 3] += rng.normal(0, 0.01, (CPU_BODIES, 3)).astype(np.float32)
        cpu = {}
        for k in (1, CPU_BODIES):
            cpu[k] = cpu_timed(lambda: pso.score_poses([(reduced, v)], np.zeros(k, np.int32), est_cpu[:k], gt_cpu[:k],
                                                       lib=native))
        for n in (1, 128, 1024):
            ctx = capi.Context(0, max_bodies=n, max_cameras=1, max_models=1)
            ctx.set_evaluation_model(0, v, N_EVAL)
            for b in range(n):
                ctx.set_body_evaluation_model(b, 0)
            gt = poses(n, rng)
            est = gt.copy()
            est[:, :, 3] += rng.normal(0, 0.01, (n, 3)).astype(np.float32)
            ctx.set_poses(est)
            bodies = np.arange(n)
            g = torch.from_numpy(gt).cuda()
            out = torch.zeros((n, 7), dtype=torch.float32, device="cuda")
            ca = torch.zeros((n, 100), dtype=torch.float32, device="cuda")
            cs = torch.zeros((n, 100), dtype=torch.float32, device="cuda")
            reps = max(3, min(200, int(2e11 / (n * N_EVAL * n_full))))
            gpu = timed(ctx, lambda: ctx.score_poses_to(bodies, g.data_ptr(), 1, out.data_ptr(), ca.data_ptr(),
                                                        cs.data_ptr()), reps)
            dev = ctx.score_poses(bodies, gt)[0]
            strict, _ = pso.score_poses([(reduced, v)], np.zeros(min(n, 8), np.int32), est[:8], gt[:8])
            equal = all(np.array_equal(dev[f][:len(strict)], strict[:, i], equal_nan=True) for i, f in
                        enumerate(["add_error", "adds_error", "add_auc", "adds_auc", "translation_error"]))
            k = 1 if n == 1 else CPU_BODIES
            per_body = cpu[k][0] / k
            flop = FLOPS_PER_PAIR * n * N_EVAL * n_full
            row = dict(case="score", bodies=n, n_full=n_full, n_eval=N_EVAL, gpu_ms_median_min_max=r(gpu, 4),
                       gpu_tflops=round(flop / gpu[0] / 1e9, 2), cpu_bodies_measured=k,
                       cpu_ms_median_min_max=r(cpu[k], 2), cpu_ms_per_body=round(per_body, 3),
                       cpu_ms_all_bodies_extrapolated=round(per_body * n, 1), speedup=round(per_body * n / gpu[0], 1),
                       equal_to_strict_restatement=bool(equal))
            print(json.dumps(row), flush=True)
            rows.append(row)
            ctx.close()
        ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
        ctx.set_evaluation_model(0, v, 0)
        gpu = timed(ctx, lambda: ctx.calculate_diameters([0]), 5)
        d = ctx.calculate_diameters([0])[0]
        row = dict(case="diameter", n_full=n_full, gpu_ms_median_min_max=r(gpu),
                   gpu_tflops=round(FLOPS_PER_PAIR * n_full * n_full / 2 / gpu[0] / 1e9, 2))
        if n_full <= 20000:
            row.update(cpu_ms_median_min_max=r(cpu_timed(lambda: pso.diameter(v, lib=native)), 2),
                       equal=bool(pso.diameter(v) == d))
        else:
            row.update(cpu_ms_median_min_max=None, equal=None)
        print(json.dumps(row), flush=True)
        rows.append(row)
        ctx.close()
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()

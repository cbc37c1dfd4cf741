"""Benchmark of the batched absolute pose estimator (csrc/abs_pose.cu) on a localization-shaped workload: Q queries,
each 1000-4000 2D-3D correspondences with 50 % outliers, SIMPLE_RADIAL camera, focal + extra-parameter refinement
(what hloc-style localization runs once per query image).  Prints one JSON line.

  python tools/bench_abs_pose.py [--queries 4096] [--reps 3] [--fail-queries 132] [--cpu-sample 4] [--dump-outputs DIR]

Reports: problems/s end to end (host clock around the blocking call) and from the kernel durations of a
torch.profiler trace; the cost of all-outlier queries that run to max_num_trials; a CPU arm (the numpy oracle) on a
sample with its agreement; the card name and power limit, read in the same run.

--dump-outputs DIR writes the results of the last timed call and of the all-outlier queries as DIR/<name>.npy, so that
two builds can be compared output for output on identical, seeded inputs."""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pycolmap_b200 as pb  # noqa: E402
from oracle import abs_pose as A  # noqa: E402

CAM = dict(model=2, width=1600, height=1200, params=[1200.0, 800.0, 600.0, 0.02])
REFINE = dict(refine_focal_length=True, refine_extra_params=True)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unavailable ({e})"


def make_queries(rng, nq):
    sizes = rng.integers(1000, 4001, nq)
    return [(CAM,) + tuple(A.planted_scene(rng, int(n), CAM, outlier_ratio=0.5, noise_px=0.5)[2:4]) for n in sizes]


def kernel_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        m = re.search(r"b2m_abs_\w+_kernel", e.name)
        if m and e.device_type.name == "CUDA":
            tot[m.group(0)] = tot.get(m.group(0), 0.0) + e.device_time_total / 1e3
    return tot


def dump_outputs(out_dir, prefix, res):
    """success, inlier count, pose (quaternion x, y, z, w and translation; NaN on failure), camera parameters (NaN on
    failure) and the concatenated inlier masks of one estimate_absolute_poses call."""
    ok = [r is not None for r in res]
    nan = np.full(7, np.nan)
    arrays = {
        "success": np.array(ok, np.uint8),
        "num_inliers": np.array([r["num_inliers"] if r is not None else 0 for r in res], np.int64),
        "pose": np.array([np.r_[r["cam_from_world"].rotation.quat, r["cam_from_world"].translation] if r is not None
                          else nan for r in res], np.float64),
        "camera_params": np.array([r["camera_params"] if r is not None else np.full(len(CAM["params"]), np.nan)
                                   for r in res], np.float64),
        "inliers": np.concatenate([np.asarray(r["inliers"], np.uint8) for r in res if r is not None] +
                                  [np.zeros(0, np.uint8)]),
    }
    os.makedirs(out_dir, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, f"{prefix}_{name}.npy"), a)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--fail-queries", type=int, default=132)
    ap.add_argument("--cpu-sample", type=int, default=4)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the results of the last timed call and of the failing queries as DIR/<name>.npy")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no GPU: this benchmark measures the H100 kernels and has no CPU fallback")
    rng = np.random.default_rng(0)
    queries = make_queries(rng, a.queries)
    n_corr = sum(len(q[1]) for q in queries)
    out = dict(gpu=gpu_info(), queries=a.queries, correspondences=n_corr)
    pb.estimate_absolute_poses(queries[:64], refinement_options=REFINE)   # warm-up (module load, allocations)
    times = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        res = pb.estimate_absolute_poses(queries, refinement_options=REFINE)
        times.append(time.perf_counter() - t0)
    best = min(times)
    out["end_to_end_s"] = [round(t, 4) for t in times]
    out["problems_per_s_end_to_end"] = round(a.queries / best, 1)
    out["success"] = int(sum(r is not None for r in res))
    km = kernel_ms(lambda: pb.estimate_absolute_poses(queries, refinement_options=REFINE))
    ksum = sum(km.values())
    out["kernel_ms"] = {k: round(v, 3) for k, v in km.items()}
    out["problems_per_s_kernels"] = round(a.queries / (ksum / 1e3), 1) if ksum > 0 else None
    # failing queries: all outliers, default max_num_trials (100000)
    fq = []
    for _ in range(a.fail_queries):
        n = 1000
        fq.append((CAM, np.c_[rng.uniform(0, 1600, n), rng.uniform(0, 1200, n)], rng.uniform(-2, 2, (n, 3)) + [0, 0, 8]))
    t0 = time.perf_counter()
    fres = pb.estimate_absolute_poses(fq, refinement_options=REFINE)
    tf = time.perf_counter() - t0
    out["fail_kernel_ms"] = {k: round(v, 3) for k, v in
                             kernel_ms(lambda: pb.estimate_absolute_poses(fq[:1], refinement_options=REFINE)).items()}
    out["fail_queries"] = a.fail_queries
    out["fail_end_to_end_s"] = round(tf, 3)
    out["fail_success"] = int(sum(r is not None for r in fres))
    if a.dump_outputs:
        dump_outputs(a.dump_outputs, "queries", res)
        dump_outputs(a.dump_outputs, "fail_queries", fres)
    # CPU arm: the numpy oracle on a sample, agreement of inlier counts with the GPU
    t0 = time.perf_counter()
    agree = []
    for k in range(a.cpu_sample):
        w = A.absolute_pose_estimation(queries[k][1], queries[k][2], CAM, refinement_options=A.RefinementOptions(**REFINE))
        g = res[k]
        agree.append(bool((w is None) == (g is None) and (g is None or abs(g["num_inliers"] - w["num_inliers"])
                                                          <= max(2, 0.01 * w["num_inliers"]))))
    tc = time.perf_counter() - t0
    out["cpu_oracle_s_per_query"] = round(tc / max(1, a.cpu_sample), 3)
    out["cpu_oracle_agreement"] = f"{sum(agree)}/{len(agree)}"
    print(json.dumps(out))


if __name__ == "__main__":
    main()

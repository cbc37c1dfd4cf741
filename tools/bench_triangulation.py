"""Benchmark of batched triangulation (csrc/triangulation.cu) on a mapper-shaped workload: 1,000 cameras on a ring and
10^6 tracks whose lengths follow a geometric distribution (minimum 2, mean about 5, truncated at 300); 0.5 px noise at
f = 1200, 10 % gross outlier observations and 12 % placed 0.8-1.2 x max_error off their ray; max_error = 2 degrees and
min_tri_angle = 1.5 degrees (the incremental triangulator's settings).  Prints one JSON line.

  python tools/bench_triangulation.py [--tracks 1000000] [--reps 3] [--cpu-sample 2000]

Reports: the card name and power limit, read in the same run; end-to-end seconds (host clock around the blocking
call, best of --reps) and tracks/s; from a separate torch.profiler run, the kernel time and the host-to-device and
device-to-host copy times, the rest of the end-to-end time being host work (argument checks, packing into the
pinned staging buffers, unpacking); models scored and residual evaluations per second of kernel time; and exact
agreement with the numpy oracle on a sample, with the oracle's seconds per track.  The oracle is a specification,
not a CPU baseline, so no speedup is derived from it."""
import argparse
import json
import math
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pycolmap_b200 as pb  # noqa: E402
from oracle import triangulation as T  # noqa: E402

MAX_ERROR, MIN_TRI_ANGLE = math.radians(2.0), math.radians(1.5)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unavailable ({e})"


def track_lengths(rng, n, mean=5.0, cap=300):
    return np.minimum(1 + rng.geometric(1.0 / (mean - 1.0), n), cap)


def profile_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {"kernel": 0.0, "h2d": 0.0, "d2h": 0.0}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        if re.search(r"b2m_tri_ransac_kernel", e.name):
            tot["kernel"] += e.device_time_total / 1e3
        elif "HtoD" in e.name:
            tot["h2d"] += e.device_time_total / 1e3
        elif "DtoH" in e.name:
            tot["d2h"] += e.device_time_total / 1e3
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=1000000)
    ap.add_argument("--images", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-sample", type=int, default=2000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no GPU: this benchmark measures the H100 kernel and has no CPU fallback")
    rng = np.random.default_rng(0)
    L = track_lengths(rng, a.tracks)
    sc = T.planted_tracks(rng, L, n_images=a.images, max_error=MAX_ERROR, min_tri_angle=MIN_TRI_ANGLE)
    args = (sc["points_normalized"], L, sc["image_idx"], sc["cams_from_world"])
    opts = pb.EstimateTriangulationOptions(min_tri_angle=MIN_TRI_ANGLE, ransac=dict(max_error=MAX_ERROR))
    out = dict(gpu=gpu_info(), tracks=a.tracks, observations=int(L.sum()), mean_length=round(float(L.mean()), 3),
               max_length=int(L.max()), images=a.images)
    ctx = pb.Context(device=0)
    m0 = int(L[:1000].sum())
    ctx.estimate_triangulations(args[0][:m0], L[:1000], args[2][:m0], args[3], opts)   # warm-up (allocations)
    times = []
    for _ in range(a.reps):
        ctx.reset_stats()
        t0 = time.perf_counter()
        res = ctx.estimate_triangulations(*args, opts)
        times.append(time.perf_counter() - t0)
    st = ctx.stats()
    best = min(times)
    out["end_to_end_s"] = [round(t, 4) for t in times]
    out["tracks_per_s_end_to_end"] = round(a.tracks / best, 1)
    out["success"] = int(res["success"].sum())
    prof = profile_ms(lambda: ctx.estimate_triangulations(*args, opts))
    out["profile_ms"] = {k: round(v, 3) for k, v in prof.items()}
    out["host_ms_outside_copies_and_kernel"] = round(best * 1e3 - sum(prof.values()), 1)
    ks = prof["kernel"] / 1e3
    out["models_scored"] = int(st["tri_models_scored"])
    out["residuals"] = int(st["tri_residuals"])
    out["models_scored_per_s_kernel"] = round(st["tri_models_scored"] / ks, 1) if ks > 0 else None
    out["residuals_per_s_kernel"] = round(st["tri_residuals"] / ks, 1) if ks > 0 else None
    out["tracks_per_s_kernel"] = round(a.tracks / ks, 1) if ks > 0 else None
    # exact agreement with the oracle on the first tracks
    k = a.cpu_sample
    m = int(L[:k].sum())
    t0 = time.perf_counter()
    want = T.estimate_triangulations(args[0][:m], L[:k], args[2][:m], args[3], MIN_TRI_ANGLE,
                                     T.ransac_defaults(max_error=MAX_ERROR))
    tc = time.perf_counter() - t0
    same = (np.array_equal(want["success"], res["success"][:k]) and np.array_equal(want["num_inliers"], res["num_inliers"][:k])
            and np.array_equal(want["inliers"], res["inliers"][:m]))
    ok = want["success"]
    out["oracle_sample_tracks"] = k
    out["oracle_exact_agreement"] = bool(same)
    out["oracle_max_abs_xyz_diff"] = float(np.abs(want["xyz"][ok] - res["xyz"][:k][ok]).max()) if ok.any() else 0.0
    out["oracle_s_per_track"] = round(tc / k, 6)
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

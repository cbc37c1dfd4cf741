"""Stereo fusion (K9) on a rendered planar_scene with exact maps (no PatchMatch run): end-to-end seconds of the device
call, the counters, torch.profiler kernel time in a separate run, the card's name and power limit read in the same
process, and optionally the oracle's `rows` order on the same input as a CPU arm (a restatement of upstream, not
upstream).  Prints one JSON line.

    python tools/bench_stereo_fusion.py [--views 48 --width 1600 --height 1200] [--cpu-arm]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def scene_images(views, width, height, check_num_images):
    from pycolmap_b200 import mvs, synthetic as syn
    scene = syn.planar_scene(np.random.default_rng(0), views, width, height)
    images = []
    for i, cam in enumerate(scene["cameras"]):
        grey = syn.render_planar(scene, i)[0]
        d, n = syn.fusion_maps(scene, i)
        rgb = np.ascontiguousarray(np.stack([grey] * 3, -1))
        # every other view overlaps (the planar scene is seen by all of them); nearest grid neighbours first
        C = [-c["R"].T @ c["t"] for c in scene["cameras"]]
        ov = sorted((j for j in range(views) if j != i), key=lambda j: (np.linalg.norm(C[j] - C[i]), j))[:check_num_images]
        im = dict(depth=d, normal=n, rgb=rgb, color=rgb, overlap=ov)
        im.update(mvs.fusion_camera(cam["K"], cam["R"], cam["t"], (width, height), (width, height)))
        images.append(im)
    return images


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=48)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--height", type=int, default=1200)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--cpu-arm", action="store_true", help="also run oracle/fusion.cpp in `rows` order (slow)")
    a = ap.parse_args()
    import pycolmap_b200 as pb
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_stereo_fusion: no CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    opts = pb.StereoFusionOptions()
    t0 = time.time()
    images = scene_images(a.views, a.width, a.height, opts.check_num_images)
    prep = time.time() - t0
    times = []
    for _ in range(a.repeats):
        s0 = pb._core._stereo_fusion_stats(0)
        t = time.time()
        r = pb._core._stereo_fusion_run(images, opts, 0)  # returns after the device work and the download
        times.append(time.time() - t)
        s1 = pb._core._stereo_fusion_stats(0)
    cnt = {k: s1[k] - s0[k] for k in s1}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pb._core._stereo_fusion_run(images, opts, 0)
    import re
    kern = {}
    for e in prof.key_averages():
        m = re.search(r"b2m_fu_\w+", e.key)
        if m:
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1e6
            kern[m.group(0)] = round(kern.get(m.group(0), 0.0) + t, 4)
    out = dict(bench="stereo_fusion", card=card, views=a.views, width=a.width, height=a.height,
               scene_prep_s=round(prep, 2), device_call_s=[round(x, 3) for x in times], points=len(r["xyz"]),
               seeds=cnt["fusion_seeds"], rounds=cnt["fusion_rounds"], pops=cnt["fusion_pops"],
               deferred=cnt["fusion_deferred"],
               traversals_per_seed=round(cnt["fusion_traversals"] / max(1, cnt["fusion_seeds"]), 3),
               kernel_s_profiled=kern)
    if a.cpu_arm:
        from oracle import fusion as F
        t = time.time()
        rc = F.run(images, opts, "rows")
        out["cpu_arm_rows_restatement_s"] = round(time.time() - t, 2)
        out["cpu_arm_points"] = len(rc["xyz"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()

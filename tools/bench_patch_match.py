"""PatchMatch stereo (K8) on a rendered dense workspace: end-to-end seconds per reference image for each pass,
window samples per second from the pm_window_samples counter, kernel time per kernel family from torch.profiler in a
separate run, and the card name and power limit read in the same call.

    python tools/bench_patch_match.py --views 48 --width 1600 --height 1200 --sources "__auto__, 20" --out DIR

The workspace is written under a temporary directory (or --workdir); nothing is written in the repository."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pycolmap_b200 as pb  # noqa: E402
from pycolmap_b200 import _core, mvs  # noqa: E402
from pycolmap_b200 import synthetic as syn  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=48)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--height", type=int, default=1200)
    ap.add_argument("--sources", default="__auto__, 20")
    ap.add_argument("--workdir", default=None)
    ap.add_argument("--out", default=None, help="directory for the profiler table")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no GPU: this benchmark measures the H100")
    root = a.workdir or tempfile.mkdtemp(prefix="bench_pm_")
    ws = os.path.join(root, "ws")
    sc = syn.planar_scene(np.random.default_rng(0), a.views, a.width, a.height)
    t0 = time.time()
    syn.write_dense_workspace(ws, sc, sources=a.sources)
    render_s = time.time() - t0
    timings = {}
    orig = mvs._run

    def timed(images, cameras, depth_maps, problems, options, geom, filt):
        before = _core._patch_match_stats(0)["pm_window_samples"]
        t = time.time()
        out = orig(images, cameras, depth_maps, problems, options, geom, filt)
        dt = time.time() - t
        n = _core._patch_match_stats(0)["pm_window_samples"] - before
        timings["geometric" if geom else "photometric"] = dict(
            device_call_s=dt, problems=len(problems), s_per_image=dt / len(problems), window_samples=n,
            window_samples_per_s=n / dt)
        return out

    mvs._run = timed
    t = time.time()
    pb.patch_match_stereo(ws)
    total = time.time() - t
    res = dict(card=card(), views=a.views, width=a.width, height=a.height, sources=a.sources, render_s=render_s,
               end_to_end_s=total, end_to_end_s_per_image=total / a.views, passes=timings)
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for kind in ("photometric", "geometric"):
            for i in range(a.views):
                for p in mvs.map_paths(ws, f"view_{i:03d}.png", kind):
                    os.remove(p)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            pb.patch_match_stereo(ws)
        fam = {}
        for e in prof.key_averages():
            if "b2m_pm" in e.key:
                k = e.key.split("b2m_pm_")[1].split("_kernel")[0]
                fam[k] = fam.get(k, 0.0) + e.device_time_total / 1e6
        res["kernel_s"] = fam
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "pm_profile.txt"), "w") as f:
                f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=20))
    print(json.dumps(res))


if __name__ == "__main__":
    main()

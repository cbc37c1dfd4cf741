"""Image undistortion (K10): N JPEG files (q90) under one OPENCV camera, default UndistortCameraOptions.  Reports the
end-to-end rate of `undistort_images` from files to a written workspace (best of three), kernel time per kernel family
from torch.profiler in a separate run, and a CPU arm: OpenCV's initUndistortRectifyMap + remap (bilinear) + imencode
(quality 100) on all cores, with the same undistorted camera.  The CPU arm is an independent baseline, not upstream.
The card's name and power limit are read in the same process.  Everything is written under a temporary directory.
Prints one JSON line.

    python tools/bench_undistort.py [--n 256 --width 1600 --height 1200] [--no-cpu-arm] [--no-profile]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_input(root, n, width, height):
    """n JPEG files (quality 90) of smooth random texture, and a sparse model with one OPENCV camera."""
    from PIL import Image
    from pycolmap_b200 import mvs
    rng = np.random.default_rng(0)
    small = rng.random((height // 8 + 2, width // 8 + 2, 3))
    base = np.asarray(Image.fromarray((255 * small).astype(np.uint8)).resize((width + 64, height + 64),
                                                                              Image.BILINEAR))
    os.makedirs(os.path.join(root, "images"))
    m = mvs.SparseModel()
    f = 0.9 * width
    m.cameras[1] = (4, width, height, np.array([f, f, width / 2, height / 2, -0.18, 0.03, 0.0008, -0.0006]))
    for i in range(n):
        dx, dy = (7 * i) % 64, (13 * i) % 64
        name = f"img_{i:04d}.jpg"
        Image.fromarray(base[dy:dy + height, dx:dx + width]).save(os.path.join(root, "images", name), quality=90)
        m.images[i + 1] = (name, 1, np.eye(3), np.zeros(3))
        m.image_raw[i + 1] = (np.array([1.0, 0.0, 0.0, 0.0]), np.zeros(3), np.zeros((0, 2)), np.zeros(0, np.int64))
    mvs.write_sparse_bin(os.path.join(root, "sparse"), m)
    return m


def run_once(root, out):
    import pycolmap_b200 as pb
    shutil.rmtree(out, ignore_errors=True)
    t0 = time.perf_counter()
    pb.undistort_images(out, os.path.join(root, "sparse"), os.path.join(root, "images"))
    return time.perf_counter() - t0


def profile(root, out):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as p:
        run_once(root, out)
    fam = {}
    for e in p.key_averages():
        if e.device_type.name != "CUDA" and getattr(e, "self_device_time_total", 0) == 0:
            continue
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = e.self_cuda_time_total
        if us <= 0:
            continue
        k = e.key
        name = ("warp" if "undistort_warp" in k else "rescale" if "rescale" in k else
                "memcpy" if "Memcpy" in k or "memcpy" in k else "nvjpeg" if "nvjpeg" in k.lower() or "jpeg" in k.lower()
                else "other")
        fam[name] = fam.get(name, 0.0) + us / 1e3
    torch.cuda.synchronize()
    return {k: round(v, 2) for k, v in sorted(fam.items())}


def cpu_arm(root, model):
    import cv2
    from concurrent.futures import ThreadPoolExecutor
    import pycolmap_b200 as pb
    mid, w, h, p = model.cameras[1]
    und = pb._core._undistort_camera(pb.UndistortCameraOptions(), dict(model=mid, width=w, height=h, params=list(p)))
    K = np.array([[p[0], 0, p[2]], [0, p[1], p[3]], [0, 0, 1.0]])
    fx, fy, cx, cy = und["params"]
    newK = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    m1, m2 = cv2.initUndistortRectifyMap(K, np.array(p[4:8]), None, newK, (und["width"], und["height"]), cv2.CV_32FC1)
    names = [v[0] for v in model.images.values()]
    out = tempfile.mkdtemp(prefix="undist_cpu_", dir=root)

    def one(name):
        img = cv2.imread(os.path.join(root, "images", name), cv2.IMREAD_COLOR)
        res = cv2.remap(img, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT)
        ok, buf = cv2.imencode(".jpg", res, [cv2.IMWRITE_JPEG_QUALITY, 100])
        with open(os.path.join(out, name), "wb") as f:
            f.write(buf.tobytes())

    cv2.setNumThreads(1)
    best = None
    for _ in range(3):
        t0 = time.perf_counter()
        with ThreadPoolExecutor(os.cpu_count()) as ex:
            list(ex.map(one, names))
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return dict(images_per_s=round(len(names) / best, 2), seconds=round(best, 3), cores=os.cpu_count(),
                kind="OpenCV initUndistortRectifyMap + remap + imencode (independent CPU baseline, not upstream)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--height", type=int, default=1200)
    ap.add_argument("--no-cpu-arm", action="store_true")
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    import pycolmap_b200 as pb
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory(prefix="bench_undistort_") as root:
        model = make_input(root, a.n, a.width, a.height)
        out = os.path.join(root, "ws")
        run_once(root, out)  # warm-up: module load, nvJPEG handles, buffers
        times = [run_once(root, out) for _ in range(3)]
        best = min(times)
        mid, w, h, p = model.cameras[1]
        und = pb._core._undistort_camera(pb.UndistortCameraOptions(), dict(model=mid, width=w, height=h, params=list(p)))
        res = dict(metric="undistorted images/s, files to a written workspace", n=a.n, size=[a.width, a.height],
                   undistorted_size=[und["width"], und["height"]], value=round(a.n / best, 2), unit="images/s",
                   seconds=[round(t, 3) for t in times], input_bytes=sum(
                       os.path.getsize(os.path.join(root, "images", v[0])) for v in model.images.values()),
                   gpu=gpu[0] if gpu else "unknown")
        if not a.no_profile:
            res["kernel_ms_by_family"] = profile(root, out)
        if not a.no_cpu_arm:
            res["cpu_arm"] = cpu_arm(root, model)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

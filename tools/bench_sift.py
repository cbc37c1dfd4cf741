"""SIFT extraction benchmark: rendered 1600 x 1200 views through Sift.extract_batch, under pycolmap's Sift() defaults
and under the C++ defaults (first_octave = -1).

Per configuration: images/s end to end (host checks, copies, every kernel, results back), features per image; then, in
a separate profiled run (torch.profiler, CUDA activities), the kernel time per kernel family, the host <-> device
copies, and the achieved bytes/s of the pyramid kernels against the H100 SXM's 3.35 TB/s HBM3 (data sheet, not
measured).  Agreement with the numpy oracle is checked on one image.  The card's name and power limit are read in the
same run.

The images are `--distinct` rendered views (homography pairs of textured planes), cycled to `--images`: rendering 500
views in numpy would take longer than the benchmark, and the extractor does not cache anything across images.

    python tools/bench_sift.py [--images 512] [--distinct 16] [--out DIR]
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

import pycolmap_b200 as pb  # noqa: E402
from oracle import sift as X  # noqa: E402
from pycolmap_b200 import synthetic as syn  # noqa: E402

W, H = 1600, 1200
HBM_PEAK = 3.35e12


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                  text=True)
    return out.strip().splitlines()[0]


def pyramid_bytes(opts, n_images):
    """HBM bytes the blur passes must move per the algorithm: the vertical pass reads and writes a level, the horizontal
    pass reads it, writes the level and (for every level but the first) reads the previous level and writes the DoG."""
    S, o_min = opts["octave_resolution"], opts["first_octave"]
    total = 0
    first = True
    for o in range(o_min, o_min + opts["num_octaves"]):
        w, h = X.octave_dims(W, H, o)
        if w < 3 or h < 3:
            break
        A = 4 * w * h
        if first and X.first_level_sigma(S, o_min) > 0:
            total += 2 * A + 2 * A
        first = False
        total += (S + 2) * (2 * A + 4 * A)
    return total * n_images


def family(name):
    if "b2m_sift_" in name:
        return name.split("b2m_sift_")[1].split("_kernel")[0]
    if "Memcpy" in name or "memcpy" in name:
        return "copy " + ("HtoD" if "HtoD" in name else "DtoH" if "DtoH" in name else "DtoD" if "DtoD" in name else name)
    if "Memset" in name or "memset" in name:
        return "memset"
    return None


def profile(sift, imgs):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    torch.cuda.init()
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        sift.extract_batch(imgs)
    fam = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        f = family(e.name)
        if f is None:
            continue
        d = fam.setdefault(f, [0.0, 0])
        d[0] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
        d[1] += 1
    return {k: dict(ms=round(v[0], 3), launches=v[1]) for k, v in sorted(fam.items(), key=lambda kv: -kv[1][0])}


def oracle_agreement(sift, img, opts):
    kp, desc = sift.extract(img)
    want = X.extract(img, opts)
    same = len(kp) == len(want["keypoints"])
    r = dict(features=len(kp), oracle_features=len(want["keypoints"]), same_count=same)
    if same:
        r["xy_bit_equal"] = bool(np.array_equal(kp[:, :2], want["keypoints"][:, :2]))
        r["max_angle_diff"] = float(np.abs(np.angle(np.exp(1j * (kp[:, 3] - want["keypoints"][:, 3])))).max())
        r["max_descriptor_diff"] = int(np.abs(np.round(desc * 512) - want["descriptors"]).max())
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--distinct", type=int, default=16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    views = []
    while len(views) < a.distinct:
        v1, v2, _ = syn.homography_pair(rng, W, H, 1024)
        views += [v1, v2]
    imgs = [views[i % len(views)] for i in range(a.images)]
    result = dict(card=card(), images=a.images, distinct=len(views), size=f"{W}x{H}", configs={})
    for name, opts in [("pycolmap Sift() defaults", X.pycolmap_defaults()), ("C++ defaults (first_octave -1)", X.defaults())]:
        sift = pb.Sift(pb.SiftExtractionOptions(dict(opts)))
        sift.extract_batch(views[:4])           # warm-up: module load, buffers sized for this shape
        t0 = time.perf_counter()
        out = sift.extract_batch(imgs)
        dt = time.perf_counter() - t0
        feats = np.array([len(k) for k, _ in out])
        prof_imgs = imgs[:32]
        fam = profile(sift, prof_imgs)
        blur_ms = sum(fam[k]["ms"] for k in ("blur_v", "blur_h_dog") if k in fam)
        kernel_ms = sum(v["ms"] for k, v in fam.items() if not k.startswith("copy") and k != "memset")
        pb_bytes = pyramid_bytes(opts, len(prof_imgs))
        result["configs"][name] = dict(
            images_per_s=round(a.images / dt, 2), seconds=round(dt, 3), features_per_image=float(feats.mean()),
            profiled_images=len(prof_imgs), kernel_ms_per_image=round(kernel_ms / len(prof_imgs), 3),
            families=fam,
            pyramid=dict(bytes=pb_bytes, ms=round(blur_ms, 3),
                         TBps=round(pb_bytes / (blur_ms / 1e3) / 1e12, 3) if blur_ms else None,
                         share_of_hbm_peak=round(pb_bytes / (blur_ms / 1e3) / HBM_PEAK, 3) if blur_ms else None),
            oracle_sample=oracle_agreement(sift, views[0], opts))
        print(name, json.dumps(result["configs"][name]), file=sys.stderr, flush=True)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_sift.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

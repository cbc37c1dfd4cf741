"""Images/s of extract_features from JPEG files to a committed database, against the route without it (Pillow decode on
the host, Rec709 grey, Sift.extract_batch, database writes by hand), in one run, and the time K6 alone takes on the
same grey images (Sift.extract_batch of the device-decoded images); then, with --profile, the kernel time
of decode, grey + rescale and K6 by torch.profiler.  Prints one JSON line with the card name and power limit.

    python tools/bench_extract_features.py [--n 512] [--n-large 32] [--profile]"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pycolmap_b200 as nat  # noqa: E402
from oracle import image_io as O  # noqa: E402
from pycolmap_b200 import synthetic as syn  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def write_set(folder, n, w, h, seed):
    os.makedirs(folder)
    rng = np.random.default_rng(seed)
    tex = syn.textured_plane(rng, 1024)
    for k in range(n):
        a = 0.05 * k
        s = 0.9 * min(w, h) / 1024
        H = np.array([[s * np.cos(a), -s * np.sin(a), 0.2 * w], [s * np.sin(a), s * np.cos(a), 0.05 * h], [0, 0, 1.0]])
        Image.fromarray(syn.render_view(tex, H, w, h)).save(os.path.join(folder, f"{k:05d}.jpg"), quality=90)


def today(folder, db_path, max_image_size):
    """The route without extract_features: Pillow decode, grey, downscale by Pillow, Sift.extract_batch, writes."""
    sift = nat.Sift(nat.SiftExtractionOptions())
    names = sorted(os.listdir(folder))
    with nat.Database(db_path) as db:
        for k in range(0, len(names), 32):
            greys, dims = [], []
            for name in names[k:k + 32]:
                im = Image.open(os.path.join(folder, name))
                g = O.to_grey(np.asarray(im.convert("RGB")))
                W, H = im.size
                tw, th = O.target_size(W, H, max_image_size)
                if (tw, th) != (W, H):
                    g = np.asarray(Image.fromarray(g).resize((tw, th), Image.BILINEAR))
                greys.append(g)
                dims.append((W, H, tw, th))
            feats = sift.extract_batch(greys)
            for name, (W, H, tw, th), (kp, desc) in zip(names[k:k + 32], dims, feats):
                cid = db.add_camera(2, W, H, [1.2 * max(W, H), W / 2, H / 2, 0.0], False)
                iid = db.add_image(name, cid)
                k6 = O.keypoints6(kp, W / tw, H / th) if (tw, th) != (W, H) else O.keypoints6(kp)
                db.write_keypoints(iid, k6)
                db.write_descriptors(iid, np.round(desc * 512).astype(np.uint8))


def timed(fn):
    t = time.perf_counter()
    fn()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--n-large", type=int, default=32)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="bench_extract_")
    sets = {"1600x1200": (a.n, 1600, 1200), "4000x3000": (a.n_large, 4000, 3000)}
    out = {"card": card()}
    for label, (n, w, h) in sets.items():
        folder = os.path.join(tmp, label)
        write_set(folder, n, w, h, 1)
        nat.extract_features(os.path.join(tmp, f"warm_{label}.db"), folder, image_list=sorted(os.listdir(folder))[:2])
        t_new = timed(lambda: nat.extract_features(os.path.join(tmp, f"new_{label}.db"), folder))
        t_old = timed(lambda: today(folder, os.path.join(tmp, f"old_{label}.db"), 3200))
        # the split: K6 alone (Sift.extract_batch with the C++ defaults) on the grey images the device decoder gives
        names = sorted(os.listdir(folder))
        ctx = nat.Context(device=0)
        greys = [ctx.debug_decode_grey(open(os.path.join(folder, f), "rb").read()) for f in names]
        hw = ctx.stats()["sift_decode_hardware"] // 2
        ctx.close()
        sift = nat.Sift(nat.SiftExtractionOptions())
        sift.extract_batch(greys[:2])
        t_k6 = timed(lambda: [sift.extract_batch(greys[k:k + 32]) for k in range(0, n, 32)])
        out[label] = {"images": n, "extract_features_img_s": round(n / t_new, 2), "pillow_route_img_s": round(n / t_old, 2),
                      "extract_features_s": round(t_new, 3), "k6_alone_s": round(t_k6, 3), "hardware_decoded": hw}
    if a.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        folder = os.path.join(tmp, "4000x3000")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            nat.extract_features(os.path.join(tmp, "prof.db"), folder)
        groups = {"decode": 0.0, "grey_rescale": 0.0, "k6": 0.0, "keypoints": 0.0}
        for e in prof.key_averages():
            t = e.self_device_time_total if hasattr(e, "self_device_time_total") else e.self_cuda_time_total
            name = e.key
            if "b2m_grey" in name or "b2m_rescale" in name:
                groups["grey_rescale"] += t
            elif "b2m_sift" in name:
                groups["k6"] += t
            elif "b2m_keypoint_finish" in name:
                groups["keypoints"] += t
            elif "nvjpeg" in name.lower() or "idct" in name.lower() or "huff" in name.lower() or "jpeg" in name.lower():
                groups["decode"] += t
        out["kernel_ms_4000x3000"] = {k: round(v / 1000.0, 2) for k, v in groups.items()}
        del torch
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""ctypes front end of oracle/fusion.cpp: scalar restatement of COLMAP's stereo fusion (U:mvs/fusion.cc) over the
images K9 takes, in three seed orders -- `rows` (upstream with one thread), `schedule` (K9's rounds) and `replay` (an
explicit seed list).  TEST INFRASTRUCTURE ONLY, and the CPU arm of tools/bench_stereo_fusion.py.

An image is a dict: depth (H, W) float32 or None (no maps: neither a seed nor a target), normal (H, W, 3), mask
(H, W) uint8 or None (0 = never fused), rgb (h, w, 3) uint8 (the bitmap at camera size), P (3, 4), inv_P (3, 4),
inv_R (3, 3) and bitmap_scale (2,) as float32 (pycolmap_b200.mvs.fusion_camera), overlap [image indices]."""
import ctypes
import math
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "fusion.cpp")
_HDR = os.path.join(_HERE, "..", "pycolmap_b200", "csrc", "fusion_math.h")
_LIB = None
LATTICE = 16  # K9's lattice spacing s (csrc/fusion.cu kLattice)


def library_path():
    return os.path.join(_HERE, "liboracle_fusion.so")


def build(out=None):
    """Compile oracle/fusion.cpp into `out` (default: next to this file) unless it is up to date; returns the path."""
    so = out or library_path()
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(_SRC), os.path.getmtime(_HDR)):
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wextra", "-fno-fast-math",
                               "-ffp-contract=off", "-o", so + ".tmp", _SRC])
        os.replace(so + ".tmp", so)
    return so


def _lib():
    global _LIB
    if _LIB is None:
        try:
            so = build()
        except OSError:  # a read-only tree: build into a temporary directory
            so = build(os.path.join(tempfile.mkdtemp(prefix="b2m_oracle_"), "liboracle_fusion.so"))
        lib = ctypes.CDLL(so)
        lib.orc_fu_run.restype = ctypes.c_void_p
        lib.orc_fu_count.restype = ctypes.c_int64
        lib.orc_fu_count.argtypes = [ctypes.c_void_p, ctypes.c_int]
        lib.orc_fu_copy.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        lib.orc_fu_free.argtypes = [ctypes.c_void_p]
        _LIB = lib
    return _LIB


def options_array(opts):
    """The 12 doubles of orc_fu_run from a StereoFusionOptions-like object or dict."""
    g = (lambda k: opts[k]) if isinstance(opts, dict) else (lambda k: getattr(opts, k))
    box = g("bounding_box")
    lo, hi = box
    return np.array([g("min_num_pixels"), g("max_num_pixels"), g("max_traversal_depth"), g("max_reproj_error"),
                     g("max_depth_error"), np.float32(math.cos(float(np.float32(g("max_normal_error"))) * math.pi / 180.0)), *lo, *hi],
                    np.float64)


def run(images, options, order="schedule", seeds=None, lattice=LATTICE):
    """Fuse `images`.  Returns dict(xyz (N, 3) f32, normals (N, 3) f32, colors (N, 3) u8, visibility [int32 arrays],
    seeds (N, 3) int32 (image, row, col), order (M, 4) int32 (image, row, col, round), stats dict)."""
    mode = {"rows": 0, "schedule": 1, "replay": 2}[order]
    n = len(images)
    keep = []

    def ptr(a, dt):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dt)
        keep.append(a)
        return a.ctypes.data

    dims = np.zeros((n, 4), np.int32)
    cams = np.zeros((n, 35), np.float32)
    P = ctypes.c_void_p * max(1, n)
    dp, npp, mp, rp = P(), P(), P(), P()
    ov_off = np.zeros(n + 1, np.int32)
    ov = []
    for i, im in enumerate(images):
        has = im.get("depth") is not None
        if has:
            dims[i, :2] = im["depth"].shape[1], im["depth"].shape[0]
        rgb = np.asarray(im["rgb"], np.uint8)
        dims[i, 2:] = rgb.shape[1], rgb.shape[0]
        cams[i, :12] = np.asarray(im["P"], np.float32).ravel()
        cams[i, 12:24] = np.asarray(im["inv_P"], np.float32).ravel()
        cams[i, 24:33] = np.asarray(im["inv_R"], np.float32).ravel()
        cams[i, 33:] = np.asarray(im["bitmap_scale"], np.float32)
        dp[i] = ptr(im.get("depth") if has else None, np.float32)
        npp[i] = ptr(im.get("normal") if has else None, np.float32)
        mp[i] = ptr(im.get("mask") if has else None, np.uint8)
        rp[i] = ptr(rgb, np.uint8)
        ov += [int(j) for j in im["overlap"]]
        ov_off[i + 1] = len(ov)
    ova = np.array(ov + [0], np.int32)
    op = options_array(options)
    sd = np.ascontiguousarray(np.asarray(seeds if seeds is not None else np.zeros((0, 3)), np.int32).reshape(-1, 3))
    lib = _lib()
    h = lib.orc_fu_run(ctypes.c_int(n), dims.ctypes.data_as(ctypes.c_void_p), dp, npp, mp, rp,
                       cams.ctypes.data_as(ctypes.c_void_p), ov_off.ctypes.data_as(ctypes.c_void_p),
                       ova.ctypes.data_as(ctypes.c_void_p), op.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(mode),
                       ctypes.c_int(lattice), sd.ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(len(sd)))
    try:
        def get(what, dt, shape):
            a = np.zeros(lib.orc_fu_count(h, what), dt)
            if a.size:
                lib.orc_fu_copy(h, what, a.ctypes.data)
            return a.reshape(shape)
        xyz = get(0, np.float32, (-1, 3))
        nrm = get(1, np.float32, (-1, 3))
        col = get(2, np.uint8, (-1, 3))
        voff = get(3, np.int64, (-1,))
        vis = get(4, np.int32, (-1,))
        seeds_out = get(5, np.int32, (-1, 3))
        order_out = get(6, np.int32, (-1, 4))
        st = get(7, np.int64, (-1,))
    finally:
        lib.orc_fu_free(h)
    return dict(xyz=xyz, normals=nrm, colors=col, visibility=[vis[voff[k]:voff[k + 1]] for k in range(len(xyz))],
                seeds=seeds_out, order=order_out,
                stats=dict(pops=int(st[0]), traversals=int(st[1]), rounds=int(st[2]), deferred=int(st[3]),
                           seeds=int(st[4])))

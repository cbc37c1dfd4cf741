"""PatchMatch stereo over a COLMAP dense workspace: `patch_match_stereo` (R:pipeline/mvs.h:5-90).

A workspace is what upstream's `undistort_images` writes: `images/`, `sparse/` (cameras, images, points3D as .bin or
.txt) and `stereo/patch-match.cfg`.  This module reads the part of the sparse model PatchMatch needs (pinhole K,
cam_from_world, image names, each point's xyz and track image ids), the problem list of the configuration file, and
writes `stereo/depth_maps/<name>.<type>.bin` and `stereo/normal_maps/<name>.<type>.bin` in COLMAP's `Mat<float>`
layout, which upstream's `stereo_fusion` and `read_array` read.  The maps come from K8 (csrc/patch_match.cu) through
`_core._patch_match_run`; there is no CPU path.
"""
import math
import os
import struct
import sys

import numpy as np

from . import _core

# COLMAP camera model ids and parameter counts (U:sensor/models.h); PatchMatch takes the two pinhole models only.
_NUM_PARAMS = {0: 3, 1: 4, 2: 4, 3: 5, 4: 8, 5: 8, 6: 12, 7: 5, 8: 4, 9: 5, 10: 12}
_MODEL_NAMES = ["SIMPLE_PINHOLE", "PINHOLE", "SIMPLE_RADIAL", "RADIAL", "OPENCV", "OPENCV_FISHEYE", "FULL_OPENCV", "FOV",
                "SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE", "THIN_PRISM_FISHEYE"]


def _warn(msg):
    print(f"W [mvs.py] {msg}", file=sys.stderr, flush=True)


# ---- sparse model ----------------------------------------------------------------------------------------------------

def _quat_to_R(q):
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


class SparseModel:
    """cameras {id: (model_id, width, height, params)}, images {id: (name, camera_id, R, t)}, points {id: (xyz,
    [image ids of the track])}.  What a writer needs besides: image_raw {id: (qvec, tvec as read, xy (n, 2) float64,
    point3D ids (n,) int64)}, point_raw {id: (rgb (3,) uint8, error, track (n, 2) int64 of (image id, point2D
    index))}."""

    def __init__(self):
        self.cameras, self.images, self.points = {}, {}, {}
        self.image_raw, self.point_raw = {}, {}


def _read_bin(path):
    m = SparseModel()
    with open(os.path.join(path, "cameras.bin"), "rb") as f:
        for _ in range(struct.unpack("<Q", f.read(8))[0]):
            cid, model, w, h = struct.unpack("<iiQQ", f.read(24))
            n = _NUM_PARAMS[model]
            m.cameras[cid] = (model, w, h, np.array(struct.unpack(f"<{n}d", f.read(8 * n))))
    with open(os.path.join(path, "images.bin"), "rb") as f:
        for _ in range(struct.unpack("<Q", f.read(8))[0]):
            iid = struct.unpack("<i", f.read(4))[0]
            q = np.array(struct.unpack("<4d", f.read(32)))
            t = np.array(struct.unpack("<3d", f.read(24)))
            cid = struct.unpack("<i", f.read(4))[0]
            name = b""
            while (c := f.read(1)) != b"\0":
                name += c
            n2d = struct.unpack("<Q", f.read(8))[0]
            p2d = np.frombuffer(f.read(24 * n2d), np.dtype([("xy", "<f8", 2), ("id", "<i8")]))
            m.images[iid] = (name.decode(), cid, _quat_to_R(q), t)
            m.image_raw[iid] = (q, t, p2d["xy"].astype(np.float64).reshape(-1, 2), p2d["id"].astype(np.int64))
    with open(os.path.join(path, "points3D.bin"), "rb") as f:
        for _ in range(struct.unpack("<Q", f.read(8))[0]):
            pid = struct.unpack("<Q", f.read(8))[0]
            xyz = np.array(struct.unpack("<3d", f.read(24)))
            rgb = np.frombuffer(f.read(3), np.uint8).copy()
            err = struct.unpack("<d", f.read(8))[0]
            n = struct.unpack("<Q", f.read(8))[0]
            full = np.frombuffer(f.read(8 * n), np.int32).reshape(n, 2).astype(np.int64)
            m.points[pid] = (xyz, [int(i) for i in full[:, 0]])
            m.point_raw[pid] = (rgb, err, full)
    return m


def _lines(path):
    with open(path) as f:
        return [ln.strip() for ln in f if ln.strip() and not ln.lstrip().startswith("#")]


def _read_txt(path):
    m = SparseModel()
    for ln in _lines(os.path.join(path, "cameras.txt")):
        e = ln.split()
        m.cameras[int(e[0])] = (_MODEL_NAMES.index(e[1]), int(e[2]), int(e[3]), np.array([float(v) for v in e[4:]]))
    # images.txt: two lines per image; the second (the 2-D points) may be empty, so empty lines are kept here
    with open(os.path.join(path, "images.txt")) as f:
        rows = [ln.rstrip("\n") for ln in f if not ln.startswith("#")]
    for k in range(0, len(rows) - 1, 2):
        e = rows[k].split()
        if not e:
            continue
        q = np.array([float(v) for v in e[1:5]])
        t = np.array([float(v) for v in e[5:8]])
        m.images[int(e[0])] = (" ".join(e[9:]), int(e[8]), _quat_to_R(q), t)
        p2d = rows[k + 1].split()
        xy = np.array([[float(p2d[j]), float(p2d[j + 1])] for j in range(0, len(p2d), 3)], np.float64).reshape(-1, 2)
        m.image_raw[int(e[0])] = (q, t, xy, np.array([int(p2d[j + 2]) for j in range(0, len(p2d), 3)], np.int64))
    for ln in _lines(os.path.join(path, "points3D.txt")):
        e = ln.split()
        track = [int(v) for v in e[8::2]]
        m.points[int(e[0])] = (np.array([float(v) for v in e[1:4]]), track)
        m.point_raw[int(e[0])] = (np.array([int(v) for v in e[4:7]], np.uint8), float(e[7]),
                                  np.array([int(v) for v in e[8:]], np.int64).reshape(-1, 2))
    return m


def read_sparse(path):
    """The sparse model under `path`: the .bin files, or the .txt files when the binaries are absent
    (Reconstruction::Read)."""
    if all(os.path.isfile(os.path.join(path, f + ".bin")) for f in ("cameras", "images", "points3D")):
        return _read_bin(path)
    if all(os.path.isfile(os.path.join(path, f + ".txt")) for f in ("cameras", "images", "points3D")):
        return _read_txt(path)
    raise ValueError(f"[mvs.py] Check Failed: {path} holds cameras, images and points3D as .bin or .txt")


def pinhole_K(camera):
    """(fx, fy, cx, cy) of a SIMPLE_PINHOLE or PINHOLE camera; other models are refused (the workspace must be
    undistorted)."""
    model, _, _, p = camera
    if model == 0:
        return p[0], p[0], p[1], p[2]
    if model == 1:
        return p[0], p[1], p[2], p[3]
    raise ValueError(f"[mvs.py] Check Failed: camera model {_MODEL_NAMES[model]} is PINHOLE or SIMPLE_PINHOLE "
                     "(patch_match_stereo needs an undistorted workspace)")


# ---- problems, source selection, depth ranges --------------------------------------------------------------------------

def _tri_angles(model, ref_id, src_id, point_ids):
    c1 = -model.images[ref_id][2].T @ model.images[ref_id][3]
    c2 = -model.images[src_id][2].T @ model.images[src_id][3]
    X = np.array([model.points[p][0] for p in point_ids])
    r1, r2 = X - c1, X - c2
    cos = np.sum(r1 * r2, 1) / (np.linalg.norm(r1, axis=1) * np.linalg.norm(r2, axis=1))
    return np.degrees(np.arccos(np.clip(cos, -1.0, 1.0)))


def auto_sources(model, ref_id, num, min_triangulation_angle):
    """`__auto__, num`: the images sharing points with the reference, by number of shared points (descending; ties by
    ascending image id), keeping those whose 75th-percentile triangulation angle over the shared points is at least
    `min_triangulation_angle` degrees, the first `num` of them."""
    shared = {}
    for pid, (_, track) in model.points.items():
        ids = set(track)
        if ref_id in ids:
            for i in ids - {ref_id}:
                shared.setdefault(i, []).append(pid)
    order = sorted(shared, key=lambda i: (-len(shared[i]), i))
    out = []
    for i in order:
        if np.percentile(_tri_angles(model, ref_id, i, shared[i]), 75) >= min_triangulation_angle:
            out.append(i)
        if len(out) == num:
            break
    return out


def depth_range(model, image_id):
    """(depth_min, depth_max) of an image from the camera z of its observed points: the floor(0.01 n)-th and
    floor(0.99 n)-th smallest, times 0.75 and 1.25; None without points in front of the camera."""
    _, _, R, t = model.images[image_id]
    X = np.array([xyz for xyz, track in model.points.values() if image_id in track]).reshape(-1, 3)
    d = np.sort((X @ R.T + t)[:, 2])
    d = d[d > 0]
    if len(d) == 0:
        return None
    n = len(d)
    return float(d[min(int(0.01 * n), n - 1)]) * 0.75, float(d[min(int(0.99 * n), n - 1)]) * 1.25


def read_config(path, model, min_triangulation_angle):
    """patch-match.cfg: pairs of lines, a reference image name, then `__all__`, `__auto__, N` or a comma-separated list
    of source names.  Returns [(ref image id, [source image ids])]."""
    by_name = {v[0]: k for k, v in model.images.items()}
    lines = _lines(path)
    if len(lines) % 2:
        raise ValueError(f"[mvs.py] Check Failed: {path} holds pairs of lines (reference, sources)")
    problems = []
    for k in range(0, len(lines), 2):
        ref_name, spec = lines[k], lines[k + 1]
        if ref_name not in by_name:
            raise ValueError(f"[mvs.py] Check Failed: reference image {ref_name} of {path} is in the sparse model")
        ref = by_name[ref_name]
        if spec == "__all__":
            src = [i for i in sorted(model.images) if i != ref]
        elif spec.startswith("__auto__"):
            parts = [p.strip() for p in spec.split(",")]
            if len(parts) != 2 or not parts[1].isdigit():
                raise ValueError(f"[mvs.py] Check Failed: `__auto__, N` in {path}, got `{spec}`")
            src = auto_sources(model, ref, int(parts[1]), min_triangulation_angle)
        else:
            names = [p.strip() for p in spec.split(",") if p.strip()]
            missing = [n for n in names if n not in by_name]
            if missing:
                raise ValueError(f"[mvs.py] Check Failed: source images {missing} of {path} are in the sparse model")
            src = [by_name[n] for n in names]
        problems.append((ref, src))
    return problems


# ---- map files -------------------------------------------------------------------------------------------------------

def write_array(path, array):
    """COLMAP's Mat<float> file: `W&H&C&`, then float32 channel after channel, each row-major."""
    a = np.asarray(array, np.float32)
    a3 = a[:, :, None] if a.ndim == 2 else a
    h, w, c = a3.shape
    os.makedirs(os.path.dirname(path), exist_ok=True)
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        f.write(f"{w}&{h}&{c}&".encode())
        f.write(np.ascontiguousarray(np.transpose(a3, (2, 0, 1))).tobytes())
    os.replace(tmp, path)


def read_array(path):
    """The inverse of write_array, as upstream's scripts/python/read_write_dense.py reads it: (H, W) or (H, W, C)."""
    with open(path, "rb") as f:
        data = f.read()
    pos = 0
    dims = []
    for _ in range(3):
        end = data.index(b"&", pos)
        dims.append(int(data[pos:end]))
        pos = end + 1
    w, h, c = dims
    a = np.frombuffer(data[pos:], np.float32).reshape((w, h, c), order="F")
    return np.transpose(a, (1, 0, 2)).squeeze()


def map_paths(workspace, name, kind):
    return (os.path.join(workspace, "stereo", "depth_maps", f"{name}.{kind}.bin"),
            os.path.join(workspace, "stereo", "normal_maps", f"{name}.{kind}.bin"))


# ---- images ------------------------------------------------------------------------------------------------------------

def _decode(path, max_image_size, device):
    """Grey image of a workspace file as K7 makes it: decode (nvJPEG / host PNG), Rec709 grey, FreeImage bilinear
    rescale when larger than max_image_size."""
    with open(path, "rb") as f:
        data = f.read()
    return _core.debug_decode_grey(data, max_image_size if max_image_size > 0 else 1 << 30, device)


def scaled_K(K, orig_wh, new_wh):
    """K of an image rescaled from orig_wh to new_wh, per axis."""
    fx, fy, cx, cy = K
    sx, sy = new_wh[0] / orig_wh[0], new_wh[1] / orig_wh[1]
    return fx * sx, fy * sy, cx * sx, cy * sy


def _run(images, cameras, depth_maps, problems, options, geom, filt):
    return _core._patch_match_run(images, cameras, depth_maps, problems, options, geom, filt)


# ---- controller ----------------------------------------------------------------------------------------------------------

def patch_match_stereo(workspace_path, workspace_format="COLMAP", pmvs_option_name="option-all", options=None,
                       config_path=""):
    """Compute depth and normal maps of every reference image listed in the workspace's patch-match.cfg (or
    `config_path`), with geometric consistency when `options.geom_consistency`: first a photometric pass over every
    problem (no filter), then the geometric pass, which starts from the reference's photometric maps and reads the
    sources' photometric depth maps.  Problems whose output files exist are skipped (resume)."""
    workspace_path = os.fspath(workspace_path)
    if not os.path.isdir(workspace_path):
        raise ValueError(f"[mvs.h:20] Check Failed: ExistsDir(workspace_path) : Directory {workspace_path} does not exist.")
    fmt = workspace_format.lower()
    if fmt not in ("colmap", "pmvs"):
        raise ValueError("Invalid `workspace_format` - supported values are 'COLMAP' or 'PMVS'.")
    if fmt == "pmvs":
        raise ValueError("[mvs.py] Check Failed: workspace_format == 'COLMAP' (the PMVS workspace format is not supported)")
    if options is None:
        options = _core.PatchMatchOptions()
    elif isinstance(options, dict):
        options = _core.PatchMatchOptions(options)
    device = _core._check_patch_match_options(options)
    if options.write_consistency_graph:
        raise ValueError("[mvs.py] Check Failed: write_consistency_graph is not supported")

    model = read_sparse(os.path.join(workspace_path, "sparse"))
    cfg = config_path or os.path.join(workspace_path, "stereo", "patch-match.cfg")
    problems = read_config(cfg, model, options.min_triangulation_angle)
    passes = [("photometric", False, False), ("geometric", True, options.filter)] if options.geom_consistency else \
        [("photometric", False, options.filter)]

    grey = {}  # image id -> (grey uint8, (fx, fy, cx, cy) of the rescaled image); decoded once per call

    def load(iid):
        if iid not in grey:
            name, cid, _, _ = model.images[iid]
            path = os.path.join(workspace_path, "images", name)
            K = pinhole_K(model.cameras[cid])
            if not os.path.isfile(path):
                grey[iid] = None
            else:
                img = _decode(path, options.max_image_size, device)
                cam = model.cameras[cid]
                grey[iid] = (np.ascontiguousarray(img), scaled_K(K, (cam[1], cam[2]), (img.shape[1], img.shape[0])))
        return grey[iid]

    for kind, geom, filt in passes:
        todo = []
        for ref, src in problems:
            name = model.images[ref][0]
            if all(os.path.isfile(p) for p in map_paths(workspace_path, name, kind)):
                continue
            if not src:
                _warn(f"{name}: no source images, skipped")
                continue
            if options.depth_min != -1.0 or options.depth_max != -1.0:
                rng = (options.depth_min, options.depth_max)
            else:
                rng = depth_range(model, ref)
                if rng is None:
                    _warn(f"{name}: no sparse points in front of the camera to take a depth range from, skipped")
                    continue
            ids = [ref] + src
            missing = [model.images[i][0] for i in ids if load(i) is None]
            if geom:
                missing += [p for i in ids for p in map_paths(workspace_path, model.images[i][0], "photometric")[:1]
                            if not os.path.isfile(p)]
                missing += [p for p in map_paths(workspace_path, name, "photometric")[1:] if not os.path.isfile(p)]
            if missing:
                if not options.allow_missing_files:
                    raise ValueError(f"[mvs.py] Check Failed: the files of problem {name} exist: missing {missing}")
                _warn(f"{name}: missing {missing}, skipped")
                continue
            todo.append((ref, src, rng))
        if not todo:
            continue
        used = sorted({i for ref, src, _ in todo for i in [ref] + src})
        slot = {iid: k for k, iid in enumerate(used)}
        images = [grey[i][0] for i in used]
        cameras = np.zeros((len(used), 16))
        for k, i in enumerate(used):
            _, _, R, t = model.images[i]
            cameras[k, :4] = grey[i][1]
            cameras[k, 4:13] = R.ravel()
            cameras[k, 13:] = t
        depth_maps = None
        probs = []
        for ref, src, (dmin, dmax) in todo:
            p = dict(ref=slot[ref], image_id=ref, src=[slot[s] for s in src], depth_min=dmin, depth_max=dmax)
            if geom:
                dpath, npath = map_paths(workspace_path, model.images[ref][0], "photometric")
                p["init_depth"] = read_array(dpath)
                p["init_normal"] = read_array(npath)
            probs.append(p)
        if geom:
            depth_maps = [None] * len(used)
            for ref, src, _ in todo:
                for s in src:
                    if depth_maps[slot[s]] is None:
                        depth_maps[slot[s]] = read_array(map_paths(workspace_path, model.images[s][0], "photometric")[0])
        maps = _run(images, cameras, depth_maps, probs, options, geom, filt)
        for (ref, _, _), (depth, normal) in zip(todo, maps):
            dpath, npath = map_paths(workspace_path, model.images[ref][0], kind)
            write_array(dpath, depth)
            write_array(npath, normal)


# ---- stereo fusion (R:pipeline/mvs.h:43-90; U:mvs/fusion.cc) ----------------------------------------------------------

def fusion_camera(K, R, t, camera_wh, map_wh):
    """The per-image arrays of stereo fusion, computed in fp64 and rounded to fp32 once: P = K [R | t] with K scaled
    per axis by bitmap_scale = map size / camera size, inv_P = the top 3 rows of [P; 0 0 0 1]^-1, inv_R = R^T."""
    sx, sy = map_wh[0] / camera_wh[0], map_wh[1] / camera_wh[1]
    fx, fy, cx, cy = K
    Km = np.array([[fx * sx, 0.0, cx * sx], [0.0, fy * sy, cy * sy], [0.0, 0.0, 1.0]])
    P = Km @ np.c_[np.asarray(R, float), np.asarray(t, float)]
    inv_P = np.linalg.inv(np.r_[P, [[0.0, 0.0, 0.0, 1.0]]])[:3]
    return dict(P=P.astype(np.float32), inv_P=inv_P.astype(np.float32), inv_R=np.asarray(R, float).T.astype(np.float32),
                bitmap_scale=np.array([sx, sy], np.float32))


def overlapping_images(model, check_num_images):
    """Per image index (sparse model order), the indices of the images that share sparse points with it, by number of
    shared points (descending; ties by ascending index), the first `check_num_images` of them
    (Model::GetMaxOverlappingImages(check_num_images, 0))."""
    index = {iid: k for k, iid in enumerate(model.images)}
    n = len(index)
    shared = np.zeros((n, n), np.int64)
    for _, track in model.points.values():
        ids = sorted({index[i] for i in track if i in index})
        for a in ids:
            for b in ids:
                if a != b:
                    shared[a, b] += 1
    out = []
    for a in range(n):
        cand = [b for b in range(n) if shared[a, b] > 0]
        cand.sort(key=lambda b: (-shared[a, b], b))
        out.append(cand[:check_num_images])
    return out


def read_fusion_config(path):
    """stereo/fusion.cfg: one image name per line."""
    return _lines(path)


def write_ply(path, xyz, normals, colors):
    """Binary little-endian PLY: float x y z nx ny nz, uchar red green blue (WriteBinaryPlyPoints)."""
    n = len(xyz)
    head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
            "property float z\nproperty float nx\nproperty float ny\nproperty float nz\nproperty uchar red\n"
            "property uchar green\nproperty uchar blue\nend_header\n" % n)
    rec = np.zeros(n, np.dtype([("p", "<f4", 6), ("c", "u1", 3)]))
    rec["p"][:, :3] = xyz
    rec["p"][:, 3:] = normals
    rec["c"] = colors
    with open(path, "wb") as f:
        f.write(head.encode())
        f.write(rec.tobytes())


def read_ply(path):
    """The points of a PLY written by write_ply: (xyz (N, 3) f32, normals (N, 3) f32, colors (N, 3) u8)."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    n = int(next(ln.split()[2] for ln in data[:end].decode().splitlines() if ln.startswith("element vertex")))
    rec = np.frombuffer(data[end:], np.dtype([("p", "<f4", 6), ("c", "u1", 3)]), count=n)
    return rec["p"][:, :3].copy(), rec["p"][:, 3:].copy(), rec["c"].copy()


def write_points_visibility(path, visibility):
    """WritePointsVisibility: uint64 count, then per point a uint32 count and its uint32 image indices."""
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(visibility)))
        for v in visibility:
            f.write(struct.pack("<I", len(v)))
            f.write(np.asarray(v, "<u4").tobytes())


def read_points_visibility(path):
    with open(path, "rb") as f:
        data = f.read()
    n = struct.unpack_from("<Q", data, 0)[0]
    pos, out = 8, []
    for _ in range(n):
        m = struct.unpack_from("<I", data, pos)[0]
        out.append(np.frombuffer(data, "<u4", m, pos + 4).astype(np.int32))
        pos += 4 + 4 * m
    return out


def _write_points3D(path, xyz, colors, first_id):
    """points3D.bin of fused points: empty tracks, error -1, ids from first_id."""
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(xyz)))
        for k in range(len(xyz)):
            f.write(struct.pack("<Q3d3Bd", first_id + k, *map(float, xyz[k]), *map(int, colors[k]), -1.0))
            f.write(struct.pack("<Q", 0))


def _fusion_run(images, options, device):
    return _core._stereo_fusion_run(images, options, device)


def stereo_fusion(output_path, workspace_path, workspace_format="COLMAP", pmvs_option_name="option-all",
                  input_type="geometric", options=None):
    """Fuse the `input_type` depth and normal maps of the images listed in the workspace's stereo/fusion.cfg into a
    point cloud (K9, csrc/fusion.cu).  `output_path` is a directory (cameras.bin, images.bin of the workspace and a
    points3D.bin of the fused points) or a .ply file (plus `<output_path>.vis`).  Returns dict(xyz, normals, colors,
    visibility [int32 arrays of image indices])."""
    output_path = os.fspath(output_path)
    workspace_path = os.fspath(workspace_path)
    if not os.path.isdir(workspace_path):
        raise ValueError(f"[mvs.h:56] Check Failed: ExistsDir(workspace_path) : Directory {workspace_path} does not exist.")
    fmt = workspace_format.lower()
    if fmt not in ("colmap", "pmvs"):
        raise ValueError("Invalid `workspace_format` - supported values are 'COLMAP' or 'PMVS'.")
    if input_type not in ("photometric", "geometric"):
        raise ValueError("Invalid input type - supported values are 'photometric' and 'geometric'.")
    if fmt == "pmvs":
        raise ValueError("[mvs.py] Check Failed: workspace_format == 'COLMAP' (the PMVS workspace format is not supported)")
    if options is None:
        options = _core.StereoFusionOptions()
    elif isinstance(options, dict):
        options = _core.StereoFusionOptions(options)
    _core._check_stereo_fusion_options(options)
    to_dir = os.path.isdir(output_path)
    if not to_dir and not output_path.lower().endswith(".ply"):
        raise ValueError(f"[mvs.h:66] Check Failed: HasFileExtension(output_path, \".ply\") : Path {output_path} "
                         "does not have extension .ply")

    sparse = os.path.join(workspace_path, "sparse")
    model = read_sparse(sparse)
    ids = list(model.images)
    index = {iid: k for k, iid in enumerate(ids)}
    by_name = {v[0]: k for k, v in model.images.items()}
    names = read_fusion_config(os.path.join(workspace_path, "stereo", "fusion.cfg"))
    used = set()
    for name in names:
        if name not in by_name:
            raise ValueError(f"[mvs.py] Check Failed: image {name} of fusion.cfg is in the sparse model")
        dpath, npath = map_paths(workspace_path, name, input_type)
        if not (os.path.isfile(dpath) and os.path.isfile(npath)):
            _warn(f"{name}: no {input_type} depth and normal maps, skipped")
            continue
        used.add(index[by_name[name]])
    overlap = overlapping_images(model, options.check_num_images)
    images = []
    for k, iid in enumerate(ids):
        name, cid, R, t = model.images[iid]
        cam = model.cameras[cid]
        K = pinhole_K(cam)
        entry = dict(overlap=overlap[k], depth=None, normal=None, mask=None, color=None)
        map_wh = (cam[1], cam[2])
        if k in used:
            if options.max_image_size > 0 and max(cam[1], cam[2]) > options.max_image_size:
                raise ValueError(f"[mvs.py] Check Failed: max_image_size <= 0 or >= the image size ({name}: "
                                 f"{cam[1]} x {cam[2]}); downsized maps are not supported")
            dpath, npath = map_paths(workspace_path, name, input_type)
            depth = np.ascontiguousarray(read_array(dpath), np.float32)
            normal = np.ascontiguousarray(read_array(npath), np.float32)
            map_wh = (depth.shape[1], depth.shape[0])
            entry.update(depth=depth, normal=normal)
            if options.mask_path:
                mpath = os.path.join(options.mask_path, name + ".png")
                if os.path.isfile(mpath):
                    with open(mpath, "rb") as f:
                        mk = _core.debug_decode_png(f.read())[:, :, 0]
                    if mk.shape != depth.shape:
                        raise ValueError(f"[mvs.py] Check Failed: mask {mpath} ({mk.shape[1]} x {mk.shape[0]}) has the "
                                         f"depth map's size ({depth.shape[1]} x {depth.shape[0]})")
                    entry["mask"] = np.ascontiguousarray(mk)
            ipath = os.path.join(workspace_path, "images", name)
            if os.path.isfile(ipath):
                with open(ipath, "rb") as f:
                    entry["color"] = f.read()
        entry.update(fusion_camera(K, R, t, (cam[1], cam[2]), map_wh))
        images.append(entry)
    r = _fusion_run(images, options, 0)
    voff = r["vis_off"]
    vis = [r["vis"][voff[k]:voff[k + 1]] for k in range(len(r["xyz"]))]
    if to_dir:
        import shutil
        for f in ("cameras", "images"):
            for ext in (".bin", ".txt"):
                src = os.path.join(sparse, f + ext)
                if os.path.isfile(src):
                    shutil.copyfile(src, os.path.join(output_path, f + ext))
                    break
        _write_points3D(os.path.join(output_path, "points3D.bin"), r["xyz"], r["colors"],
                        max(model.points, default=0) + 1)
    else:
        write_ply(output_path, r["xyz"], r["normals"], r["colors"])
        write_points_visibility(output_path + ".vis", vis)
    return dict(xyz=r["xyz"], normals=r["normals"], colors=r["colors"], visibility=vis)


# ---- image undistortion (R:pipeline/images.h:96-261; U:image/undistortion.cc COLMAPUndistorter, recalled) -----------

def write_sparse_bin(path, model):
    """cameras.bin, images.bin and points3D.bin of `model` (a read_sparse model with its raw fields) under `path`, in
    the model's order.  Poses are written from the raw qvec / tvec, so they carry the input's values bit for bit."""
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "cameras.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(model.cameras)))
        for cid, (mid, w, h, p) in model.cameras.items():
            f.write(struct.pack("<iiQQ", cid, mid, w, h) + np.asarray(p, "<f8").tobytes())
    with open(os.path.join(path, "images.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(model.images)))
        for iid, (name, cid, _, _) in model.images.items():
            q, t, xy, ids = model.image_raw[iid]
            f.write(struct.pack("<i4d3di", iid, *map(float, q), *map(float, t), cid) + name.encode() + b"\0")
            rec = np.zeros(len(xy), np.dtype([("xy", "<f8", 2), ("id", "<i8")]))
            rec["xy"], rec["id"] = xy, ids
            f.write(struct.pack("<Q", len(xy)) + rec.tobytes())
    with open(os.path.join(path, "points3D.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(model.points)))
        for pid, (xyz, _) in model.points.items():
            rgb, err, track = model.point_raw[pid]
            f.write(struct.pack("<Q3d3Bd", pid, *map(float, xyz), *map(int, rgb), float(err)))
            f.write(struct.pack("<Q", len(track)) + np.asarray(track, "<i4").tobytes())


def _camera_dict(camera):
    model, w, h, p = camera
    return dict(model=int(model), width=int(w), height=int(h), params=[float(v) for v in p])


def _same_pinhole(camera, undistorted):
    """True when the undistorted camera describes the input image as it is: a pinhole input whose size, focal lengths
    and principal point UndistortCamera left unchanged.  Only such an image is copied instead of warped, so that every
    file in images/ has its camera's size and model."""
    model, w, h, p = camera
    if model not in (0, 1) or (w, h) != (undistorted["width"], undistorted["height"]):
        return False
    fx, fy, cx, cy = (p[0], p[0], p[1], p[2]) if model == 0 else tuple(p)
    return [float(fx), float(fy), float(cx), float(cy)] == [float(v) for v in undistorted["params"]]


def _write_file(path, data):
    with open(path, "wb") as f:
        f.write(data)


def _undistort_points(camera, undistorted, xy):
    """undistorted.ImgFromCam(camera.CamFromImg(xy)): the pinhole models in closed form, the others through
    b2m_cam_from_img on the device."""
    model, _, _, p = camera
    if len(xy) == 0:
        return xy
    if model in (0, 1):
        fx, fy, cx, cy = (p[0], p[0], p[1], p[2]) if model == 0 else tuple(p)
        uv = np.stack([(xy[:, 0] - cx) / fx, (xy[:, 1] - cy) / fy], 1)
    else:
        uv = _core.cam_from_img(_camera_dict(camera), np.ascontiguousarray(xy, np.float64))
    fx, fy, cx, cy = undistorted["params"]
    return np.stack([fx * uv[:, 0] + cx, fy * uv[:, 1] + cy], 1)


def _link_or_copy(src, dst, policy):
    """FileCopy(src, dst, policy): a copy, a symbolic link or a hard link."""
    import shutil
    if os.path.lexists(dst):
        os.remove(dst)
    if policy == _core.CopyType.copy:
        shutil.copyfile(src, dst)
    elif policy == getattr(_core.CopyType, "soft-link"):
        os.symlink(os.path.abspath(src), dst)
    else:
        os.link(src, dst)


_CHUNK_IMAGES = 32
_CHUNK_BYTES = 256 << 20


def _undistort_run(items, options, device):
    return _core._undistort_run(items, options, device)


def undistort_images(output_path, input_path, image_path, image_list=[], output_type="COLMAP",
                     copy_policy=None, num_patch_match_src_images=20, undistort_options=None):
    """Undistort the images of the sparse model at `input_path` (files under `image_path`) into a COLMAP dense workspace
    at `output_path`: images/ (K10, csrc/undistort.cu), sparse/ (every camera replaced by its undistorted PINHOLE
    camera, the 2-D points mapped through it; poses, points and tracks unchanged) and stereo/ (patch-match.cfg,
    fusion.cfg and the empty map directories), which patch_match_stereo and stereo_fusion read."""
    from concurrent.futures import ThreadPoolExecutor

    output_path, input_path, image_path = map(os.fspath, (output_path, input_path, image_path))
    if not os.path.isdir(input_path):
        raise ValueError(f"[images.h:105] Check Failed: ExistsDir(input_path) : Directory {input_path} does not exist.")
    if not os.path.isdir(image_path):
        raise ValueError(f"[images.h:106] Check Failed: ExistsDir(image_path) : Directory {image_path} does not exist.")
    fmt = output_type.lower()
    if fmt not in ("colmap", "pmvs", "cmp-mvs"):
        raise ValueError("Invalid `output_type` - supported values are 'COLMAP', 'PMVS' or 'CMP-MVS'.")
    if fmt != "colmap":
        raise ValueError(f"[mvs.py] Check Failed: output_type == 'COLMAP' (the {output_type} format is not supported)")
    if copy_policy is None:
        copy_policy = _core.CopyType.copy
    elif isinstance(copy_policy, str):
        copy_policy = _core.CopyType(copy_policy)
    if undistort_options is None:
        undistort_options = _core.UndistortCameraOptions()
    elif isinstance(undistort_options, dict):
        undistort_options = _core.UndistortCameraOptions(undistort_options)
    _core._check_undistort_options(undistort_options)

    model = read_sparse(input_path)
    by_name = {v[0]: k for k, v in model.images.items()}
    if image_list:
        ids = []
        for name in image_list:
            if name in by_name:
                ids.append(by_name[name])
            else:
                _warn(f"Cannot find image {name}")
    else:
        ids = list(model.images)
    for d in ("images", "sparse", "stereo/depth_maps", "stereo/normal_maps", "stereo/consistency_graphs"):
        os.makedirs(os.path.join(output_path, d), exist_ok=True)
    undistorted = {cid: _core._undistort_camera(undistort_options, _camera_dict(c)) for cid, c in model.cameras.items()}

    todo = []  # (image id, input file, output file, "jpeg" | "pixels")
    written = set()  # the images whose file is in images/
    for iid in ids:
        name, cid, _, _ = model.images[iid]
        src, dst = os.path.join(image_path, name), os.path.join(output_path, "images", name)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if _same_pinhole(model.cameras[cid], undistorted[cid]) and os.path.isfile(src):
            _link_or_copy(src, dst, copy_policy)
            written.add(iid)
            continue
        ext = os.path.splitext(name)[1].lower()
        if ext not in (".jpg", ".jpeg", ".png"):
            _warn(f"{name}: only JPEG and PNG images are written, skipped")
            continue
        if not os.path.isfile(src):
            _warn(f"Cannot read image at path {src}")
            continue
        todo.append((iid, src, dst, "pixels" if ext == ".png" else "jpeg"))

    chunks, cur, size = [], [], 0
    for t in todo:
        b = os.path.getsize(t[1])
        if cur and (len(cur) == _CHUNK_IMAGES or size + b > _CHUNK_BYTES):
            chunks.append(cur)
            cur, size = [], 0
        cur.append(t)
        size += b
    if cur:
        chunks.append(cur)

    def read(chunk):
        out = []
        for iid, src, _, kind in chunk:
            with open(src, "rb") as f:
                out.append((f.read(), _camera_dict(model.cameras[model.images[iid][1]]), kind))
        return out

    def write(chunk, results):
        for (iid, _, dst, kind), r in zip(chunk, results):
            if r["status"] != 0:
                _warn(f"{model.images[iid][0]}: {r['error'] or 'does not undistort'}, skipped")
                continue
            _write_file(dst, r["data"] if kind == "jpeg" else _core._encode_png(r["data"]))
            written.add(iid)

    # the files of chunk k + 1 are read and those of chunk k - 1 written while chunk k runs on the device
    with ThreadPoolExecutor(1) as reader, ThreadPoolExecutor(1) as writer:
        pending = reader.submit(read, chunks[0]) if chunks else None
        writing = None
        for k, chunk in enumerate(chunks):
            items = pending.result()
            if k + 1 < len(chunks):
                pending = reader.submit(read, chunks[k + 1])
            results = _undistort_run(items, undistort_options, 0)
            if writing is not None:
                writing.result()
            writing = writer.submit(write, chunk, results)
        if writing is not None:
            writing.result()

    distorted = dict(model.cameras)
    for cid in model.cameras:
        u = undistorted[cid]
        model.cameras[cid] = (u["model"], u["width"], u["height"], np.array(u["params"], np.float64))
    for iid in model.images:
        cid = model.images[iid][1]
        q, t, xy, pids = model.image_raw[iid]
        model.image_raw[iid] = (q, t, _undistort_points(distorted[cid], undistorted[cid], xy), pids)
    write_sparse_bin(os.path.join(output_path, "sparse"), model)
    # the configurations name the images that were written; a skipped image stays in sparse/ only
    done = [iid for iid in ids if iid in written]
    with open(os.path.join(output_path, "stereo", "patch-match.cfg"), "w") as f:
        for iid in done:
            f.write(model.images[iid][0] + "\n")
            f.write(f"__auto__, {num_patch_match_src_images}\n" if num_patch_match_src_images > 0 else "__all__\n")
    with open(os.path.join(output_path, "stereo", "fusion.cfg"), "w") as f:
        for iid in done:
            f.write(model.images[iid][0] + "\n")

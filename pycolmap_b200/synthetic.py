"""Seeded synthetic inputs for tests and bench.py (SURVEY.md section 8(d)).

SIFT-like descriptors follow the upstream test recipe (U:feature/sift_test.cc
CreateRandomFeatureDescriptors): g = U(0,1)^2 per element, L2-normalise, round(512 g) saturated
to uint8 -- so that dot products of matching descriptors sit near 2^18 and the acos/ratio tests
behave as on real SIFT.  Uniform random bytes would clamp every distance to acos(1) = 0.
"""
import numpy as np


def sift_like(rng, n):
    g = rng.random((n, 128)) ** 2
    g /= np.linalg.norm(g, axis=1, keepdims=True)
    return np.clip(np.round(512.0 * g), 0, 255).astype(np.uint8)


def perturb(rng, d, sigma=4.0):
    """Noisy copy of descriptors (a re-observation of the same 3-D point)."""
    x = d.astype(np.float64) + rng.normal(0.0, sigma, d.shape)
    x = np.clip(x, 0, None)
    x *= 512.0 / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-9)
    return np.clip(np.round(x), 0, 255).astype(np.uint8)


def matching_pair(rng, n1, n2, n_common, sigma=4.0):
    """Two descriptor sets sharing `n_common` (perturbed) descriptors at random positions."""
    d1 = sift_like(rng, n1)
    d2 = sift_like(rng, n2)
    n_common = min(n_common, n1, n2)
    i1 = rng.choice(n1, n_common, replace=False)
    i2 = rng.choice(n2, n_common, replace=False)
    d2[i2] = perturb(rng, d1[i1], sigma)
    return d1, d2, np.stack([i1, i2], 1)


def exhaustive_pairs(n):
    """All unordered pairs (i < j), the pair SET of ExhaustiveFeatureMatcher (row P1)."""
    i, j = np.triu_indices(n, 1)
    return np.stack([i, j], 1).astype(np.int32)


# ---------------------------------------------------------------------------------------------
# Synthetic multi-view scene (torch; runs on CPU or CUDA).  SURVEY.md section 8(d).
# ---------------------------------------------------------------------------------------------

def make_scene(n_images, n_feat, seed=0, device="cpu", window_images=24.0, vis_frac=0.45, detect_prob=0.7,
               desc_sigma=5.0, px_sigma=0.5, width=1600, height=1200, focal=1200.0, image_range=None):
    """Cameras on a circle looking at a rough cylindrical surface; SIMPLE_PINHOLE.

    Image i observes the surface points whose azimuth lies within +-w of the camera azimuth
    (w = window_images * 2*pi / n_images), each detected with probability `detect_prob`; the
    observations (noisy projections + re-normalised noisy copies of the point's base descriptor)
    are padded to exactly `n_feat` rows with distractors (fresh SIFT-like descriptors, uniform
    keypoints).  Image pairs further apart than ~2*window_images share nothing.

    image_range=(lo, hi) generates only that slice of images (same world for every slice; used by
    the multi-GPU bench where each rank produces its own shard before the NCCL all-gather).

    Returns dict(desc uint8 [n,K,128], kpts float32 [n,K,2], point_id int64 [n,K] (-1 = distractor),
                 cameras list of dict).
    """
    import math
    import torch

    dev = torch.device(device)
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    N, K = n_images, n_feat
    w = window_images * 2.0 * math.pi / N
    n_vis_target = int(vis_frac * K / detect_prob)
    P = max(16, int(n_vis_target * math.pi / w))  # a 2w window holds ~n_vis_target points
    r0, R = 4.0, 10.0
    phi = torch.rand(P, generator=g, device=dev) * (2 * math.pi)
    phi, _ = torch.sort(phi)
    rad = r0 + 0.8 * (torch.rand(P, generator=g, device=dev) - 0.5)
    zz = 3.0 * (torch.rand(P, generator=g, device=dev) - 0.5)
    X = torch.stack([rad * torch.cos(phi), rad * torch.sin(phi), zz], 1)  # [P,3]
    base = torch.rand(P, 128, generator=g, device=dev) ** 2
    base = base / base.norm(dim=1, keepdim=True) * 512.0

    lo_i, hi_i = image_range if image_range is not None else (0, N)
    n_out = hi_i - lo_i
    desc = torch.empty(n_out, K, 128, dtype=torch.uint8, device=dev)
    kpts = torch.empty(n_out, K, 2, dtype=torch.float32, device=dev)
    pid = torch.full((n_out, K), -1, dtype=torch.int64, device=dev)
    cx, cy = width / 2.0, height / 2.0
    phi_c = phi.cpu()

    def bound(x):
        return int(torch.searchsorted(phi_c, torch.tensor([x])).item())

    for i in range(lo_i, hi_i):
        gi = torch.Generator(device=dev)
        gi.manual_seed(seed * 1000003 + i + 1)  # per-image stream: independent of sharding
        o = i - lo_i
        th = 2 * math.pi * i / N
        C = torch.tensor([R * math.cos(th), R * math.sin(th), 0.0], device=dev)
        zc = -C / C.norm()                     # optical axis towards the origin
        xc = torch.tensor([-math.sin(th), math.cos(th), 0.0], device=dev)
        yc = torch.linalg.cross(zc, xc)
        Rm = torch.stack([xc, yc, zc], 0)      # world -> camera
        idx = torch.arange(bound(th - w), bound(th + w), device=dev)
        if th - w < 0:
            idx = torch.cat([torch.arange(bound(th - w + 2 * math.pi), P, device=dev), idx])
        if th + w > 2 * math.pi:
            idx = torch.cat([idx, torch.arange(0, bound(th + w - 2 * math.pi), device=dev)])
        keep = torch.rand(len(idx), generator=gi, device=dev) < detect_prob
        idx = idx[keep]
        Xc = (X[idx] - C) @ Rm.T
        u = focal * Xc[:, 0] / Xc[:, 2] + cx
        v = focal * Xc[:, 1] / Xc[:, 2] + cy
        inside = (Xc[:, 2] > 0.1) & (u >= 0) & (u < width) & (v >= 0) & (v < height)
        idx, u, v = idx[inside], u[inside], v[inside]
        nv = min(len(idx), K)
        if len(idx) > nv:
            sel = torch.randperm(len(idx), generator=gi, device=dev)[:nv]
            idx, u, v = idx[sel], u[sel], v[sel]
        d = base[idx] + desc_sigma * torch.randn(nv, 128, generator=gi, device=dev)
        d = torch.clamp(d, min=0)
        d = d / d.norm(dim=1, keepdim=True).clamp_min(1e-9) * 512.0
        d = torch.clamp(torch.round(d), 0, 255).to(torch.uint8)
        perm = torch.randperm(K, generator=gi, device=dev)
        rows_v, rows_d = perm[:nv], perm[nv:]
        desc[o, rows_v] = d
        kpts[o, rows_v, 0] = u + px_sigma * torch.randn(nv, generator=gi, device=dev)
        kpts[o, rows_v, 1] = v + px_sigma * torch.randn(nv, generator=gi, device=dev)
        pid[o, rows_v] = idx
        nd = K - nv
        if nd > 0:
            x = torch.rand(nd, 128, generator=gi, device=dev) ** 2
            x = x / x.norm(dim=1, keepdim=True) * 512.0
            desc[o, rows_d] = torch.clamp(torch.round(x), 0, 255).to(torch.uint8)
            kpts[o, rows_d, 0] = torch.rand(nd, generator=gi, device=dev) * width
            kpts[o, rows_d, 1] = torch.rand(nd, generator=gi, device=dev) * height
    cams = [dict(model=0, width=width, height=height, params=[focal, cx, cy], has_prior_focal_length=1)
            for _ in range(n_out)]
    return dict(desc=desc, kpts=kpts, point_id=pid, cameras=cams)


def textured_plane(rng, size=1024, octaves=(4, 8, 16, 32, 64)):
    """Seeded band-limited random texture in [0, 1]: a sum of bilinearly upsampled white-noise grids (one per
    period in pixels), so it has blob-like structure at every scale SIFT looks at."""
    tex = np.zeros((size, size))
    for period in octaves:
        n = size // period + 2
        g = rng.random((n, n))
        t = (np.arange(size) + 0.5) / period
        i = np.floor(t).astype(np.int64)
        f = t - i
        rows = g[i] * (1 - f)[:, None] + g[i + 1] * f[:, None]
        tex += rows[:, i] * (1 - f)[None, :] + rows[:, i + 1] * f[None, :]
    tex -= tex.min()
    return tex / tex.max()


def render_view(texture, H, width, height):
    """uint8 view of the texture plane through the homography H (texture pixel coordinates -> view pixel
    coordinates, both with pixel centres at +0.5, COLMAP's keypoint convention): bilinear sampling, clamped at the
    texture border, quantised to uint8."""
    ys, xs = np.mgrid[0:height, 0:width]
    p = np.stack([xs.ravel() + 0.5, ys.ravel() + 0.5, np.ones(xs.size)])
    q = np.linalg.solve(H, p)
    u = np.clip(q[0] / q[2] - 0.5, 0, texture.shape[1] - 1.000001)
    v = np.clip(q[1] / q[2] - 0.5, 0, texture.shape[0] - 1.000001)
    i, j = np.floor(v).astype(np.int64), np.floor(u).astype(np.int64)
    fv, fu = v - i, u - j
    val = (texture[i, j] * (1 - fu) * (1 - fv) + texture[i, j + 1] * fu * (1 - fv)
           + texture[i + 1, j] * (1 - fu) * fv + texture[i + 1, j + 1] * fu * fv)
    return np.clip(np.round(255.0 * val), 0, 255).astype(np.uint8).reshape(height, width)


def homography_pair(rng, width, height, size=1024):
    """Two rendered views of one textured plane and the planted homography from view 1 to view 2 (pixel
    coordinates with centres at +0.5)."""
    tex = textured_plane(rng, size)
    s = 0.8 * min(width, height) / size
    H1 = np.array([[s, 0.0, 0.1 * width], [0.0, s, 0.1 * height], [0.0, 0.0, 1.0]])
    a = 0.15
    R = np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])
    P = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [1e-4 / max(width, height) * 100, 0.0, 1.0]])
    c = np.array([[1.0, 0.0, width / 2], [0.0, 1.0, height / 2], [0.0, 0.0, 1.0]])
    H12 = c @ P @ R @ np.linalg.inv(c)
    H2 = H12 @ H1
    return render_view(tex, H1, width, height), render_view(tex, H2, width, height), H12


# ---------------------------------------------------------------------------------------------
# Piecewise-planar dense scene (PatchMatch stereo tests and tools/bench_patch_match.py).
# ---------------------------------------------------------------------------------------------

def planar_scene(rng, n_views, width, height, focal=None, texture_size=512, distorted=None):
    """A textured back wall and two textured, tilted rectangles in front of it (they occlude the wall and, from some
    views, each other), seen by `n_views` PINHOLE cameras on a grid near z = 0 looking towards +z.  `distorted`: None,
    or per view a COLMAP camera dict(model, params) of the width x height image that view is rendered through instead
    (stored as the camera's "camera"; K stays the pinhole one).

    Returns dict(planes, cameras [dict(K=(fx, fy, cx, cy), R, t) with x_cam = R x_world + t], width, height)."""
    focal = focal or 0.9 * width
    planes = []
    for centre, normal, half, period in (((0.0, 0.0, 12.0), (0.15, -0.1, -1.0), 12.0, 2),
                                         ((-1.2, -0.3, 7.0), (0.35, 0.1, -1.0), 1.6, 2),
                                         ((1.3, 0.6, 8.5), (-0.3, -0.25, -1.0), 1.4, 2)):
        n = np.asarray(normal, float)
        n /= np.linalg.norm(n)
        a1 = np.cross(n, [0.0, 1.0, 0.0])
        a1 /= np.linalg.norm(a1)
        a2 = np.cross(n, a1)
        tex = textured_plane(rng, texture_size, octaves=(period, 2 * period, 4 * period, 8 * period, 16 * period))
        planes.append(dict(c=np.asarray(centre, float), n=n, a1=a1, a2=a2, half=half, tex=tex))
    cams = []
    side = int(np.ceil(np.sqrt(n_views)))
    for i in range(n_views):
        gx, gy = i % side, i // side
        C = np.array([(gx - (side - 1) / 2) * 0.8, (gy - (side - 1) / 2) * 0.6, 0.0]) + rng.normal(0, 0.05, 3)
        z = np.array([0.0, 0.0, 9.0]) - C
        z /= np.linalg.norm(z)
        x = np.cross([0.0, 1.0, 0.0], z)
        x /= np.linalg.norm(x)
        y = np.cross(z, x)
        R = np.stack([x, y, z])
        cams.append(dict(K=(focal, focal, width / 2.0, height / 2.0), R=R, t=-R @ C))
        if distorted is not None:
            cams[-1]["camera"] = dict(model=distorted[i]["model"], width=width, height=height,
                                      params=list(distorted[i]["params"]))
    return dict(planes=planes, cameras=cams, width=width, height=height)


def render_planar(scene, i, offset=0.5):
    """View i of a planar_scene by ray casting: (grey uint8 [H, W], depth [H, W] (camera z), normal [H, W, 3] (camera
    frame, facing the camera), plane index [H, W]).  Rays through pixel (x + offset, y + offset): pixel centres at +0.5
    by default, integer pixel coordinates (stereo fusion's convention) with offset=0.  A view with a distorted camera
    casts its rays through CamFromImg of those pixels (oracle/ransac.py)."""
    cam = scene["cameras"][i]
    W, H = scene["width"], scene["height"]
    fx, fy, cx, cy = cam["K"]
    ys, xs = np.mgrid[0:H, 0:W]
    if "camera" in cam:
        from oracle import ransac as R
        uv = R.cam_from_img(cam["camera"], np.stack([xs.ravel() + offset, ys.ravel() + offset], 1)).reshape(H, W, 2)
        rays = np.concatenate([uv, np.ones((H, W, 1))], -1)
    else:
        rays = np.stack([(xs + offset - cx) / fx, (ys + offset - cy) / fy, np.ones((H, W))], -1)  # camera frame, z = 1
    R, t = cam["R"], cam["t"]
    C = -R.T @ t
    rw = rays @ R  # world directions (R^T r)
    best = np.full((H, W), np.inf)
    label = np.full((H, W), -1)
    for k, p in enumerate(scene["planes"]):
        den = rw @ p["n"]
        s = ((p["c"] - C) @ p["n"]) / np.where(np.abs(den) > 1e-12, den, np.nan)
        X = C + s[..., None] * rw
        u, v = (X - p["c"]) @ p["a1"], (X - p["c"]) @ p["a2"]
        hit = (s > 0) & (np.abs(u) <= p["half"]) & (np.abs(v) <= p["half"]) & (s < best)
        best = np.where(hit, s, best)
        label = np.where(hit, k, label)
    grey = np.zeros((H, W))
    normal = np.zeros((H, W, 3))
    for k, p in enumerate(scene["planes"]):
        m = label == k
        X = C + best[m][:, None] * rw[m]
        size = p["tex"].shape[0]
        u = np.clip(((X - p["c"]) @ p["a1"] / (2 * p["half"]) + 0.5) * size - 0.5, 0, size - 1.000001)
        v = np.clip(((X - p["c"]) @ p["a2"] / (2 * p["half"]) + 0.5) * size - 0.5, 0, size - 1.000001)
        i0, j0 = np.floor(v).astype(np.int64), np.floor(u).astype(np.int64)
        fv, fu = v - i0, u - j0
        tex = p["tex"]
        grey[m] = (tex[i0, j0] * (1 - fu) * (1 - fv) + tex[i0, j0 + 1] * fu * (1 - fv) + tex[i0 + 1, j0] * (1 - fu) * fv
                   + tex[i0 + 1, j0 + 1] * fu * fv)
        nc = R @ p["n"]
        if nc @ np.array([0.0, 0.0, 1.0]) > 0:  # face the camera
            nc = -nc
        normal[m] = nc
    depth = np.where(label >= 0, best, 0.0)  # s is the camera z, since the rays have z = 1 in the camera frame
    return (np.clip(np.round(255.0 * grey), 0, 255).astype(np.uint8), depth.astype(np.float32),
            normal.astype(np.float32), label)


def write_dense_workspace(path, scene, sources="__auto__, 5", points_per_view=300, seed=0):
    """A COLMAP dense workspace of a planar_scene under `path`: images/view_XXX.png, sparse/{cameras,images,
    points3D}.bin (one PINHOLE camera per view; points sampled from the views' true depths, tracked into every view
    that sees them unoccluded) and stereo/patch-match.cfg with `sources` for every view.  Returns the renders."""
    import os
    import struct
    from PIL import Image

    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(path, "images"), exist_ok=True)
    os.makedirs(os.path.join(path, "sparse"), exist_ok=True)
    os.makedirs(os.path.join(path, "stereo"), exist_ok=True)
    n = len(scene["cameras"])
    renders = [render_planar(scene, i) for i in range(n)]
    names = [f"view_{i:03d}.png" for i in range(n)]
    for i in range(n):
        Image.fromarray(renders[i][0]).save(os.path.join(path, "images", names[i]))
    W, H = scene["width"], scene["height"]
    points = []
    for i in range(n):
        cam = scene["cameras"][i]
        d = renders[i][1]
        ys, xs = rng.integers(0, H, points_per_view), rng.integers(0, W, points_per_view)
        ok = d[ys, xs] > 0
        fx, fy, cx, cy = cam["K"]
        Xc = np.stack([(xs + 0.5 - cx) / fx, (ys + 0.5 - cy) / fy, np.ones(len(xs))], 1) * d[ys, xs][:, None]
        Xw = (Xc - cam["t"]) @ cam["R"]
        for X in Xw[ok]:
            track = []
            for j in range(n):
                cj = scene["cameras"][j]
                y = cj["R"] @ X + cj["t"]
                u, v = cj["K"][0] * y[0] / y[2] + cj["K"][2], cj["K"][1] * y[1] / y[2] + cj["K"][3]
                if y[2] > 0 and 0 <= u < W and 0 <= v < H and abs(renders[j][1][int(v), int(u)] - y[2]) < 0.01 * y[2]:
                    track.append(j + 1)
            if len(track) >= 2:
                points.append((X, track))
    with open(os.path.join(path, "sparse", "cameras.bin"), "wb") as f:
        f.write(struct.pack("<Q", n))
        for i, c in enumerate(scene["cameras"]):
            f.write(struct.pack("<iiQQ4d", i + 1, 1, W, H, *c["K"]))
    with open(os.path.join(path, "sparse", "images.bin"), "wb") as f:
        f.write(struct.pack("<Q", n))
        for i, c in enumerate(scene["cameras"]):
            f.write(struct.pack("<i4d3di", i + 1, *_rot_to_quat(c["R"]), *c["t"], i + 1))
            f.write(names[i].encode() + b"\0")
            f.write(struct.pack("<Q", 0))
    with open(os.path.join(path, "sparse", "points3D.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(points)))
        for k, (X, track) in enumerate(points):
            f.write(struct.pack("<Q3d3Bd", k + 1, *X, 128, 128, 128, 0.5))
            f.write(struct.pack("<Q", len(track)))
            for j in track:
                f.write(struct.pack("<ii", j, 0))
    with open(os.path.join(path, "stereo", "patch-match.cfg"), "w") as f:
        for i in range(n):
            f.write(f"{names[i]}\n{sources}\n")
    with open(os.path.join(path, "stereo", "fusion.cfg"), "w") as f:
        for i in range(n):
            f.write(f"{names[i]}\n")
    return renders


def write_input_workspace(path, scene, points_per_view=300, seed=0, ext=".png"):
    """The input of undistort_images for a planar_scene rendered through distorted cameras: images/view_XXX<ext> and
    sparse/{cameras,images,points3D}.bin with one camera per view (its "camera", else PINHOLE K) and the 2-D
    observations of the points (sampled from the views' true depths, tracked into every view that sees them
    unoccluded).  Returns the renders."""
    import os
    from PIL import Image
    from oracle import ransac as R
    from . import mvs

    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(path, "images"), exist_ok=True)
    n = len(scene["cameras"])
    W, H = scene["width"], scene["height"]
    renders = [render_planar(scene, i) for i in range(n)]
    names = [f"view_{i:03d}{ext}" for i in range(n)]
    for i in range(n):
        Image.fromarray(renders[i][0]).save(os.path.join(path, "images", names[i]), quality=95)
    cams = [c.get("camera", dict(model=1, width=W, height=H, params=list(c["K"]))) for c in scene["cameras"]]
    m = mvs.SparseModel()
    obs = [([], []) for _ in range(n)]
    for i in range(n):
        c = scene["cameras"][i]
        d = renders[i][1]
        ys, xs = rng.integers(0, H, points_per_view), rng.integers(0, W, points_per_view)
        ok = d[ys, xs] > 0
        uv = R.cam_from_img(cams[i], np.stack([xs + 0.5, ys + 0.5], 1))
        Xc = np.c_[uv, np.ones(len(xs))] * d[ys, xs][:, None]
        for X in ((Xc - c["t"]) @ c["R"])[ok]:
            track = []
            for j in range(n):
                cj = scene["cameras"][j]
                y = cj["R"] @ X + cj["t"]
                if y[2] <= 0:
                    continue
                u, v = R.img_from_cam(cams[j], (y[:2] / y[2])[None])[0]
                if 0 <= u < W and 0 <= v < H and abs(renders[j][1][int(v), int(u)] - y[2]) < 0.01 * y[2]:
                    track.append((j, u, v))
            if len(track) >= 2:
                pid = len(m.points) + 1
                full = []
                for j, u, v in track:
                    full.append((j + 1, len(obs[j][0])))
                    obs[j][0].append((u, v))
                    obs[j][1].append(pid)
                m.points[pid] = (X, [j + 1 for j, _, _ in track])
                m.point_raw[pid] = (np.array([128, 128, 128], np.uint8), 0.5, np.array(full, np.int64))
    for i, c in enumerate(scene["cameras"]):
        m.cameras[i + 1] = (cams[i]["model"], W, H, np.array(cams[i]["params"], np.float64))
        m.images[i + 1] = (names[i], i + 1, c["R"], c["t"])
        m.image_raw[i + 1] = (np.array(_rot_to_quat(c["R"])), np.asarray(c["t"], np.float64),
                              np.array(obs[i][0], np.float64).reshape(-1, 2), np.array(obs[i][1], np.int64))
    mvs.write_sparse_bin(os.path.join(path, "sparse"), m)
    return renders


def fusion_maps(scene, i, rng=None, noise=0.0, outliers=0.0):
    """Exact depth and normal maps of view i of a planar_scene in stereo fusion's pixel convention (rays through
    integer pixel coordinates), as float32 (depth [H, W], normal [H, W, 3]).  With `rng`: depths times (1 + N(0,
    noise)), and a fraction `outliers` of the valid pixels replaced by depths uniform in [0.5, 2] x the true one."""
    _, depth, normal, _ = render_planar(scene, i, offset=0.0)
    depth = depth.astype(np.float64)
    if rng is not None:
        valid = depth > 0
        depth = np.where(valid, depth * (1.0 + rng.normal(0.0, noise, depth.shape)), 0.0)
        out = valid & (rng.random(depth.shape) < outliers)
        depth[out] *= rng.uniform(0.5, 2.0, out.sum())
    return depth.astype(np.float32), np.ascontiguousarray(normal, np.float32)


def _rot_to_quat(R):
    """(w, x, y, z) of a rotation matrix, w >= 0."""
    w = np.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    x = np.sqrt(max(0.0, 1.0 + R[0, 0] - R[1, 1] - R[2, 2])) / 2
    y = np.sqrt(max(0.0, 1.0 - R[0, 0] + R[1, 1] - R[2, 2])) / 2
    z = np.sqrt(max(0.0, 1.0 - R[0, 0] - R[1, 1] + R[2, 2])) / 2
    x = np.copysign(x, R[2, 1] - R[1, 2])
    y = np.copysign(y, R[0, 2] - R[2, 0])
    z = np.copysign(z, R[1, 0] - R[0, 1])
    return w, x, y, z

"""Stereo fusion inputs built from a rendered planar_scene: exact (or noisy) maps in fusion's pixel convention, the
renders as colours, overlap lists from the views' mutual visibility.  One image dict serves both the oracle
(oracle/fusion.py reads `rgb`) and the device call (pycolmap_b200._core._stereo_fusion_run reads `color`)."""
import numpy as np

from pycolmap_b200 import mvs, synthetic as syn


def fusion_images(n_views, width, height, seed=0, noise=0.0, outliers=0.0, check_num_images=50, no_maps=(),
                  masks=False):
    scene = syn.planar_scene(np.random.default_rng(seed), n_views, width, height)
    rng = np.random.default_rng(seed + 1) if (noise or outliers) else None
    images = []
    for i, cam in enumerate(scene["cameras"]):
        grey = syn.render_planar(scene, i)[0]
        rgb = np.ascontiguousarray(np.stack([grey, 255 - grey, grey // 2], -1))
        d, n = syn.fusion_maps(scene, i, rng, noise, outliers)
        im = dict(rgb=rgb, color=rgb, overlap=[j for j in range(n_views) if j != i][:check_num_images],
                  depth=None if i in no_maps else d, normal=None if i in no_maps else n, mask=None)
        if masks and i not in no_maps:
            mk = np.ones((height, width), np.uint8)
            mk[: height // 4, : width // 3] = 0
            im["mask"] = mk
        im.update(mvs.fusion_camera(cam["K"], cam["R"], cam["t"], (width, height), (width, height)))
        images.append(im)
    return scene, images


def surface_distance(scene, xyz):
    """Per point, the distance to the nearest plane of the scene (within its extent) relative to the point's depth
    from the first camera."""
    best = np.full(len(xyz), np.inf)
    for p in scene["planes"]:
        rel = xyz - p["c"]
        u, v = rel @ p["a1"], rel @ p["a2"]
        ok = (np.abs(u) <= p["half"] + 1e-3) & (np.abs(v) <= p["half"] + 1e-3)
        dist = np.where(ok, np.abs(rel @ p["n"]), np.inf)
        best = np.minimum(best, dist)
    cam = scene["cameras"][0]
    z = (xyz @ cam["R"].T + cam["t"])[:, 2]
    return best / np.abs(z)

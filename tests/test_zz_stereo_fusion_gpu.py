"""GPU: K9 (csrc/fusion.cu) against the scalar oracle (oracle/fusion.cpp) -- bit-exact points, normals, colours,
visibility, seeds and committed order against the oracle's `schedule`, the reported order replayed exactly, the
overflow path, determinism, counters and the end-to-end PatchMatch -> fusion accuracy on a rendered scene."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import pycolmap_b200 as pb  # noqa: E402
from oracle import fusion as F  # noqa: E402
from helpers.fusion_scenes import fusion_images, surface_distance  # noqa: E402


def _device(images, opts):
    r = pb._core._stereo_fusion_run(images, opts, 0)
    voff = r["vis_off"]
    r["visibility"] = [r["vis"][voff[k]:voff[k + 1]] for k in range(len(r["xyz"]))]
    return r


def _assert_equal(got, want):
    for k in ("xyz", "normals", "colors", "seeds", "order"):
        assert got[k].shape == want[k].shape, (k, got[k].shape, want[k].shape)
        assert np.array_equal(got[k], want[k]), k
    assert len(got["visibility"]) == len(want["visibility"])
    assert all(np.array_equal(a, b) for a, b in zip(got["visibility"], want["visibility"]))


VARIANTS = {
    "defaults": (dict(), dict()),
    "noisy_outliers": (dict(noise=0.003, outliers=0.05), dict()),
    "check_num_images_2": (dict(check_num_images=2), dict(check_num_images=2)),
    "traversal_depth_2": (dict(), dict(max_traversal_depth=2)),
    "max_num_pixels_3": (dict(), dict(max_num_pixels=3, min_num_pixels=2)),
    "bounding_box": (dict(), dict(bounding_box=([-1.5, -1.0, 0.0], [1.0, 1.0, 9.0]))),
    "masks": (dict(masks=True), dict()),
    "no_maps": (dict(no_maps=(1, 3)), dict()),
}


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_bit_exact_against_the_oracle_schedule(name):
    scene_kw, opt_kw = VARIANTS[name]
    _, images = fusion_images(5, 96, 72, seed=3, **scene_kw)
    opts = pb.StereoFusionOptions(opt_kw)
    got = _device(images, opts)
    want = F.run(images, opts, "schedule")
    _assert_equal(got, want)
    assert len(got["xyz"]) > 0 or name == "bounding_box"
    # the reported order is a serialisation: the sequential traversal over it gives the same cloud
    rep = F.run(images, opts, "replay", seeds=got["order"][:, :3])
    for k in ("xyz", "normals", "colors", "seeds"):
        assert np.array_equal(rep[k], got[k]), k


def test_overflow_path_is_exact():
    # large tolerances grow clusters past a candidate slot (512 pixels), so the one-thread overflow path runs
    _, images = fusion_images(6, 80, 60, seed=5)
    opts = pb.StereoFusionOptions(dict(max_reproj_error=12.0, max_depth_error=0.2, max_normal_error=60.0))
    before = pb._core._stereo_fusion_stats(0)
    got = _device(images, opts)
    after = pb._core._stereo_fusion_stats(0)
    want = F.run(images, opts, "schedule")
    _assert_equal(got, want)
    # traversals beyond one per candidate are the overflow path's redos
    live = after["fusion_seeds"] - before["fusion_seeds"] + after["fusion_deferred"] - before["fusion_deferred"]
    assert after["fusion_traversals"] - before["fusion_traversals"] > live


def test_deterministic_and_counters():
    _, images = fusion_images(5, 96, 72, seed=7, noise=0.002, outliers=0.02)
    opts = pb.StereoFusionOptions()
    s0 = pb._core._stereo_fusion_stats(0)
    a = _device(images, opts)
    s1 = pb._core._stereo_fusion_stats(0)
    b = _device(images, opts)
    _assert_equal(a, b)
    assert s1["fusion_points"] - s0["fusion_points"] == len(a["xyz"])
    assert s1["fusion_seeds"] - s0["fusion_seeds"] == len(a["order"])
    assert s1["fusion_rounds"] - s0["fusion_rounds"] == int(a["order"][-1, 3]) + 1
    assert s1["fusion_pops"] - s0["fusion_pops"] >= s1["fusion_traversals"] - s0["fusion_traversals"]
    # every valid pixel ends fused: replaying the order leaves no live pixel for a `rows` pass to seed
    want = F.run(images, opts, "schedule")
    assert want["stats"]["seeds"] == len(a["order"])


def test_jpeg_and_png_colour_sources(tmp_path):
    from PIL import Image
    _, images = fusion_images(4, 64, 48, seed=9)
    opts = pb.StereoFusionOptions()
    for k, im in enumerate(images):
        p = tmp_path / f"{k}.png"
        Image.fromarray(im["rgb"]).save(p)
        im["color"] = p.read_bytes()
    got = _device(images, opts)
    _assert_equal(got, F.run(images, opts, "schedule"))
    # JPEG: decoded by nvJPEG, so colours may differ from the host render; geometry and order do not
    for k, im in enumerate(images):
        p = tmp_path / f"{k}.jpg"
        Image.fromarray(im["rgb"]).save(p, quality=95)
        im["color"] = p.read_bytes()
    got_j = _device(images, opts)
    for k in ("xyz", "normals", "seeds", "order"):
        assert np.array_equal(got_j[k], got[k]), k
    assert np.abs(got_j["colors"].astype(int) - got["colors"].astype(int)).mean() < 8


def test_patch_match_then_fusion_end_to_end(tmp_path):
    from pycolmap_b200 import mvs, synthetic as syn
    ws = str(tmp_path / "ws")
    scene = syn.planar_scene(np.random.default_rng(11), 8, 640, 480)
    syn.write_dense_workspace(ws, scene, sources="__auto__, 5")
    pb.patch_match_stereo(ws)
    out = str(tmp_path / "fused.ply")
    r = pb.stereo_fusion(out, ws)
    xyz, nrm, col = mvs.read_ply(out)
    assert np.array_equal(xyz, r["xyz"]) and np.array_equal(col, r["colors"])
    vis = mvs.read_points_visibility(out + ".vis")
    assert all(np.array_equal(a, b) for a, b in zip(vis, r["visibility"]))
    d = surface_distance(scene, r["xyz"])
    frac = float(np.mean(d < 0.01))
    min_vis = min(len(v) for v in r["visibility"])
    print(f"end to end: {len(xyz)} points, {100 * frac:.1f} % within 1 % of depth, min visibility {min_vis}")
    assert len(xyz) > 10000
    assert frac >= 0.95
    assert min_vis >= 2

"""CPU: the scalar stereo fusion oracle (oracle/fusion.cpp) -- accuracy on exact maps, the schedule as a serialisation,
`rows` against `schedule`, and hand-built cases for each check of the traversal."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import pycolmap_b200 as pb
from oracle import fusion as F
from helpers.fusion_scenes import fusion_images, surface_distance


@pytest.fixture(scope="module")
def scene6():
    return fusion_images(6, 160, 120)


def test_points_lie_on_the_true_surface(scene6):
    scene, images = scene6
    r = F.run(images, pb.StereoFusionOptions(), "schedule")
    assert len(r["xyz"]) > 3000
    assert surface_distance(scene, r["xyz"]).max() < 2e-3  # median of exact points of one plane, fp32
    assert all(len(v) >= 2 for v in r["visibility"])
    assert np.allclose(np.linalg.norm(r["normals"], axis=1), 1.0, atol=1e-5)


def test_schedule_is_a_serialisation(scene6):
    _, images = scene6
    o = pb.StereoFusionOptions()
    r = F.run(images, o, "schedule")
    rep = F.run(images, o, "replay", seeds=r["order"][:, :3])
    for k in ("xyz", "normals", "colors", "seeds"):
        assert np.array_equal(rep[k], r[k]), k
    # every valid pixel ends fused: a `rows` pass after the replayed order finds no seed left
    tail = F.run(images, o, "replay", seeds=np.r_[r["order"][:, :3], [[i, y, x] for i in range(6) for y in range(120)
                                                                       for x in range(160)]])
    assert len(tail["order"]) == len(r["order"])
    assert np.all(np.diff(r["order"][:, 3]) >= 0) and r["stats"]["rounds"] == r["order"][-1, 3] + 1


def test_rows_against_schedule(scene6):
    # measured on this scene with s = 16: counts 95.5 %, 98.2 % / 99.6 % of points within 1 % of depth of the other cloud
    _, images = scene6
    o = pb.StereoFusionOptions()
    a = F.run(images, o, "rows")["xyz"]
    b = F.run(images, o, "schedule")["xyz"]
    assert abs(len(b) - len(a)) <= 0.05 * len(a)
    da = cKDTree(b).query(a)[0] / np.linalg.norm(a, axis=1)
    db = cKDTree(a).query(b)[0] / np.linalg.norm(b, axis=1)
    assert np.mean(da < 0.01) >= 0.95 and np.mean(db < 0.01) >= 0.95


def _plane_pair(W=12, H=10, shifts=(0.0, -0.05)):
    """Views of the plane z = 5 (focal 10) from x = -shift: every pixel of one view maps onto the others.  Red of
    view i at column c is 10 c + i, green is 10 x the row."""
    images = []
    from pycolmap_b200 import mvs
    n = len(shifts)
    for i, tx in enumerate(shifts):
        R = np.eye(3)
        t = np.array([tx, 0.0, 0.0])
        d = np.full((H, W), 5.0, np.float32)
        nm = np.zeros((H, W, 3), np.float32)
        nm[..., 2] = -1.0
        rgb = np.zeros((H, W, 3), np.uint8)
        rgb[..., 0] = np.arange(W, dtype=np.uint8)[None, :] * 10 + i
        rgb[..., 1] = np.arange(H, dtype=np.uint8)[:, None] * 10
        im = dict(depth=d, normal=nm, rgb=rgb, overlap=[j for j in range(n) if j != i], mask=None)
        im.update(mvs.fusion_camera((10.0, 10.0, W / 2, H / 2), R, t, (W, H), (W, H)))
        images.append(im)
    return images


def _opts(**kw):
    o = pb.StereoFusionOptions()
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def test_max_num_pixels_break_and_traversal_depth():
    images = _plane_pair()
    r = F.run(images, _opts(min_num_pixels=1, max_num_pixels=1), "rows")
    assert len(r["xyz"]) == 2 * 12 * 10  # each cluster stops after its seed
    r = F.run(images, _opts(min_num_pixels=1, max_traversal_depth=1), "rows")
    assert all(len(v) == 1 for v in r["visibility"])  # no child is pushed
    r = F.run(images, _opts(min_num_pixels=2), "rows")
    assert all(len(v) == 2 for v in r["visibility"]) and len(r["xyz"]) > 50


def test_even_and_odd_medians():
    # n identical views: every cluster holds the same pixel of each view, red values 10 c + (0 .. n - 1)
    for n, extra in ((2, 1), (3, 1), (4, 2)):  # even: round(mean of the middle two), half away from zero
        r = F.run(_plane_pair(shifts=(0.0,) * n), _opts(min_num_pixels=n), "rows")
        assert len(r["xyz"]) == 12 * 10
        assert np.array_equal(r["colors"][:, 0], 10 * r["seeds"][:, 2] + extra), n
        assert np.array_equal(r["colors"][:, 1], 10 * r["seeds"][:, 1])
        assert all(len(v) == n for v in r["visibility"])


def test_bounding_box_and_normal_below_epsilon():
    images = _plane_pair()
    r = F.run(images, _opts(min_num_pixels=1, bounding_box=([-10, -10, 6.0], [10, 10, 10])), "rows")
    assert len(r["xyz"]) == 0 and len(r["order"]) > 0  # pixels are fused (seeds committed) but never accumulated
    for im in images:
        im["normal"][:] = 0.0
    r = F.run(images, _opts(min_num_pixels=1), "rows")
    assert len(r["xyz"]) == 0 and len(r["order"]) > 0


def test_masks():
    images = _plane_pair()
    for im in images:
        im["mask"] = np.zeros((10, 12), np.uint8)
    r = F.run(images, _opts(min_num_pixels=1), "schedule")
    assert len(r["order"]) == 0
    images[0]["mask"][:, :6] = 1
    r = F.run(images, _opts(min_num_pixels=1), "schedule")
    assert set(r["order"][:, 0]) == {0} and r["order"][:, 2].max() < 6

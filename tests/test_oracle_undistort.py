"""CPU: oracle/undistort.py, the specification K10 is held to, on checks that need no recollection of upstream."""
import numpy as np
import pytest

from oracle import undistort as U

OPENCV = dict(model=4, width=80, height=60, params=[70.0, 72.0, 40.0, 30.0, -0.25, 0.06, 0.001, -0.002])


def test_pinhole_with_default_options_is_the_identity():
    cam = dict(model=1, width=40, height=30, params=[35.0, 36.0, 20.5, 14.5])
    assert U.undistort_camera({}, cam) == dict(model=1, width=40, height=30, params=[35.0, 36.0, 20.5, 14.5])
    img = np.random.default_rng(0).integers(0, 256, (30, 40, 3), dtype=np.uint8)
    out = U.warp(img, cam, U.undistort_camera({}, cam))
    # exact at every pixel whose bilinear footprint is inside; the bottom-up boundary rule blacks out row 0 and column W-1
    assert np.array_equal(out[1:, :-1], img[1:, :-1])
    assert not out[0].any() and not out[:, -1].any()


def test_barrel_distortion_without_blank_pixels_has_no_black_pixel():
    img = np.full((60, 80), 200, np.uint8)
    out, und = U.undistort_image(dict(blank_pixels=0.0), img, OPENCV)
    assert out.shape == (und["height"], und["width"], 3)
    assert out[1:-1, 1:-1].min() > 0


def test_all_border_samples_land_inside_with_blank_pixels_one():
    und = U.undistort_camera(dict(blank_pixels=1.0), OPENCV)
    ys = np.arange(60) + 0.5
    xs = np.arange(80) + 0.5
    border = np.r_[np.c_[np.full(60, 0.5), ys], np.c_[np.full(60, 79.5), ys], np.c_[xs, np.full(80, 0.5)],
                   np.c_[xs, np.full(80, 59.5)]]
    p = U.undistort_points(OPENCV, und, border)
    # the scale maps the near border to 0 and the far one to size - 0.5; the size is then truncated to whole pixels
    # (and cx scaled with it), which can cost the far border up to one pixel
    assert p[:, 0].min() >= -1e-6 and p[:, 0].max() <= und["width"] + 0.5
    assert p[:, 1].min() >= -1e-6 and p[:, 1].max() <= und["height"] + 0.5


def test_min_and_max_scale_clamp():
    strong = dict(OPENCV, params=[70.0, 72.0, 40.0, 30.0, -0.6, 0.2, 0.0, 0.0])
    free = U.undistort_camera(dict(blank_pixels=1.0, max_scale=10.0), strong)
    assert free["width"] > 80 * 1.1
    capped = U.undistort_camera(dict(blank_pixels=1.0, max_scale=1.1), strong)
    assert capped["width"] == int(1.1 * 80) and capped["height"] == int(1.1 * 60)
    low = U.undistort_camera(dict(min_scale=1.5, max_scale=2.0), OPENCV)
    assert low["width"] == 120 and low["height"] == 90


def test_roi_origin_shifts_the_principal_point():
    cam = dict(model=1, width=100, height=80, params=[90.0, 90.0, 50.0, 40.0])
    und = U.undistort_camera(dict(roi_min_x=0.2, roi_min_y=0.25, roi_max_x=0.8, roi_max_y=1.0, min_scale=1.0,
                                  max_scale=1.0), cam)
    assert (und["width"], und["height"]) == (60, 60)
    assert und["params"][2] == pytest.approx(50.0 - 20.0) and und["params"][3] == pytest.approx(40.0 - 20.0)


def test_max_image_size_rescale_rounds_like_camera_rescale():
    cam = dict(model=1, width=101, height=77, params=[90.0, 91.0, 50.5, 38.5])
    und = U.undistort_camera(dict(max_image_size=50), cam)
    s = min(50 / 101, 50 / 77)
    assert (und["width"], und["height"]) == (round(s * 101), round(s * 77)) == (50, 38)
    sx, sy = 50 / 101, 38 / 77
    assert und["params"] == pytest.approx([90.0 * sx, 91.0 * sy, 50.5 * sx, 38.5 * sy], rel=1e-15)


def test_bilinear_boundary_rule_on_3x3_images():
    img = np.arange(27, dtype=np.uint8).reshape(3, 3, 3) * 9
    x = np.array([0.0, 1.0, 1.5, 1.999, 2.0, -0.001, 1.0, 1.0, 1.0])
    y = np.array([1.0, 1.0, 1.5, 1.0, 1.0, 1.0, 0.0, 0.001, 2.0])
    out = U.interpolate_bilinear(img, x, y)
    inside = out.any(1)
    # x in [0, W - 1) and y in (0, H - 1]: not symmetric, FreeImage's rows run bottom-up
    assert list(inside) == [True, True, True, True, False, False, False, True, True]
    assert np.array_equal(out[0], img[1, 0]) and np.array_equal(out[8], img[2, 1])
    assert np.array_equal(out[2], np.floor((img[1, 1].astype(float) + img[1, 2] + img[2, 1] + img[2, 2]) / 4 + 0.5))


def test_option_checks():
    for bad in (dict(blank_pixels=-0.1), dict(blank_pixels=1.1), dict(min_scale=0.0), dict(min_scale=3.0),
                dict(max_image_size=0), dict(roi_min_x=-0.1), dict(roi_max_y=1.1), dict(roi_min_x=0.5, roi_max_x=0.5)):
        with pytest.raises(ValueError):
            U.undistort_camera(bad, OPENCV)

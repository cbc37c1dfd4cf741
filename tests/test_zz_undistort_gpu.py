"""GPU: K10 (csrc/undistort.cu) against oracle/undistort.py -- cameras, pixels, JPEG output, 2-D points -- a truth
check against a pinhole render, undistort_images -> patch_match_stereo -> stereo_fusion end to end, repeatability."""
import copy
import io
import os

import numpy as np
import pytest

import pycolmap_b200 as pb
from oracle import undistort as U
from pycolmap_b200 import mvs, synthetic as syn

pytestmark = pytest.mark.gpu

W, H = 97, 71
CAMS = {
    0: [80.0, 48.0, 35.0], 1: [80.0, 82.0, 48.5, 35.5], 2: [80.0, 48.0, 35.0, -0.12],
    3: [80.0, 48.0, 35.0, -0.1, 0.02], 4: [80.0, 82.0, 48.5, 35.5, -0.2, 0.05, 0.002, -0.001],
    5: [80.0, 82.0, 48.5, 35.5, 0.05, -0.01, 0.002, -0.001],
    6: [80.0, 82.0, 48.5, 35.5, -0.2, 0.05, 0.002, -0.001, 0.01, 0.02, -0.01, 0.005], 7: [80.0, 82.0, 48.5, 35.5, 0.6],
    8: [80.0, 48.0, 35.0, 0.05], 9: [80.0, 48.0, 35.0, 0.05, -0.01],
    10: [80.0, 82.0, 48.5, 35.5, 0.05, -0.01, 0.001, 0.001, 0.002, 0.001, 0.001, -0.001]}
POLY = (0, 1, 2, 3, 4, 6)
OPTS = [dict(), dict(blank_pixels=0.5), dict(blank_pixels=1.0),
        dict(roi_min_x=0.1, roi_min_y=0.2, roi_max_x=0.85, roi_max_y=0.9), dict(max_image_size=60)]


def _cam(model, w=W, h=H):
    return dict(model=model, width=w, height=h, params=CAMS[model])


def _png(img):
    return pb._core._encode_png(img)


@pytest.mark.parametrize("model", sorted(CAMS))
def test_cameras_match_the_oracle(model):
    for o in OPTS:
        got = pb._core._undistort_camera(pb.UndistortCameraOptions(o), _cam(model))
        want = U.undistort_camera(o, _cam(model))
        assert (got["width"], got["height"]) == (want["width"], want["height"]), (model, o)
        assert np.allclose(got["params"], want["params"], rtol=1e-12, atol=0), (model, o)


def test_pixels_match_the_oracle():
    rng = np.random.default_rng(0)
    base = syn.textured_plane(rng, 128)[:H, :W]
    grey = np.clip(np.round(255 * base), 0, 255).astype(np.uint8)
    rgb = np.stack([grey, np.roll(grey, 7, 1), 255 - grey], -1)
    rgba = np.concatenate([rgb, np.full((H, W, 1), 9, np.uint8)], -1)
    report = []
    for model in sorted(CAMS):
        for o, img in ((OPTS[0], rgb), (OPTS[2], grey), (OPTS[3], rgba), (OPTS[4], rgb)):
            cam = _cam(model)
            got = pb._core.debug_undistort_pixels(_png(img), cam, pb.UndistortCameraOptions(o))
            want, und = U.undistort_image(o, img, cam)
            assert got.shape == want.shape, (model, o)
            d = np.abs(got.astype(int) - want.astype(int))
            if model in POLY:
                assert np.array_equal(got, want), (model, o, int(d.max()), int((d > 0).sum()))
            else:  # CUDA's and numpy's atan / tan differ by ulps
                share = (d > 0).mean()
                report.append((model, share))
                assert d.max() <= 1 and share <= 0.01, (model, o, int(d.max()), share)
    print("atan/tan models, share of differing samples:", max((s for _, s in report), default=0.0))


def test_png_and_jpeg_outputs():
    from PIL import Image
    rng = np.random.default_rng(1)
    img = np.clip(np.round(255 * syn.textured_plane(rng, 256)[:240, :200]), 0, 255).astype(np.uint8)
    img = np.stack([img, np.roll(img, 5, 0), img[::-1]], -1)
    cam = dict(model=4, width=200, height=240, params=[180.0, 180.0, 100.0, 120.0, -0.2, 0.04, 0.001, 0.001])
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, "JPEG", quality=95)
    jpg = buf.getvalue()
    res = pb._core._undistort_run([(_png(img), cam, "pixels"), (jpg, cam, "jpeg"), (b"not an image", cam, "jpeg"),
                                   (_png(img[:100]), cam, "pixels")], pb.UndistortCameraOptions(), 0)
    assert [r["status"] for r in res] == [0, 0, -1, -1] and "camera" in res[3]["error"]
    assert np.array_equal(res[0]["data"], pb._core.debug_undistort_pixels(_png(img), cam, pb.UndistortCameraOptions()))
    assert np.array_equal(pb._core.debug_decode_png(_png(res[0]["data"])), res[0]["data"])
    want = pb._core.debug_undistort_pixels(jpg, cam, pb.UndistortCameraOptions())
    dec = np.asarray(Image.open(io.BytesIO(res[1]["data"])).convert("RGB")).astype(int)
    d = np.abs(dec - want.astype(int))
    print(f"JPEG q100 4:2:0 output vs its pixels: max {d.max()}, mean {d.mean():.3f}")
    # measured on an H100 80GB HBM3: max 22, mean 2.24; held at one level more
    assert d.max() <= 23 and d.mean() < 3.24


def _scene(model_params, n=8, w=640, h=480, seed=2):
    cams = [dict(model=m, params=p) for m, p in model_params(n, w, h)]
    return syn.planar_scene(np.random.default_rng(seed), n, w, h, distorted=cams)


def _opencv(n, w, h):
    f = 0.9 * w
    return [(4, [f, f * 1.01, w / 2 + 3, h / 2 - 2, -0.18 + 0.01 * i, 0.03, 0.0008, -0.0006]) for i in range(n)]


def _fisheye(n, w, h):
    f = 0.9 * w
    return [(5, [f, f, w / 2, h / 2, 0.04, -0.01, 0.002, 0.0]) for _ in range(n)]


def _truth(scene, out, i):
    """The scene for rendering view i through the undistorted pinhole camera of out/sparse (cameras differ in size)."""
    m = mvs.read_sparse(os.path.join(out, "sparse"))
    s = copy.deepcopy(scene)
    s["width"], s["height"] = int(m.cameras[i + 1][1]), int(m.cameras[i + 1][2])
    for k, c in enumerate(s["cameras"]):
        c.pop("camera")
        c["K"] = tuple(m.cameras[k + 1][3])
    return s


def test_points_and_truth_render(tmp_path):
    scene = _scene(_opencv, n=3, w=320, h=240)
    syn.write_input_workspace(str(tmp_path / "in"), scene, points_per_view=200)
    pb.undistort_images(tmp_path / "out", tmp_path / "in" / "sparse", tmp_path / "in" / "images")
    src, out = mvs.read_sparse(str(tmp_path / "in" / "sparse")), mvs.read_sparse(str(tmp_path / "out" / "sparse"))
    for iid in src.images:
        truth = _truth(scene, str(tmp_path / "out"), iid - 1)
        cam = mvs._camera_dict(src.cameras[iid])
        und = mvs._camera_dict(out.cameras[iid])
        xy = src.image_raw[iid][2]
        got = out.image_raw[iid][2]
        want = U.undistort_points(cam, und, xy)
        fx, fy = und["params"][:2]
        assert np.abs((got - want) / [fx, fy]).max() < 1e-9
        # the true projection of each observed point through the undistorted camera
        c = scene["cameras"][iid - 1]
        X = np.array([src.points[p][0] for p in src.image_raw[iid][3]])
        y = X @ c["R"].T + c["t"]
        proj = y[:, :2] / y[:, 2:] * [fx, fy] + und["params"][2:]
        assert np.abs(got - proj).max() < 1e-4
        # the undistorted image against the pinhole render of the same view (interior, away from occlusion edges)
        img = pb._core.debug_decode_png(open(tmp_path / "out" / "images" / src.images[iid][0], "rb").read())
        ref = syn.render_planar(truth, iid - 1)[0].astype(int)
        g = (img[..., 0] if img.ndim == 3 else img).astype(int)
        hh, ww = ref.shape
        inner = np.abs(g - ref)[hh // 8:-hh // 8, ww // 8:-ww // 8]
        print(f"view {iid}: undistorted vs pinhole render, median |diff| {np.median(inner):.2f}, mean {inner.mean():.2f}")
        # measured on an H100 80GB HBM3: median 4 (two bilinear resamplings of a fine texture); held at one level more
        assert np.median(inner) <= 5


@pytest.mark.parametrize("kind", ["opencv", "fisheye"])
def test_end_to_end_undistort_patch_match_fusion(tmp_path, kind):
    scene = _scene(_opencv if kind == "opencv" else _fisheye)
    syn.write_input_workspace(str(tmp_path / "in"), scene, points_per_view=300)
    ws = tmp_path / "ws"
    pb.undistort_images(ws, tmp_path / "in" / "sparse", tmp_path / "in" / "images", num_patch_match_src_images=5)
    pb.patch_match_stereo(ws)
    truth = [_truth(scene, str(ws), i) for i in range(len(scene["cameras"]))]
    m = mvs.read_sparse(str(ws / "sparse"))
    ok = tot = 0
    for iid, (name, _, _, _) in m.images.items():
        d = mvs.read_array(mvs.map_paths(str(ws), name, "geometric")[0])
        t = syn.render_planar(truth[iid - 1], iid - 1)[1]
        keep = (d > 0) & (t > 0)
        ok += int((np.abs(d[keep] - t[keep]) < 0.01 * t[keep]).sum())
        tot += int(keep.sum())
    depth_share = ok / max(tot, 1)
    pts = pb.stereo_fusion(str(ws / "fused.ply"), ws)
    xyz = pts["xyz"].astype(np.float64)
    fused_share = _fused_share(truth, xyz, pts["visibility"])
    print(f"{kind}: {tot} kept depths, {100 * depth_share:.1f} % within 1 %; {len(xyz)} fused points, "
          f"{100 * fused_share:.1f} % within 1 % of the surface")
    assert depth_share >= 0.90 and fused_share >= 0.95


def _fused_share(truth, xyz, vis):
    depths = {}
    ok = 0
    for k in range(len(xyz)):
        i = int(vis[k][0])
        if i not in depths:
            depths[i] = syn.render_planar(truth[i], i, offset=0.0)[1]
        c = truth[i]["cameras"][i]
        y = c["R"] @ xyz[k] + c["t"]
        fx, fy, cx, cy = c["K"]
        u, v = int(round(fx * y[0] / y[2] + cx)), int(round(fy * y[1] / y[2] + cy))
        d = depths[i]
        if 0 <= v < d.shape[0] and 0 <= u < d.shape[1] and d[v, u] > 0 and abs(y[2] - d[v, u]) < 0.01 * d[v, u]:
            ok += 1
    return ok / max(len(xyz), 1)


def test_repeatable_and_counted(tmp_path):
    scene = _scene(_opencv, n=2, w=160, h=120)
    syn.write_input_workspace(str(tmp_path / "in"), scene, points_per_view=50, ext=".jpg")
    before = pb._core._undistort_stats(0)
    for out in ("a", "b"):
        pb.undistort_images(tmp_path / out, tmp_path / "in" / "sparse", tmp_path / "in" / "images")
    after = pb._core._undistort_stats(0)
    assert after["undistort_images"] - before["undistort_images"] == 4
    assert after["undistort_encoded_bytes"] > before["undistort_encoded_bytes"]
    for root, _, files in os.walk(tmp_path / "a"):
        for f in files:
            p = os.path.join(root, f)
            assert open(p, "rb").read() == open(p.replace(str(tmp_path / "a"), str(tmp_path / "b")), "rb").read(), p


@pytest.mark.parametrize("camera,options", [((2, [60.0, 40.0, 30.0, 0.0]), dict()),
                                            ((1, [60.0, 61.0, 40.0, 30.0]), dict(roi_min_x=0.1, roi_max_y=0.8))])
def test_written_images_have_their_cameras_size(tmp_path, camera, options):
    """A distortion-free SIMPLE_RADIAL camera and a PINHOLE camera under an ROI change size: such images are warped."""
    scene = syn.planar_scene(np.random.default_rng(4), 2, 80, 60, texture_size=64,
                             distorted=[dict(model=camera[0], params=camera[1])] * 2)
    syn.write_input_workspace(str(tmp_path / "in"), scene, points_per_view=20)
    pb.undistort_images(tmp_path / "out", tmp_path / "in" / "sparse", tmp_path / "in" / "images",
                        undistort_options=options)
    m = mvs.read_sparse(str(tmp_path / "out" / "sparse"))
    for name, cid, _, _ in m.images.values():
        img = pb._core.debug_decode_png(open(tmp_path / "out" / "images" / name, "rb").read())
        cam = m.cameras[cid]
        assert cam[0] == 1 and (img.shape[1], img.shape[0]) == (cam[1], cam[2]) != (80, 60)
        assert not os.path.islink(tmp_path / "out" / "images" / name)

"""GPU: extract_features from image files (K7, csrc/image_io.cu, in front of K6).  The database rows must equal what
Sift.extract computes on the grey image the reader feeds it: PNG decoded on the host, JPEG decoded by nvJPEG, images
above max_image_size downscaled bit-equal to oracle/image_io.py; keypoints in FeatureKeypoint's 6 columns, in
original-image coordinates, with the masks applied."""
import io
import os
import sqlite3

import numpy as np
import pytest
from PIL import Image

from helpers.native_import import load_native
from oracle import image_io as O
from pycolmap_b200 import synthetic as syn

nat = load_native()
pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "images")
JPEGS = ["baseline_420.jpg", "baseline_444.jpg", "progressive.jpg", "grey.jpg", "exif_focal.jpg"]


def _rows(db_path):
    """{name: (keypoints (N, 6), descriptors (N, 128) uint8, camera dict)}"""
    out = {}
    with nat.Database(db_path) as db:
        for iid, name, cid in db.read_all_images():
            out[name] = (np.asarray(db.read_keypoints(iid)), np.asarray(db.read_descriptors(iid)), db.read_camera(cid))
    return out


def _sift6(grey, W=None, H=None, **opts):
    """Sift.extract (the C++ option defaults) of `grey`, as 6-column keypoints mapped to a W x H original."""
    o = nat.SiftExtractionOptions(opts) if opts else nat.SiftExtractionOptions()
    kp, desc = nat.Sift(o).extract(grey)
    h, w = grey.shape
    sx = None if W is None or (W, H) == (w, h) else np.float32(W) / np.float32(w)
    sy = None if sx is None else np.float32(H) / np.float32(h)
    return O.keypoints6(kp, sx, sy), np.round(desc * 512).astype(np.uint8)


def _assert_rows_equal(got, want, what):
    kg, dg = got
    kw, dw = want
    assert kg.shape == kw.shape and kg.shape[1] == 6, (what, kg.shape, kw.shape)
    assert np.array_equal(dg, dw), what
    assert np.array_equal(kg[:, :2], kw[:, :2]), what
    err = np.abs(kg[:, 2:] - kw[:, 2:]).max() if len(kg) else 0.0
    scale = np.abs(kw[:, 2:]).max() if len(kw) else 1.0
    assert err <= 2.5e-7 * scale, (what, err)  # cos / sin of the device vs numpy: at most about one fp32 ulp


def _colour(rng, w, h):
    a, b, _ = syn.homography_pair(rng, w, h, 512)
    return np.stack([a, b, np.roll(a, 3, 0)], -1)


@pytest.mark.parametrize("w,h,mode", [(160, 120, "RGB"), (97, 61, "P"), (200, 150, "L"), (128, 96, "RGBA"),
                                      (321, 203, "LA")])
def test_png_rows_equal_sift_extract(tmp_path, w, h, mode):
    rgb = _colour(np.random.default_rng(w), w, h)
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    img = Image.fromarray(rgb)
    img = img.convert(mode) if mode != "P" else img.quantize(64)
    img.save(imgs / "view.png")
    ref = Image.open(imgs / "view.png")
    arr = np.asarray(ref.convert("RGB")) if mode in ("P", "RGB", "RGBA") else np.asarray(ref)
    grey = O.to_grey(arr[..., 0] if mode == "LA" else arr)
    dec = O.decode_png((imgs / "view.png").read_bytes())
    dec = dec[..., 0] if mode == "LA" else (dec[..., :3] if mode == "RGBA" else dec)
    assert np.array_equal(dec, arr[..., 0] if mode == "LA" else arr)
    assert np.array_equal(nat.debug_decode_grey((imgs / "view.png").read_bytes()), grey)
    nat.extract_features(tmp_path / "f.db", imgs)
    rows = _rows(tmp_path / "f.db")
    kp6, desc, cam = rows["view.png"]
    assert (cam["width"], cam["height"], cam["has_prior_focal_length"]) == (w, h, 0)
    _assert_rows_equal((kp6, desc), _sift6(grey), f"{mode} {w}x{h}")
    assert len(kp6) > 10


@pytest.mark.parametrize("w,h", [(400, 300), (401, 300), (300, 401), (520, 130)])
def test_downscale_is_freeimage_bilinear(tmp_path, w, h):
    rgb = _colour(np.random.default_rng(h), w, h)
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    Image.fromarray(rgb).save(imgs / "big.png")
    tw, th = O.target_size(w, h, 256)
    want = O.rescale(O.to_grey(rgb), tw, th)
    got = nat.debug_decode_grey((imgs / "big.png").read_bytes(), 256)
    assert got.shape == (th, tw) and np.array_equal(got, want)
    nat.extract_features(tmp_path / "f.db", imgs, sift_options={"max_image_size": 256})
    kp6, desc, cam = _rows(tmp_path / "f.db")["big.png"]
    assert (cam["width"], cam["height"]) == (w, h)
    _assert_rows_equal((kp6, desc), _sift6(want, w, h, max_image_size=256), f"{w}x{h} -> {tw}x{th}")


# Largest and mean |nvJPEG - libjpeg| in grey levels per fixture, as measured on an H100 (CUDA 12.9 nvJPEG) plus a
# margin of one level: the IDCT and, for subsampled chroma, the upsampling of the two decoders differ.  A wrong
# upsampling mode or colour conversion moves these by far more.
JPEG_DIFF = {"baseline_420.jpg": (8, 1.25), "baseline_444.jpg": (3, 0.6), "progressive.jpg": (8, 1.25),
             "grey.jpg": (2, 0.05), "exif_focal.jpg": (8, 1.25)}


def test_jpeg_decode_against_libjpeg_and_features(tmp_path):
    ref = np.load(os.path.join(GOLDEN, "pillow_grey.npz"))
    lines, bad = [], []
    for name in JPEGS:
        got = nat.debug_decode_grey(open(os.path.join(GOLDEN, name), "rb").read())
        want = ref[name]
        assert got.shape == want.shape
        d = np.abs(got.astype(np.int32) - want.astype(np.int32))
        lines.append(f"{name}: max {d.max()}, mean {d.mean():.4f}")
        if d.max() > JPEG_DIFF[name][0] or d.mean() > JPEG_DIFF[name][1]:
            bad.append(name)
    print("\nnvJPEG vs libjpeg (Pillow), grey levels: " + "; ".join(lines))
    assert not bad, lines
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    for name in JPEGS:
        (imgs / name).write_bytes(open(os.path.join(GOLDEN, name), "rb").read())
    nat.extract_features(tmp_path / "j.db", imgs)
    rows = _rows(tmp_path / "j.db")
    assert sorted(rows) == sorted(JPEGS)
    for name in JPEGS:
        grey = nat.debug_decode_grey((imgs / name).read_bytes())
        _assert_rows_equal(rows[name][:2], _sift6(grey), name)
    assert rows["exif_focal.jpg"][2]["has_prior_focal_length"] == 1
    assert rows["exif_focal.jpg"][2]["params"][0] == pytest.approx(4.2 / 30.0 * 160, rel=1e-15)


def test_masks(tmp_path):
    w, h = 200, 150
    rgb = _colour(np.random.default_rng(4), w, h)
    imgs, masks = tmp_path / "imgs", tmp_path / "masks"
    (imgs / "sub").mkdir(parents=True)
    (masks / "sub").mkdir(parents=True)
    Image.fromarray(rgb).save(imgs / "sub" / "a.png")
    m = np.full((h, w), 255, np.uint8)
    m[:, : w // 2] = 0
    Image.fromarray(m).save(masks / "sub" / "a.png.png")
    cm = np.full((h - 10, w), 7, np.uint8)  # camera mask: rows >= h - 10 lie outside it
    cm[: h // 3] = 0
    Image.fromarray(cm).save(tmp_path / "camera_mask.png")
    nat.extract_features(tmp_path / "m.db", imgs, reader_options={"mask_path": str(masks),
                                                                 "camera_mask_path": str(tmp_path / "camera_mask.png")})
    kp6, desc, _ = _rows(tmp_path / "m.db")["sub/a.png"]
    all6, alld = _sift6(O.to_grey(rgb))
    keep = O.mask_keep(all6, m) & O.mask_keep(all6, cm)
    assert 0 < keep.sum() < len(keep)
    _assert_rows_equal((kp6, desc), (all6[keep], alld[keep]), "masked")
    x, y = kp6[:, 0].astype(int), kp6[:, 1].astype(int)
    assert (m[y, x] != 0).all() and (y < h - 10).all() and (cm[y, x] != 0).all()


def _dump(path):
    con = sqlite3.connect(path)
    try:
        return "\n".join(con.iterdump())
    finally:
        con.close()


def test_determinism_and_batch_boundaries(tmp_path):
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    rng = np.random.default_rng(8)
    for k in range(37):  # more than one device call's worth of images
        a, _, _ = syn.homography_pair(rng, 96 + k, 80, 256)
        buf = io.BytesIO()
        Image.fromarray(a).save(buf, "JPEG", quality=90) if k % 2 else Image.fromarray(a).save(buf, "PNG")
        (imgs / f"{k:03d}.{'jpg' if k % 2 else 'png'}").write_bytes(buf.getvalue())
    nat.extract_features(tmp_path / "a.db", imgs)
    nat.extract_features(tmp_path / "b.db", imgs)
    assert _dump(tmp_path / "a.db") == _dump(tmp_path / "b.db")
    rows = _rows(tmp_path / "a.db")
    assert len(rows) == 37
    for k in (0, 31, 32, 36):
        name = f"{k:03d}.{'jpg' if k % 2 else 'png'}"
        nat.extract_features(tmp_path / f"one{k}.db", imgs, image_list=[name])
        one = _rows(tmp_path / f"one{k}.db")[name]
        assert np.array_equal(one[0], rows[name][0]) and np.array_equal(one[1], rows[name][1]), name


def test_undecodable_jpeg_body_is_skipped_with_a_warning(tmp_path, capfd):
    """A JPEG whose frame header reads but whose body is cut off before the scan: the host reader accepts it, the
    device decoder refuses it, and extract_features skips it with a warning, in the middle of a call."""
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    good = open(os.path.join(GOLDEN, "baseline_444.jpg"), "rb").read()
    (imgs / "a.jpg").write_bytes(good)
    (imgs / "b_cut.jpg").write_bytes(good[:good.index(b"\xff\xda")])  # everything from the start of scan on is gone
    (imgs / "c.jpg").write_bytes(good)
    assert nat.infer_camera_from_image(imgs / "b_cut.jpg")["width"] == 160
    nat.extract_features(tmp_path / "cut.db", imgs)
    rows = _rows(tmp_path / "cut.db")
    assert sorted(rows) == ["a.jpg", "c.jpg"]
    assert np.array_equal(rows["a.jpg"][1], rows["c.jpg"][1]) and len(rows["a.jpg"][1]) > 10
    err = capfd.readouterr().err
    assert "b_cut.jpg: nvJPEG cannot decode it" in err or "b_cut.jpg: not a JPEG stream nvJPEG can read" in err, err


def test_decode_counters():
    ctx = nat.Context(device=0)
    try:
        files = [open(os.path.join(GOLDEN, n), "rb").read() for n in ("baseline_420.jpg", "progressive.jpg")]
        png = io.BytesIO()
        Image.fromarray(np.zeros((20, 30), np.uint8)).save(png, "PNG")
        for f in files + [png.getvalue()]:
            ctx.debug_decode_grey(f)
        st = ctx.stats()
        # debug_decode_grey decodes twice: once for the size, once into the array
        assert st["sift_decode_images"] == 6 and st["sift_decoded_bytes"] == 2 * sum(len(f) for f in files)
        # the hardware backend takes baseline files only, where the GPU has JPEG engines
        assert st["sift_decode_hardware"] in (0, 2), st
        print(f"\nJPEG files through the hardware backend: {st['sift_decode_hardware'] // 2} of 2 (baseline, progressive)")
    finally:
        ctx.close()


def test_end_to_end_homography_from_jpeg_files(tmp_path):
    """The committed rendered pair (tests/golden/make_image_fixtures.py) through extract_features and match_exhaustive
    gives back the planted homography."""
    w, h = 1024, 768
    H = np.load(os.path.join(GOLDEN, "homography_H.npy"))
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    for k in range(2):
        (imgs / f"view{k}.jpg").write_bytes(open(os.path.join(GOLDEN, f"homography_view{k}.jpg"), "rb").read())
    path = tmp_path / "pair.db"
    nat.extract_features(path, imgs)
    nat.match_exhaustive(path)
    with nat.Database(path) as db:
        (i0, _, _), (i1, _, _) = db.read_all_images()
        g = db.read_two_view_geometry(i0, i1)
        k0, k1 = np.asarray(db.read_keypoints(i0)), np.asarray(db.read_keypoints(i1))
    inl = np.asarray(g.inlier_matches)
    print(f"\nend to end from JPEG files: {len(k0)} / {len(k1)} features, config {g.config}, {len(inl)} inliers")
    assert int(g.config) == 6 and len(inl) >= 300  # PLANAR_OR_PANORAMIC
    p1, p2 = k0[inl[:, 0], :2].astype(np.float64), k1[inl[:, 1], :2].astype(np.float64)
    r = nat.homography_matrix_estimation(p1, p2, nat.RANSACOptions(max_error=2.0))
    c = np.array([[0, 0, 1], [w, 0, 1], [w, h, 1], [0, h, 1]], np.float64)
    pa, pb = c @ r["H"].T, c @ H.T
    err = np.linalg.norm(pa[:, :2] / pa[:, 2:] - pb[:, :2] / pb[:, 2:], axis=1).max()
    print(f"corner error {err:.3f} px")
    assert err < 1.0

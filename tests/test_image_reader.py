"""CPU: the image reader behind extract_features / import_images / infer_camera_from_image (options, argument checks,
file walk, camera assignment per CameraMode, EXIF focal length, PNG variants) and the oracle of oracle/image_io.py."""
import io
import os
import pickle
import struct
import zlib

import numpy as np
import pytest
from PIL import Image
from PIL.TiffImagePlugin import IFDRational

from oracle import image_io as O
from helpers.native_import import load_native

nat = load_native()
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "images")


def _jpeg(path, w, h, exif=None, seed=0):
    rgb = np.random.default_rng(seed).integers(0, 255, (h, w, 3), dtype=np.uint8)
    kw = {"exif": exif} if exif is not None else {}
    Image.fromarray(rgb).save(path, "JPEG", quality=90, **kw)


def _png(path, arr, **kw):
    Image.fromarray(arr).save(path, "PNG", **kw)


def _tree(root, files):
    for name, (w, h) in files.items():
        p = root / name
        p.parent.mkdir(parents=True, exist_ok=True)
        _jpeg(p, w, h)


def _db(tmp_path):
    p = tmp_path / "db.db"
    nat.Database(p).close()
    return p


def _read(path):
    with nat.Database(path) as db:
        return db.read_all_images(), {c["camera_id"]: c for c in db.read_all_cameras()}


def test_options_and_camera_mode():
    o = nat.ImageReaderOptions()
    assert (o.camera_model, o.mask_path, o.existing_camera_id, o.camera_params, o.default_focal_length_factor,
            o.camera_mask_path) == ("SIMPLE_RADIAL", "", -1, "", 1.2, "")
    o.mergedict({"camera_model": "PINHOLE", "default_focal_length_factor": 2.0})
    assert o.todict()["camera_model"] == "PINHOLE" and pickle.loads(pickle.dumps(o)).default_focal_length_factor == 2.0
    assert "camera_mask_path" in o.summary()
    assert nat.CameraMode("PER_FOLDER") == nat.CameraMode.PER_FOLDER
    assert [int(m) for m in (nat.CameraMode.AUTO, nat.CameraMode.SINGLE, nat.CameraMode.PER_FOLDER,
                             nat.CameraMode.PER_IMAGE)] == [0, 1, 2, 3]
    with pytest.raises(IndexError):
        nat.CameraMode("EVERY")


def test_extract_features_argument_checks_in_upstream_order(tmp_path):
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    existing = _db(tmp_path)
    with pytest.raises(ValueError, match="already exists"):
        nat.extract_features(existing, imgs)
    with pytest.raises(ValueError, match="does not match file extension .db"):
        nat.extract_features(tmp_path / "x.sqlite", imgs)
    with pytest.raises(ValueError, match="Could not open .* Is the path a directory"):
        nat.extract_features(tmp_path / "missing" / "x.db", imgs)
    with pytest.raises(ValueError, match="Directory .* does not exist"):
        nat.extract_features(tmp_path / "a.db", tmp_path / "nope")
    with pytest.raises(ValueError, match="no CPU path"):
        nat.extract_features(tmp_path / "b.db", imgs, device=nat.Device.cpu)
    with pytest.raises(ValueError, match="ExistsCameraModelWithName"):
        nat.extract_features(tmp_path / "c.db", imgs, camera_model="PINHOLE_X")
    with pytest.raises(ValueError, match="Invalid camera parameters"):
        nat.extract_features(tmp_path / "d.db", imgs, reader_options={"camera_params": "1,2"})
    with pytest.raises(ValueError, match="domain_size_pooling"):
        nat.extract_features(tmp_path / "e.db", imgs, sift_options={"domain_size_pooling": True})
    with pytest.raises(ValueError, match="gpu_index"):
        nat.extract_features(tmp_path / "f.db", imgs, sift_options={"gpu_index": "0,1"})


def test_import_images_checks(tmp_path):
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    with pytest.raises(ValueError, match="File .* does not exist"):
        nat.import_images(tmp_path / "none.db", imgs)
    db = _db(tmp_path)
    with pytest.raises(ValueError, match="Directory .* does not exist"):
        nat.import_images(db, tmp_path / "none")
    with pytest.raises(ValueError, match="Invalid camera model: NOPE"):
        nat.import_images(db, imgs, options={"camera_model": "NOPE"})
    with pytest.raises(ValueError, match="does not exist"):
        nat.infer_camera_from_image(tmp_path / "none.jpg")
    (tmp_path / "t.txt").write_text("x")
    with pytest.raises(ValueError, match="Cannot read image file"):
        nat.infer_camera_from_image(tmp_path / "t.txt")


def test_walk_order_names_and_image_list(tmp_path):
    imgs = tmp_path / "imgs"
    _tree(imgs, {"b.jpg": (32, 24), "a/z.jpg": (32, 24), "a.jpg": (32, 24), "a/b/c.jpg": (32, 24), "B.jpg": (32, 24)})
    db = _db(tmp_path)
    nat.import_images(db, imgs)
    names = [n for _, n, _ in _read(db)[0]]
    assert names == sorted(["b.jpg", "a/z.jpg", "a.jpg", "a/b/c.jpg", "B.jpg"])
    assert names == ["B.jpg", "a.jpg", "a/b/c.jpg", "a/z.jpg", "b.jpg"]
    db2 = tmp_path / "db2.db"
    nat.Database(db2).close()
    nat.import_images(db2, imgs, image_list=["b.jpg", "a/z.jpg"])
    assert [n for _, n, _ in _read(db2)[0]] == ["b.jpg", "a/z.jpg"]
    # images already in the database are skipped
    nat.import_images(db2, imgs, image_list=["a/z.jpg", "a.jpg"])
    assert [n for _, n, _ in _read(db2)[0]] == ["b.jpg", "a/z.jpg", "a.jpg"]


def test_camera_modes(tmp_path, capfd):
    imgs = tmp_path / "imgs"
    _tree(imgs, {"f1/a.jpg": (40, 30), "f1/b.jpg": (40, 30), "f1/c.jpg": (48, 30), "f2/d.jpg": (40, 30),
                 "f2/e.jpg": (40, 30)})

    runs = []

    def run(mode, **opts):
        runs.append(mode)
        db = tmp_path / f"run{len(runs)}.db"
        nat.Database(db).close()
        nat.import_images(db, imgs, camera_mode=mode, options=opts)
        images, cams = _read(db)
        return [(n, c) for _, n, c in images], cams

    for mode in (nat.CameraMode.AUTO, nat.CameraMode.PER_IMAGE):
        images, cams = run(mode)
        assert [c for _, c in images] == [1, 2, 3, 4, 5] and len(cams) == 5
        assert cams[3]["width"] == 48 and cams[3]["params"] == [1.2 * 48, 24.0, 15.0, 0.0]
        assert cams[3]["has_prior_focal_length"] == 0
    images, cams = run(nat.CameraMode.SINGLE)
    assert images == [("f1/a.jpg", 1), ("f1/b.jpg", 1), ("f2/d.jpg", 1), ("f2/e.jpg", 1)] and len(cams) == 1
    assert "f1/c.jpg" in capfd.readouterr().err
    images, cams = run(nat.CameraMode.PER_FOLDER)
    assert images == [("f1/a.jpg", 1), ("f1/b.jpg", 1), ("f2/d.jpg", 2), ("f2/e.jpg", 2)] and len(cams) == 2
    images, cams = run(nat.CameraMode.AUTO, camera_params="100, 20, 15, 0.1")
    assert all(c["params"] == [100.0, 20.0, 15.0, 0.1] and c["has_prior_focal_length"] == 1 for c in cams.values())
    images, cams = run(nat.CameraMode.AUTO, camera_model="PINHOLE")
    assert cams[1]["model"] == 1 and cams[1]["params"] == [48.0, 48.0, 20.0, 15.0]
    # existing_camera_id: every image of that size uses the camera, the others are skipped
    db = tmp_path / "existing.db"
    with nat.Database(db) as d:
        d.add_camera(0, 40, 30, [50.0, 20.0, 15.0], True)
    nat.import_images(db, imgs, options={"existing_camera_id": 1})
    images, cams = _read(db)
    assert [(n, c) for _, n, c in images] == [("f1/a.jpg", 1), ("f1/b.jpg", 1), ("f2/d.jpg", 1), ("f2/e.jpg", 1)]
    assert len(cams) == 1


def test_unsupported_files_are_skipped_with_a_warning(tmp_path, capfd):
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    _jpeg(imgs / "ok.jpg", 32, 24)
    (imgs / "notes.txt").write_text("not an image")
    _png(imgs / "deep.png", np.arange(32 * 24, dtype=np.uint16).reshape(24, 32))
    _png(imgs / "interlaced.png", np.zeros((24, 32, 3), np.uint8))
    raw = bytearray(open(imgs / "interlaced.png", "rb").read())
    raw[28] = 1  # IHDR interlace method (the CRC check comes with the decode, not the header)
    (imgs / "interlaced.png").write_bytes(bytes(raw))
    (imgs / "ok_named.bmp").write_bytes((imgs / "ok.jpg").read_bytes())  # format from the magic bytes
    db = _db(tmp_path)
    nat.import_images(db, imgs)
    err = capfd.readouterr().err
    assert [n for _, n, _ in _read(db)[0]] == ["ok.jpg", "ok_named.bmp"]
    for name in ("notes.txt", "deep.png", "interlaced.png"):
        assert f"{name}:" in err and "skipped" in err


def _exif(**tags):
    e = Image.Exif()
    ifd = e.get_ifd(0x8769)
    for k, v in tags.items():
        ifd[{"f35": 0xA405, "focal": 0x920A, "pxdim": 0xA002, "xres": 0xA20E, "unit": 0xA210}[k]] = (
            IFDRational(*v) if isinstance(v, tuple) else v)
    return e.tobytes()


@pytest.mark.parametrize("tags", [
    dict(f35=28),
    dict(f35=0, focal=(415, 100), pxdim=160, xres=(160, 3), unit=3),
    dict(focal=(415, 100), pxdim=160, xres=(160, 3), unit=3),
    dict(focal=(50, 1), pxdim=4000, xres=(4000, 3), unit=2),
    dict(focal=(50, 1), pxdim=4000, xres=(4000, 1), unit=2),     # an integer resolution does not parse upstream
    dict(focal=(50, 1), pxdim=4000, xres=(4000, 3), unit=4),     # millimetres: not a unit upstream reads
    dict(focal=(50, 1)),
    dict(),
])
def test_exif_focal_length(tmp_path, tags):
    p = tmp_path / "e.jpg"
    _jpeg(p, 160, 120, exif=_exif(**tags))
    cam = nat.infer_camera_from_image(p)
    names = dict(f35="f35", focal="focal", pxdim="pixel_x_dim", xres="focal_plane_x_res", unit="unit")
    want = O.exif_focal(160, 120, **{names[k]: v for k, v in tags.items()})
    if want is None:
        assert cam["has_prior_focal_length"] == 0 and cam["params"][0] == 1.2 * 160
    else:
        assert cam["has_prior_focal_length"] == 1 and cam["params"][0] == want
    assert cam["width"] == 160 and cam["height"] == 120 and cam["params"][1:] == [80.0, 60.0, 0.0]


def test_exif_fixture():
    cam = nat.infer_camera_from_image(os.path.join(GOLDEN, "exif_focal.jpg"))
    assert cam["has_prior_focal_length"] == 1 and cam["params"][0] == pytest.approx(4.2 / 30.0 * 160, rel=1e-15)


def _png_bytes(arr, ctype, filters, palette=None):
    """A PNG with the given per-row filter types, written here so that every filter is exercised."""
    h = arr.shape[0]
    spp = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype]
    rows = arr.reshape(h, -1).astype(np.int32)
    raw = bytearray()
    prev = np.zeros(rows.shape[1], np.int32)
    for y in range(h):
        f = filters[y % len(filters)]
        cur = rows[y]
        a = np.r_[np.zeros(spp, np.int32), cur[:-spp]]
        c = np.r_[np.zeros(spp, np.int32), prev[:-spp]]
        b = prev
        if f == 0:
            p = np.zeros_like(cur)
        elif f == 1:
            p = a
        elif f == 2:
            p = b
        elif f == 3:
            p = (a + b) >> 1
        else:
            q = a + b - c
            pa, pb, pc = abs(q - a), abs(q - b), abs(q - c)
            p = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        raw.append(f)
        raw += ((cur - p) & 255).astype(np.uint8).tobytes()
        prev = cur

    def chunk(kind, body):
        return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))
    w = arr.shape[1]
    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, ctype, 0, 0, 0))
    if palette is not None:
        out += chunk(b"PLTE", palette.astype(np.uint8).tobytes())
    return out + chunk(b"IDAT", zlib.compress(bytes(raw))) + chunk(b"IEND", b"")


@pytest.mark.parametrize("ctype", [0, 2, 3, 4, 6])
def test_oracle_png_decoder_equals_pillow(ctype):
    rng = np.random.default_rng(ctype)
    h, w = 9, 13
    spp = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype]
    arr = rng.integers(0, 256 if ctype != 3 else 7, (h, w, spp), dtype=np.uint8)
    pal = rng.integers(0, 256, (7, 3)) if ctype == 3 else None
    data = _png_bytes(arr if spp > 1 else arr[..., 0], ctype, [0, 1, 2, 3, 4], pal)
    got = O.decode_png(data)
    ref = Image.open(io.BytesIO(data))
    want = np.asarray(ref.convert("RGB")) if ctype == 3 else np.asarray(ref)
    assert got.shape == want.shape and np.array_equal(got, want)


@pytest.mark.parametrize("ctype", [0, 2, 3, 4, 6])
def test_host_png_decoder_equals_pillow(ctype):
    """The decoder extract_features runs (host/image_reader.cc) on rows of every filter type, and the skips."""
    rng = np.random.default_rng(10 + ctype)
    h, w = 11, 17
    spp = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype]
    arr = rng.integers(0, 256 if ctype != 3 else 9, (h, w, spp), dtype=np.uint8)
    pal = rng.integers(0, 256, (9, 3)) if ctype == 3 else None
    data = _png_bytes(arr if spp > 1 else arr[..., 0], ctype, [4, 3, 2, 1, 0], pal)
    got = nat.debug_decode_png(data)
    ref = Image.open(io.BytesIO(data))
    want = {0: lambda: np.asarray(ref)[..., None], 2: lambda: np.asarray(ref), 3: lambda: np.asarray(ref.convert("RGB")),
            4: lambda: np.asarray(ref)[..., :1], 6: lambda: np.asarray(ref)}[ctype]()
    assert got.shape == want.shape and np.array_equal(got, want)
    bad = bytearray(data)
    bad[-20] ^= 0xFF  # inside the IDAT chunk: its CRC no longer matches
    with pytest.raises(ValueError, match="CRC"):
        nat.debug_decode_png(bytes(bad))


def test_host_png_decoder_refuses_a_size_its_data_cannot_hold():
    data = bytearray(_png_bytes(np.zeros((4, 4), np.uint8), 0, [0]))
    data[16:24] = struct.pack(">II", 1 << 24, 1 << 24)  # IHDR claims 2^48 pixels
    data[29:33] = struct.pack(">I", zlib.crc32(bytes(data[12:29])))
    with pytest.raises(ValueError, match="too short for its size"):
        nat.debug_decode_png(bytes(data))


def test_oracle_rescale_self_checks():
    rng = np.random.default_rng(3)
    g = rng.integers(0, 256, (37, 53), dtype=np.uint8)
    assert np.array_equal(O.rescale(g, 53, 37), g)  # equal size: the identity
    for v in (0, 1, 128, 255):
        for (w, h) in ((40, 28), (17, 30), (53, 5)):
            out = O.rescale(np.full((37, 53), v, np.uint8), w, h)
            assert out.shape == (h, w) and (out == v).all()
    assert O.target_size(4000, 3000, 3200) == (3200, 2400)
    assert O.target_size(3000, 4001, 3200) == (2399, 3200)
    assert O.target_size(100, 50, 3200) == (100, 50)


def test_oracle_grey_rule():
    px = np.array([[[255, 0, 0], [0, 255, 0], [0, 0, 255], [10, 20, 30], [255, 255, 255]]], np.uint8)
    assert O.to_grey(px).tolist() == [[54, 182, 18, 19, 255]]
    rgba = np.dstack([px, np.zeros((1, 5, 1), np.uint8)])
    assert np.array_equal(O.to_grey(rgba), O.to_grey(px))  # alpha is ignored


def test_oracle_keypoints_and_mask():
    kp = np.array([[10.5, 3.5, 2.0, 0.0], [1.5, 2.5, 1.0, np.pi / 2]], np.float32)
    k6 = O.keypoints6(kp)
    assert np.allclose(k6[0], [10.5, 3.5, 2, 0, 0, 2]) and np.allclose(k6[1], [1.5, 2.5, 0, -1, 1, 0], atol=1e-7)
    k6s = O.keypoints6(kp, 2.0, 3.0)
    assert np.allclose(k6s[0], [21, 10.5, 4, 0, 0, 6])
    mask = np.zeros((5, 12), np.uint8)
    mask[3, 10] = 1
    assert O.mask_keep(k6, mask).tolist() == [True, False]
    mask[0, 0] = 1  # GetPixel((int)x, (int)y): x in (-1, 0) reads column 0
    assert O.mask_keep(np.array([[-0.5, 0.25, 1, 0, 0, 1]], np.float32), mask).tolist() == [True]

"""CPU: undistort_images' options, argument checks and workspace layout on PINHOLE models (copied, never decoded, so
no device is needed), the sparse writer and the PNG encoder."""
import os
import shutil

import numpy as np
import pytest

import pycolmap_b200 as pb
from pycolmap_b200 import mvs, synthetic as syn


@pytest.fixture(scope="module")
def inp(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("undist_in"))
    syn.write_input_workspace(d, syn.planar_scene(np.random.default_rng(3), 4, 48, 36, texture_size=64),
                              points_per_view=40)
    return d


def test_options_defaults_and_checks():
    o = pb.UndistortCameraOptions()
    assert (o.blank_pixels, o.min_scale, o.max_scale, o.max_image_size) == (0.0, 0.2, 2.0, -1)
    assert (o.roi_min_x, o.roi_min_y, o.roi_max_x, o.roi_max_y) == (0.0, 0.0, 1.0, 1.0)
    for bad in (dict(blank_pixels=-0.5), dict(blank_pixels=2.0), dict(min_scale=0.0), dict(min_scale=3.0),
                dict(max_image_size=0), dict(roi_min_x=-1.0), dict(roi_min_y=-1.0), dict(roi_max_x=2.0),
                dict(roi_max_y=2.0), dict(roi_min_x=0.6, roi_max_x=0.4), dict(roi_min_y=0.6, roi_max_y=0.4)):
        with pytest.raises(ValueError, match="Check Failed"):
            pb._core._check_undistort_options(pb.UndistortCameraOptions(bad))
    assert pb.CopyType("soft-link") == getattr(pb.CopyType, "soft-link")
    with pytest.raises(ValueError):
        pb.CopyType("move")


def test_argument_order_and_errors(inp, tmp_path):
    with pytest.raises(ValueError, match="input_path"):
        pb.undistort_images(tmp_path / "o", tmp_path / "missing", os.path.join(inp, "images"))
    with pytest.raises(ValueError, match="image_path"):
        pb.undistort_images(tmp_path / "o", os.path.join(inp, "sparse"), tmp_path / "missing")
    for t in ("PMVS", "CMP-MVS"):
        with pytest.raises(ValueError, match="not supported"):
            pb.undistort_images(tmp_path / "o", os.path.join(inp, "sparse"), os.path.join(inp, "images"), output_type=t)
    with pytest.raises(ValueError, match="output_type"):
        pb.undistort_images(tmp_path / "o", os.path.join(inp, "sparse"), os.path.join(inp, "images"), output_type="X")
    with pytest.raises(ValueError, match="max_scale"):
        pb.undistort_images(tmp_path / "o", os.path.join(inp, "sparse"), os.path.join(inp, "images"),
                            undistort_options=dict(min_scale=3.0))


def _write_txt(src, dst):
    m = mvs.read_sparse(src)
    os.makedirs(dst)
    with open(os.path.join(dst, "cameras.txt"), "w") as f:
        for cid, (mid, w, h, p) in m.cameras.items():
            f.write(f"{cid} {mvs._MODEL_NAMES[mid]} {w} {h} " + " ".join(repr(float(v)) for v in p) + "\n")
    with open(os.path.join(dst, "images.txt"), "w") as f:
        for iid, (name, cid, _, _) in m.images.items():
            q, t, xy, ids = m.image_raw[iid]
            f.write(f"{iid} " + " ".join(repr(float(v)) for v in list(q) + list(t)) + f" {cid} {name}\n")
            f.write(" ".join(f"{x!r} {y!r} {k}" for (x, y), k in zip(xy.tolist(), ids.tolist())) + "\n")
    with open(os.path.join(dst, "points3D.txt"), "w") as f:
        for pid, (xyz, _) in m.points.items():
            rgb, err, tr = m.point_raw[pid]
            f.write(f"{pid} " + " ".join(repr(float(v)) for v in xyz) + " " + " ".join(str(int(v)) for v in rgb) +
                    f" {float(err)!r} " + " ".join(str(int(v)) for v in tr.ravel()) + "\n")


def test_bin_and_txt_input_write_the_same_model_with_bit_identical_poses(inp, tmp_path):
    _write_txt(os.path.join(inp, "sparse"), str(tmp_path / "txt"))
    pb.undistort_images(tmp_path / "a", os.path.join(inp, "sparse"), os.path.join(inp, "images"))
    pb.undistort_images(tmp_path / "b", tmp_path / "txt", os.path.join(inp, "images"))
    for f in ("cameras.bin", "images.bin", "points3D.bin"):
        a = open(tmp_path / "a" / "sparse" / f, "rb").read()
        assert a == open(tmp_path / "b" / "sparse" / f, "rb").read(), f
        assert a == open(os.path.join(inp, "sparse", f), "rb").read(), f  # PINHOLE: the model is written unchanged
    src, out = mvs.read_sparse(os.path.join(inp, "sparse")), mvs.read_sparse(str(tmp_path / "a" / "sparse"))
    for iid in src.images:
        assert src.image_raw[iid][0].tobytes() == out.image_raw[iid][0].tobytes()
        assert src.image_raw[iid][1].tobytes() == out.image_raw[iid][1].tobytes()
    for pid in src.points:
        assert np.array_equal(src.point_raw[pid][2], out.point_raw[pid][2])


def test_configs_and_image_list(inp, tmp_path):
    pb.undistort_images(tmp_path / "a", os.path.join(inp, "sparse"), os.path.join(inp, "images"),
                        num_patch_match_src_images=7)
    names = [f"view_{i:03d}.png" for i in range(4)]
    assert open(tmp_path / "a" / "stereo" / "patch-match.cfg").read() == "".join(f"{n}\n__auto__, 7\n" for n in names)
    assert open(tmp_path / "a" / "stereo" / "fusion.cfg").read() == "".join(f"{n}\n" for n in names)
    for d in ("depth_maps", "normal_maps", "consistency_graphs"):
        assert os.path.isdir(tmp_path / "a" / "stereo" / d)
    pb.undistort_images(tmp_path / "b", os.path.join(inp, "sparse"), os.path.join(inp, "images"),
                        image_list=[names[2], "nope.png", names[0]], num_patch_match_src_images=0)
    assert open(tmp_path / "b" / "stereo" / "patch-match.cfg").read() == f"{names[2]}\n__all__\n{names[0]}\n__all__\n"
    assert sorted(os.listdir(tmp_path / "b" / "images")) == [names[0], names[2]]


def test_copy_policies_and_subdirectories(inp, tmp_path):
    m = mvs.read_sparse(os.path.join(inp, "sparse"))
    imgs = tmp_path / "imgs"
    for iid, (name, cid, R, t) in list(m.images.items()):
        new = f"sub/dir/{name}"
        os.makedirs(imgs / "sub" / "dir", exist_ok=True)
        shutil.copyfile(os.path.join(inp, "images", name), imgs / new)
        m.images[iid] = (new, cid, R, t)
    mvs.write_sparse_bin(str(tmp_path / "sparse"), m)
    for policy, check in (("copy", lambda s, d: not os.path.islink(d) and os.stat(s).st_ino != os.stat(d).st_ino),
                          ("soft-link", lambda s, d: os.path.islink(d)),
                          ("hard-link", lambda s, d: os.stat(s).st_ino == os.stat(d).st_ino)):
        out = tmp_path / policy
        pb.undistort_images(out, tmp_path / "sparse", imgs, copy_policy=policy)
        for name, _, _, _ in m.images.values():
            s, d = str(imgs / name), str(out / "images" / name)
            assert open(s, "rb").read() == open(d, "rb").read() and check(s, d), (policy, name)
        assert "sub/dir/view_000.png" in open(out / "stereo" / "fusion.cfg").read()


def test_png_encoder_round_trips_through_the_decoder():
    rng = np.random.default_rng(0)
    for shape in ((7, 5), (9, 4, 3), (3, 11, 4)):
        a = rng.integers(0, 256, shape, dtype=np.uint8)
        assert np.array_equal(pb._core.debug_decode_png(pb._core._encode_png(a)).reshape(shape), a)

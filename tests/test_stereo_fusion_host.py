"""CPU: the host side of stereo_fusion -- options, argument checks and their order, overlap ranking, fusion.cfg, the
PLY / .vis / points3D.bin layouts, skipped images, and no CPU fallback.  The device call is replaced by the oracle
where a test needs a cloud (the oracle is what the device is held to bit for bit on the GPU)."""
import os
import struct

import numpy as np
import pytest

import pycolmap_b200 as pb
from pycolmap_b200 import mvs, synthetic as syn
from oracle import fusion as F


def test_option_defaults_and_checks():
    o = pb.StereoFusionOptions()
    assert (o.mask_path, o.num_threads, o.max_image_size, o.min_num_pixels, o.max_num_pixels) == ("", -1, -1, 5, 10000)
    assert (o.max_traversal_depth, o.max_reproj_error, o.max_depth_error, o.max_normal_error) == (100, 2.0, 0.01, 10.0)
    assert (o.check_num_images, o.use_cache, o.cache_size) == (50, False, 32.0)
    lo, hi = o.bounding_box
    assert lo == [-3.4028234663852886e38] * 3 and hi == [3.4028234663852886e38] * 3
    assert pb.StereoFusionOptions({"min_num_pixels": 3}).min_num_pixels == 3
    assert pb.StereoFusionOptions(max_traversal_depth=7).max_traversal_depth == 7
    for kw, msg in ((dict(min_num_pixels=-1), "min_num_pixels >= 0"), (dict(min_num_pixels=20, max_num_pixels=10),
                    "min_num_pixels <= max_num_pixels"), (dict(max_traversal_depth=0), "max_traversal_depth > 0"),
                    (dict(max_reproj_error=-1.0), "max_reproj_error >= 0"), (dict(max_depth_error=-1.0),
                    "max_depth_error >= 0"), (dict(max_normal_error=-1.0), "max_normal_error >= 0"),
                    (dict(check_num_images=0), "check_num_images > 0"), (dict(cache_size=0.0), "cache_size > 0"),
                    (dict(num_threads=0), "num_threads")):
        with pytest.raises(ValueError, match=msg):
            pb._core._check_stereo_fusion_options(pb.StereoFusionOptions(kw))


def test_argument_checks_in_order(tmp_path):
    with pytest.raises(ValueError, match="ExistsDir"):
        pb.stereo_fusion(str(tmp_path / "x.ply"), str(tmp_path / "missing"), workspace_format="bad", input_type="bad")
    with pytest.raises(ValueError, match="workspace_format"):
        pb.stereo_fusion(str(tmp_path / "x.ply"), str(tmp_path), workspace_format="bad", input_type="bad")
    with pytest.raises(ValueError, match="Invalid input type"):
        pb.stereo_fusion(str(tmp_path / "x.ply"), str(tmp_path), input_type="bad")
    with pytest.raises(ValueError, match="PMVS"):
        pb.stereo_fusion(str(tmp_path / "x.ply"), str(tmp_path), workspace_format="PMVS")
    with pytest.raises(ValueError, match="extension .ply"):
        pb.stereo_fusion(str(tmp_path / "x.txt"), str(tmp_path))


def test_overlap_ranking_with_ties():
    m = mvs.SparseModel()
    for iid in (10, 20, 30, 40):
        m.images[iid] = (f"{iid}.png", 1, np.eye(3), np.zeros(3))
    tracks = [[10, 20], [10, 20], [10, 30], [10, 30], [10, 40], [20, 30, 30], [40, 30]]
    for k, t in enumerate(tracks):
        m.points[k + 1] = (np.zeros(3), t)
    ov = mvs.overlapping_images(m, 50)
    assert ov[0] == [1, 2, 3]          # 2 shared with 20 and 30 (tie: ascending index), 1 with 40
    assert ov[1] == [0, 2] and ov[2] == [0, 1, 3] and ov[3] == [0, 2]
    assert mvs.overlapping_images(m, 1)[0] == [1]


@pytest.fixture
def workspace(tmp_path, monkeypatch):
    ws = str(tmp_path / "ws")
    scene = syn.planar_scene(np.random.default_rng(4), 4, 64, 48)
    syn.write_dense_workspace(ws, scene, sources="__auto__, 2", points_per_view=60)
    for i in range(3):  # view 3 has no maps
        d, n = syn.fusion_maps(scene, i)
        for kind in ("geometric", "photometric"):
            mvs.write_array(mvs.map_paths(ws, f"view_{i:03d}.png", kind)[0], d)
            mvs.write_array(mvs.map_paths(ws, f"view_{i:03d}.png", kind)[1], n)
    calls = []

    def oracle_run(images, options, device):
        for im in images:
            c = im["color"]
            im["rgb"] = (pb._core.debug_decode_png(c)[:, :, :3] if c is not None else np.zeros((1, 1, 3), np.uint8))
            if im["rgb"].shape[2] == 1:
                im["rgb"] = np.repeat(im["rgb"], 3, 2)
        calls.append(images)
        r = F.run(images, options, "schedule")
        voff = np.cumsum([0] + [len(v) for v in r["visibility"]]).astype(np.int64)
        vis = np.concatenate(r["visibility"]) if r["visibility"] else np.zeros(0, np.int32)
        return dict(r, vis_off=voff, vis=vis)

    monkeypatch.setattr(mvs, "_fusion_run", oracle_run)
    return ws, calls


def test_ply_and_vis_layout(workspace, tmp_path, capfd):
    ws, calls = workspace
    out = str(tmp_path / "fused.ply")
    r = pb.stereo_fusion(out, ws)
    assert "view_003.png: no geometric depth and normal maps, skipped" in capfd.readouterr().err
    images = calls[0]
    assert [im["depth"] is None for im in images] == [False, False, False, True]
    assert len(r["xyz"]) > 100
    data = open(out, "rb").read()
    head = data[: data.index(b"end_header\n") + 11].decode()
    assert head.startswith("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % len(r["xyz"]))
    assert "property float nz\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n" in head
    assert len(data) - len(head) == 27 * len(r["xyz"])
    x, n, c = mvs.read_ply(out)
    assert np.array_equal(x, r["xyz"]) and np.array_equal(n, r["normals"]) and np.array_equal(c, r["colors"])
    vis = open(out + ".vis", "rb").read()
    assert struct.unpack_from("<Q", vis)[0] == len(r["xyz"])
    assert len(vis) == 8 + sum(4 + 4 * len(v) for v in r["visibility"])
    assert all(np.array_equal(a, b) for a, b in zip(mvs.read_points_visibility(out + ".vis"), r["visibility"]))
    assert all(set(v) <= {0, 1, 2} for v in r["visibility"])


def test_points3D_output(workspace, tmp_path):
    ws, _ = workspace
    out = tmp_path / "model"
    out.mkdir()
    r = pb.stereo_fusion(str(out), ws, input_type="photometric")
    assert (out / "cameras.bin").read_bytes() == open(os.path.join(ws, "sparse", "cameras.bin"), "rb").read()
    assert (out / "images.bin").read_bytes() == open(os.path.join(ws, "sparse", "images.bin"), "rb").read()
    first = max(mvs.read_sparse(os.path.join(ws, "sparse")).points) + 1
    data = (out / "points3D.bin").read_bytes()
    assert struct.unpack_from("<Q", data)[0] == len(r["xyz"])
    assert len(data) == 8 + 51 * len(r["xyz"])  # id, xyz, rgb, error, empty track
    pid, x, y, z, cr, cg, cb, err, tl = struct.unpack_from("<Q3d3BdQ", data, 8)
    assert pid == first and (x, y, z) == tuple(float(v) for v in r["xyz"][0]) and err == -1.0 and tl == 0
    assert (cr, cg, cb) == tuple(int(v) for v in r["colors"][0])


def test_narrowings(workspace, tmp_path):
    ws, _ = workspace
    with pytest.raises(ValueError, match="max_image_size"):
        pb.stereo_fusion(str(tmp_path / "a.ply"), ws, options=dict(max_image_size=32))
    masks = tmp_path / "masks"
    masks.mkdir()
    from PIL import Image
    Image.fromarray(np.ones((10, 10), np.uint8)).save(masks / "view_000.png.png")
    with pytest.raises(ValueError, match="depth map's size"):
        pb.stereo_fusion(str(tmp_path / "a.ply"), ws, options=dict(mask_path=str(masks)))


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        pb._core._stereo_fusion_run([], pb.StereoFusionOptions(), 0)

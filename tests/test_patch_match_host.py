"""CPU: the host side of patch_match_stereo -- PatchMatchOptions, the argument checks and refusals, the sparse model
reader (.bin and .txt), patch-match.cfg with `__auto__` selection and depth ranges, the map file format -- and the pass
controller (pass order, resume, allow_missing_files, output names, camera scaling) with the device call replaced by a
stand-in that records what it is given."""
import os
import struct

import numpy as np
import pytest

import pycolmap_b200 as pb
from pycolmap_b200 import mvs
from pycolmap_b200 import synthetic as syn


@pytest.fixture(scope="module")
def workspace(tmp_path_factory):
    ws = str(tmp_path_factory.mktemp("pm") / "ws")
    sc = syn.planar_scene(np.random.default_rng(4), 5, 96, 72)
    syn.write_dense_workspace(ws, sc, sources="__auto__, 3", points_per_view=120)
    return ws, sc


def test_option_defaults():
    o = pb.PatchMatchOptions()
    want = dict(max_image_size=-1, gpu_index="-1", depth_min=-1.0, depth_max=-1.0, window_radius=5, window_step=1,
                sigma_spatial=-1.0, sigma_color=0.2, num_samples=15, ncc_sigma=0.6, min_triangulation_angle=1.0,
                incident_angle_sigma=0.9, num_iterations=5, geom_consistency=True, geom_consistency_regularizer=0.3,
                geom_consistency_max_cost=3.0, filter=True, filter_min_ncc=0.1, filter_min_triangulation_angle=3.0,
                filter_min_num_consistent=2, filter_geom_consistency_max_cost=1.0, cache_size=32.0,
                allow_missing_files=False, write_consistency_graph=False)
    assert o.todict() == want
    assert pb.PatchMatchOptions(dict(window_radius=7)).window_radius == 7


@pytest.mark.parametrize("field,value,expr", [
    ("depth_min", 5.0, "depth_min <= depth_max"), ("window_radius", 33, "window_radius <= kMaxPatchMatchWindowRadius"),
    ("sigma_color", 0.0, "sigma_color > 0"), ("window_radius", 0, "window_radius > 0"), ("window_step", 0, "window_step > 0"),
    ("window_step", 3, "window_step <= 2"), ("num_samples", 0, "num_samples > 0"), ("ncc_sigma", 0.0, "ncc_sigma > 0"),
    ("min_triangulation_angle", -1.0, "min_triangulation_angle >= 0"),
    ("min_triangulation_angle", 180.0, "min_triangulation_angle < 180"),
    ("incident_angle_sigma", 0.0, "incident_angle_sigma > 0"), ("num_iterations", 0, "num_iterations > 0"),
    ("geom_consistency_regularizer", -1.0, "geom_consistency_regularizer >= 0"),
    ("geom_consistency_max_cost", -1.0, "geom_consistency_max_cost >= 0"), ("filter_min_ncc", -2.0, "filter_min_ncc >= -1"),
    ("filter_min_ncc", 2.0, "filter_min_ncc <= 1"),
    ("filter_min_triangulation_angle", -1.0, "filter_min_triangulation_angle >= 0"),
    ("filter_min_triangulation_angle", 181.0, "filter_min_triangulation_angle <= 180"),
    ("filter_min_num_consistent", -1, "filter_min_num_consistent >= 0"),
    ("filter_geom_consistency_max_cost", -1.0, "filter_geom_consistency_max_cost >= 0"), ("cache_size", 0.0, "cache_size > 0")])
def test_option_checks(workspace, field, value, expr):
    o = pb.PatchMatchOptions()
    setattr(o, field, value)
    with pytest.raises(ValueError, match=expr.replace("(", r"\(")):
        pb.patch_match_stereo(workspace[0], options=o)


def test_argument_checks_in_order(tmp_path, workspace):
    with pytest.raises(ValueError, match="ExistsDir"):
        pb.patch_match_stereo(str(tmp_path / "nope"), workspace_format="bad")
    with pytest.raises(ValueError, match="Invalid `workspace_format`"):
        pb.patch_match_stereo(workspace[0], workspace_format="bad", options=dict(num_iterations=0))
    with pytest.raises(ValueError, match="PMVS workspace format is not supported"):
        pb.patch_match_stereo(workspace[0], workspace_format="pmvs")
    with pytest.raises(ValueError, match="write_consistency_graph"):
        pb.patch_match_stereo(workspace[0], options=dict(write_consistency_graph=True))
    with pytest.raises(ValueError, match="one GPU"):
        pb.patch_match_stereo(workspace[0], options=dict(gpu_index="0,1"))


def test_non_pinhole_camera_refused(tmp_path):
    ws = str(tmp_path / "ws")
    syn.write_dense_workspace(ws, syn.planar_scene(np.random.default_rng(0), 2, 48, 36), sources="__all__",
                              points_per_view=50)
    p = os.path.join(ws, "sparse", "cameras.bin")
    with open(p, "wb") as f:
        f.write(struct.pack("<Q", 2))
        for i in range(2):
            f.write(struct.pack("<iiQQ4d", i + 1, 2, 48, 36, 40.0, 24.0, 18.0, 0.01))
    with pytest.raises(ValueError, match="PINHOLE or SIMPLE_PINHOLE"):
        pb.patch_match_stereo(ws)


def _write_txt(model, path):
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "cameras.txt"), "w") as f:
        f.write("# comment\n")
        for cid, (m, w, h, p) in model.cameras.items():
            f.write(f"{cid} {mvs._MODEL_NAMES[m]} {w} {h} " + " ".join(repr(float(v)) for v in p) + "\n")
    with open(os.path.join(path, "images.txt"), "w") as f:
        for iid, (name, cid, R, t) in model.images.items():
            q = syn._rot_to_quat(R)
            f.write(f"{iid} " + " ".join(repr(float(v)) for v in (*q, *t)) + f" {cid} {name}\n\n")
    with open(os.path.join(path, "points3D.txt"), "w") as f:
        for pid, (xyz, track) in model.points.items():
            f.write(f"{pid} " + " ".join(repr(float(v)) for v in xyz) + " 1 2 3 0.5 " +
                    " ".join(f"{i} 0" for i in track) + "\n")


def test_sparse_bin_equals_txt(workspace, tmp_path):
    a = mvs.read_sparse(os.path.join(workspace[0], "sparse"))
    _write_txt(a, str(tmp_path / "txt"))
    b = mvs.read_sparse(str(tmp_path / "txt"))
    assert a.cameras.keys() == b.cameras.keys() and a.images.keys() == b.images.keys()
    for k in a.cameras:
        assert a.cameras[k][:3] == b.cameras[k][:3] and np.array_equal(a.cameras[k][3], b.cameras[k][3])
    for k in a.images:
        assert a.images[k][:2] == b.images[k][:2]
        assert np.allclose(a.images[k][2], b.images[k][2], atol=1e-12) and np.array_equal(a.images[k][3], b.images[k][3])
    assert a.points.keys() == b.points.keys()
    for k in a.points:
        assert np.array_equal(a.points[k][0], b.points[k][0]) and a.points[k][1] == b.points[k][1]


def _auto_restated(model, ref, num, min_angle):
    """__auto__ restated directly: rank by shared points, keep 75th-percentile angle >= min_angle, first num."""
    C = {i: -R.T @ t for i, (_, _, R, t) in model.images.items()}
    rows = []
    for i in sorted(model.images):
        if i == ref:
            continue
        X = [xyz for xyz, tr in model.points.values() if ref in tr and i in tr]
        if not X:
            continue
        X = np.array(X)
        a, b = X - C[ref], X - C[i]
        ang = np.degrees(np.arccos(np.clip((a * b).sum(1) / np.linalg.norm(a, axis=1) / np.linalg.norm(b, axis=1), -1, 1)))
        rows.append((-len(X), i, np.percentile(ang, 75)))
    counts = [r[0] for r in rows]
    assert len(set(counts)) == len(counts), "the test scene must have no ties"
    return [i for _, i, a in sorted(rows) if a >= min_angle][:num]


def test_config_variants_auto_and_depth_ranges(workspace, tmp_path):
    model = mvs.read_sparse(os.path.join(workspace[0], "sparse"))
    names = {v[0]: k for k, v in model.images.items()}
    cfg = tmp_path / "pm.cfg"
    cfg.write_text("view_000.png\n__all__\n\n# comment\nview_001.png\n__auto__, 2\nview_002.png\nview_004.png, view_000.png\n")
    probs = mvs.read_config(str(cfg), model, 1.0)
    assert probs[0] == (names["view_000.png"], [i for i in sorted(model.images) if i != names["view_000.png"]])
    assert probs[1] == (names["view_001.png"], _auto_restated(model, names["view_001.png"], 2, 1.0))
    assert probs[2] == (names["view_002.png"], [names["view_004.png"], names["view_000.png"]])
    for iid, (_, _, R, t) in model.images.items():
        d = np.sort([(R @ xyz + t)[2] for xyz, tr in model.points.values() if iid in tr])
        n = len(d)
        assert mvs.depth_range(model, iid) == pytest.approx((d[int(0.01 * n)] * 0.75, d[int(0.99 * n)] * 1.25))
    cfg.write_text("view_000.png\n")
    with pytest.raises(ValueError, match="pairs of lines"):
        mvs.read_config(str(cfg), model, 1.0)


def test_map_files_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    d = rng.random((7, 5)).astype(np.float32)
    n = rng.random((7, 5, 3)).astype(np.float32)
    mvs.write_array(str(tmp_path / "d.bin"), d)
    mvs.write_array(str(tmp_path / "n.bin"), n)
    assert open(tmp_path / "d.bin", "rb").read(6) == b"5&7&1&"
    assert np.array_equal(mvs.read_array(str(tmp_path / "d.bin")), d)
    assert np.array_equal(mvs.read_array(str(tmp_path / "n.bin")), n)
    raw = np.frombuffer(open(tmp_path / "n.bin", "rb").read()[6:], np.float32)
    assert np.array_equal(raw[:35], n[:, :, 0].ravel())  # channel-major, each channel row-major


def test_no_cpu_fallback(workspace):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pb.patch_match_stereo(workspace[0], options=dict(num_iterations=1))


class _Recorder:
    """Stands in for the device: decodes with the host PNG reader and records every call."""

    def __init__(self, monkeypatch):
        self.calls = []
        monkeypatch.setattr(mvs, "_run", self.run)
        monkeypatch.setattr(mvs, "_decode", self.decode)

    @staticmethod
    def decode(path, max_image_size, device):
        from PIL import Image
        im = Image.open(path).convert("L")
        if max_image_size > 0 and max(im.size) > max_image_size:
            s = max_image_size / max(im.size)
            im = im.resize((int(im.size[0] * s), int(im.size[1] * s)))
        return np.asarray(im)

    def run(self, images, cameras, depth_maps, problems, options, geom, filt):
        self.calls.append(dict(geom=geom, filter=filt, cameras=cameras.copy(), problems=problems,
                               sizes=[im.shape for im in images], has_dmaps=depth_maps is not None))
        return [(np.full(images[p["ref"]].shape, p["depth_min"], np.float32),
                 np.zeros(images[p["ref"]].shape + (3,), np.float32)) for p in problems]


def test_controller_pass_order_names_and_resume(workspace, tmp_path, monkeypatch):
    import shutil
    ws = str(tmp_path / "ws")
    shutil.copytree(workspace[0], ws)
    rec = _Recorder(monkeypatch)
    pb.patch_match_stereo(ws)
    assert [(c["geom"], c["filter"]) for c in rec.calls] == [(False, False), (True, True)]
    assert len(rec.calls[0]["problems"]) == 5 and len(rec.calls[1]["problems"]) == 5
    assert rec.calls[1]["has_dmaps"] and all("init_depth" in p for p in rec.calls[1]["problems"])
    for i in range(5):
        for kind in ("photometric", "geometric"):
            for p in mvs.map_paths(ws, f"view_{i:03d}.png", kind):
                assert os.path.isfile(p)
    n = len(rec.calls)
    pb.patch_match_stereo(ws)
    assert len(rec.calls) == n  # resume: nothing left to do, no device call
    os.remove(mvs.map_paths(ws, "view_002.png", "geometric")[0])
    pb.patch_match_stereo(ws)
    assert len(rec.calls) == n + 1 and rec.calls[-1]["geom"] and len(rec.calls[-1]["problems"]) == 1


def test_controller_photometric_only_and_missing_files(workspace, tmp_path, monkeypatch):
    import shutil
    ws = str(tmp_path / "ws")
    shutil.copytree(workspace[0], ws)
    os.remove(os.path.join(ws, "images", "view_003.png"))
    rec = _Recorder(monkeypatch)
    with pytest.raises(ValueError, match="missing"):
        pb.patch_match_stereo(ws, options=dict(geom_consistency=False))
    pb.patch_match_stereo(ws, options=dict(geom_consistency=False, allow_missing_files=True))
    assert [(c["geom"], c["filter"]) for c in rec.calls] == [(False, True)]
    model = mvs.read_sparse(os.path.join(ws, "sparse"))
    involve3 = [ref for ref, src in mvs.read_config(os.path.join(ws, "stereo", "patch-match.cfg"), model, 1.0)
                if 4 in [ref] + src]
    assert len(rec.calls[0]["problems"]) == 5 - len(involve3)
    assert not any(os.path.isfile(p) for i in involve3 for p in mvs.map_paths(ws, model.images[i][0], "photometric"))


def test_controller_camera_scaling(workspace, tmp_path, monkeypatch):
    import shutil
    ws = str(tmp_path / "ws")
    shutil.copytree(workspace[0], ws)
    rec = _Recorder(monkeypatch)
    pb.patch_match_stereo(ws, options=dict(geom_consistency=False, max_image_size=48))
    c = rec.calls[0]
    assert all(s == (36, 48) for s in c["sizes"])
    fx, fy, cx, cy = workspace[1]["cameras"][0]["K"]
    assert np.allclose(c["cameras"][0, :4], [fx * 0.5, fy * 0.5, cx * 0.5, cy * 0.5])
    assert mvs.read_array(mvs.map_paths(ws, "view_000.png", "photometric")[0]).shape == (36, 48)

"""GPU: K8 (PatchMatch stereo) against the numpy oracle oracle/patch_match.py and against rendered ground truth, and
patch_match_stereo end to end on a rendered dense workspace (pycolmap_b200.synthetic.planar_scene)."""
import os
import shutil

import numpy as np
import pytest

import oracle.patch_match as O
import pycolmap_b200 as pb
from pycolmap_b200 import _core, mvs
from pycolmap_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


def _scene(n, w, h, tex, seed=3):
    sc = syn.planar_scene(np.random.default_rng(seed), n, w, h, texture_size=tex)
    r = [syn.render_planar(sc, i) for i in range(n)]
    cams = np.array([list(c["K"]) + list(c["R"].ravel()) + list(c["t"]) for c in sc["cameras"]])
    return sc, r, cams


def _opts(**kw):
    o = pb.PatchMatchOptions()
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def test_debug_cost_matches_oracle():
    sc, r, cams = _scene(3, 96, 72, 64)
    imgs = [x[0] for x in r]
    rng = np.random.default_rng(0)
    for step in (1, 2):
        o = _opts(window_step=step)
        oo = O.defaults(window_step=step)
        n = 400
        x = rng.integers(0, 96, n)
        y = rng.integers(0, 72, n)
        x[:40] = rng.choice([0, 1, 94, 95], 40)  # window border
        d = rng.uniform(4, 16, n).astype(np.float32)
        nrm = rng.normal(size=(n, 3))
        nrm[:, 2] = -np.abs(nrm[:, 2]) - 0.02
        nrm[40:80, 2] = -0.03  # grazing planes
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        s = rng.integers(0, 2, n)
        q = np.c_[x, y, d, nrm, s].astype(np.float32)
        dmaps = [x[1] for x in r]
        got = _core.debug_patch_match_cost(imgs, cams, dmaps, dict(ref=0, src=[1, 2], depth_min=4.0, depth_max=16.0), q, o)
        pr = O.Problem(imgs, [tuple(c[:4]) + (c[4:13].reshape(3, 3), c[13:]) for c in cams], 0, [1, 2], 4.0, 16.0, dmaps)
        P = O.Params(oo)
        for k in range(2):
            m = s == k
            nn = nrm[m].astype(np.float32)
            want = O.photo_cost(P, pr, k, x[m], y[m], d[m], nn)
            assert np.abs(got[m, 0] - want).max() < 2e-3, np.abs(got[m, 0] - want).max()
            wg = O.geom_error(P, pr, k, x[m], y[m], d[m], nn)
            assert np.abs(got[m, 1] - wg).max() < 1e-2
            wp = O.propagated_depth(pr.K[0], x[m], y[m], d[m], nn, x[m], y[m] + 1)
            ok = np.isfinite(wp) & (np.abs(wp) < 1e4)
            assert np.allclose(got[m, 2][ok], wp[ok], rtol=1e-4)


def _run(imgs, cams, problems, o, geom=False, filt=False, dmaps=None):
    return _core._patch_match_run(imgs, cams, dmaps, problems, o, geom, filt)


def test_tiny_scene_gpu_vs_oracle():
    sc, r, cams = _scene(4, 80, 60, 48)
    imgs = [x[0] for x in r]
    o = _opts(num_iterations=2)
    (d, n), = _run(imgs, cams, [dict(ref=0, src=[1, 2, 3], depth_min=4.0, depth_max=16.0)], o)
    pr = O.Problem(imgs, [tuple(c[:4]) + (c[4:13].reshape(3, 3), c[13:]) for c in cams], 0, [1, 2, 3], 4.0, 16.0)
    od, on = O.run(pr, O.defaults(num_iterations=2, filter=False), seed=0)
    gt = r[0][1]
    agree = (np.abs(d - od) <= 1e-3 * od).mean()
    acc_gpu = (np.abs(d - gt) < 0.05 * gt).mean()
    acc_or = (np.abs(od - gt) < 0.05 * gt).mean()
    print(f"tiny scene: GPU and oracle agree on {agree:.3f} of the pixels; within 5 %: GPU {acc_gpu:.3f}, oracle {acc_or:.3f}")
    # measured on an H100: 0.983; a flip on a near-tie propagates down a column, so the floor leaves a margin
    assert agree >= 0.95
    assert acc_gpu >= acc_or - 0.01


def _medium(tmp_path, sources="__auto__, 5"):
    sc = syn.planar_scene(np.random.default_rng(7), 8, 640, 480)
    ws = str(tmp_path / "ws")
    renders = syn.write_dense_workspace(ws, sc, sources=sources)
    return sc, ws, renders


def _visible_in_two_sources(sc, renders, i, sources):
    """Pixels of view i whose true surface point is seen, unoccluded, by at least two of `sources` (view indices)."""
    cam = sc["cameras"][i]
    d = renders[i][1].astype(np.float64)
    H, W = d.shape
    ys, xs = np.mgrid[0:H, 0:W]
    fx, fy, cx, cy = cam["K"]
    Xc = np.stack([(xs + 0.5 - cx) / fx * d, (ys + 0.5 - cy) / fy * d, d], -1)
    Xw = (Xc - cam["t"]) @ cam["R"]
    count = np.zeros((H, W), int)
    for j in sources:
        cj = sc["cameras"][j]
        Y = Xw @ cj["R"].T + cj["t"]
        with np.errstate(all="ignore"):
            u = cj["K"][0] * Y[..., 0] / Y[..., 2] + cj["K"][2]
            v = cj["K"][1] * Y[..., 1] / Y[..., 2] + cj["K"][3]
        inside = (Y[..., 2] > 0) & (u >= 0) & (v >= 0) & (u < W) & (v < H)
        ui, vi = np.where(inside, u, 0).astype(int), np.where(inside, v, 0).astype(int)
        dj = renders[j][1][vi, ui]
        count += inside & (np.abs(dj - Y[..., 2]) < 0.01 * Y[..., 2])
    return (count >= 2) & (d > 0)


def test_medium_scene_accuracy_and_resume(tmp_path):
    sc = syn.planar_scene(np.random.default_rng(7), 8, 640, 480)
    ws = str(tmp_path / "ws")
    renders = syn.write_dense_workspace(ws, sc, sources="__auto__, 5")
    pb.patch_match_stereo(ws)
    model = mvs.read_sparse(os.path.join(ws, "sparse"))
    problems = dict(mvs.read_config(os.path.join(ws, "stereo", "patch-match.cfg"), model, 1.0))
    within, off, nerr = [], [], []
    for i in range(8):
        name = f"view_{i:03d}.png"
        d = mvs.read_array(mvs.map_paths(ws, name, "geometric")[0])
        n = mvs.read_array(mvs.map_paths(ws, name, "geometric")[1])
        gt, gn = renders[i][1], renders[i][2]
        vis = _visible_in_two_sources(sc, renders, i, [s - 1 for s in problems[i + 1]])
        kept = (d > 0) & vis
        rel = np.abs(d - gt) / np.maximum(gt, 1e-6)
        within.append((rel[kept] < 0.01).mean())
        off.append((rel[kept] > 0.05).mean())
        cosang = np.clip((n[kept] * gn[kept]).sum(-1), -1, 1)
        nerr.append(np.degrees(np.median(np.arccos(cosang))))
    print(f"medium scene (8 x 640x480, __auto__, 5, defaults), kept pixels visible in >= 2 sources: within 1 %: "
          f"{np.mean(within):.4f}; more than 5 % off: {np.mean(off):.4f}; median normal error {np.mean(nerr):.2f} deg")
    assert np.mean(within) >= 0.90
    assert np.mean(off) <= 0.01
    assert np.mean(nerr) <= 5.0
    # resume: the geometric pass again from the photometric files gives the same maps
    name = "view_000.png"
    ref = mvs.read_array(mvs.map_paths(ws, name, "geometric")[0])
    for i in range(8):
        for p in mvs.map_paths(ws, f"view_{i:03d}.png", "geometric"):
            os.remove(p)
    pb.patch_match_stereo(ws)
    assert np.array_equal(mvs.read_array(mvs.map_paths(ws, name, "geometric")[0]), ref)


def test_maps_do_not_depend_on_the_other_problems(tmp_path):
    """A problem's maps are the same whether the call runs every problem of the workspace, only that problem (a config
    listing a subset), or resumes after its maps were deleted: the random numbers are keyed by the workspace image id,
    not by the position of the image in the pass's image set."""
    sc = syn.planar_scene(np.random.default_rng(9), 5, 160, 120)
    full = str(tmp_path / "full")
    syn.write_dense_workspace(full, sc, sources="__all__", points_per_view=150)
    nbrs = {0: (1, 2), 1: (0, 2), 2: (1, 3), 3: (2, 4), 4: (3, 2)}
    lines = [f"view_{i:03d}.png\n" + ", ".join(f"view_{j:03d}.png" for j in nbrs[i]) + "\n" for i in range(5)]
    with open(os.path.join(full, "stereo", "patch-match.cfg"), "w") as f:
        f.writelines(lines)
    sub = str(tmp_path / "sub")
    shutil.copytree(full, sub)
    with open(os.path.join(sub, "stereo", "patch-match.cfg"), "w") as f:
        f.write(lines[2])
    opts = dict(num_iterations=2)
    pb.patch_match_stereo(full, options=opts)
    for j in (1, 3):  # the sources' photometric depth maps the geometric pass of view 2 reads
        for p, q in zip(mvs.map_paths(full, f"view_{j:03d}.png", "photometric"),
                        mvs.map_paths(sub, f"view_{j:03d}.png", "photometric")):
            os.makedirs(os.path.dirname(q), exist_ok=True)
            shutil.copy(p, q)
    pb.patch_match_stereo(sub, options=opts)  # view 2 alone: its images are the set {1, 2, 3}, the reference at index 1
    name = "view_002.png"
    want = [mvs.read_array(p) for kind in ("photometric", "geometric") for p in mvs.map_paths(full, name, kind)]
    got = [mvs.read_array(p) for kind in ("photometric", "geometric") for p in mvs.map_paths(sub, name, kind)]
    assert all(np.array_equal(a, b) for a, b in zip(want, got))
    for kind in ("photometric", "geometric"):
        for p in mvs.map_paths(full, name, kind):
            os.remove(p)
    pb.patch_match_stereo(full, options=opts)  # resume: only view 2 runs, in the image set {1, 2, 3}
    again = [mvs.read_array(p) for kind in ("photometric", "geometric") for p in mvs.map_paths(full, name, kind)]
    assert all(np.array_equal(a, b) for a, b in zip(want, again))


def test_bit_identical_alone_and_in_batch():
    sc, r, cams = _scene(5, 120, 90, 96)
    imgs = [x[0] for x in r]
    o = _opts(num_iterations=2)
    p0 = dict(ref=2, image_id=2, src=[0, 1, 3], depth_min=4.0, depth_max=16.0)
    alone = _run(imgs, cams, [p0], o, filt=True)[0]
    # the same problem in an image set where its images sit at other indices, keyed by the same image id
    perm = [3, 2, 0, 1, 4]
    moved = _run([imgs[k] for k in perm], cams[perm], [dict(p0, ref=1, src=[2, 3, 0])], o, filt=True)[0]
    again = _run(imgs, cams, [p0], o, filt=True)[0]
    batch = _run(imgs, cams, [dict(ref=0, src=[1, 2], depth_min=4.0, depth_max=16.0),
                              dict(ref=4, src=[3, 1, 0, 2], depth_min=3.0, depth_max=18.0), p0], o, filt=True)[2]
    for a, b in ((alone, again), (alone, batch), (alone, moved)):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_max_image_size(tmp_path):
    sc = syn.planar_scene(np.random.default_rng(2), 3, 200, 150)
    ws = str(tmp_path / "ws")
    syn.write_dense_workspace(ws, sc, sources="__all__", points_per_view=200)
    pb.patch_match_stereo(ws, options=dict(max_image_size=100, num_iterations=1, geom_consistency=False))
    d = mvs.read_array(mvs.map_paths(ws, "view_000.png", "photometric")[0])
    assert d.shape == (75, 100)


def test_stats_counters():
    sc, r, cams = _scene(3, 64, 48, 32)
    imgs = [x[0] for x in r]
    before = _core._patch_match_stats(0)
    _run(imgs, cams, [dict(ref=0, src=[1, 2], depth_min=4.0, depth_max=16.0)], _opts(num_iterations=1))
    after = _core._patch_match_stats(0)
    assert after["pm_problems"] - before["pm_problems"] == 1
    assert after["pm_pixel_updates"] - before["pm_pixel_updates"] == 64 * 48 * 4
    # at least the current hypothesis against both sources over every in-image window sample of every pixel update
    assert after["pm_window_samples"] - before["pm_window_samples"] > 64 * 48 * 4 * 2 * 60
    assert "pm_window_samples" in pb.Context(device=0).stats()

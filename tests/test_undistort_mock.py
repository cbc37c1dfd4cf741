"""CPU: undistort_images through the host module against a CPU stand-in for the undistortion entry points
(tests/helpers/mock_undistort.cpp, built with tests/helpers/mock_b200match.cpp into a temporary directory and put in
front of the real library): what reaches the C ABI, the chunks of 32 images, every output file written exactly once,
and every written image the size of its written camera -- also for distortion-free non-pinhole cameras and an ROI,
whose images must be warped, not copied."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

SCRIPT = textwrap.dedent("""
    import io, json, os, sys
    sys.path.insert(0, {root!r})
    import numpy as np
    from PIL import Image
    import pycolmap_b200 as pb
    from pycolmap_b200 import mvs
    root = sys.argv[1]
    W, H = 40, 30
    m = mvs.SparseModel()
    m.cameras[1] = (2, W, H, np.array([35.0, 20.0, 15.0, 0.0]))                       # SIMPLE_RADIAL, k = 0
    m.cameras[2] = (4, W, H, np.array([35.0, 36.0, 20.0, 15.0, -0.2, 0.03, 0.0, 0.0]))  # OPENCV
    m.cameras[3] = (1, W, H, np.array([35.0, 36.0, 20.0, 15.0]))                      # PINHOLE
    os.makedirs(os.path.join(root, "images"))
    rng = np.random.default_rng(0)
    for i in range(70):
        ext = ".png" if i % 2 else ".jpg"
        name = f"v{{i:03d}}{{ext}}"
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(os.path.join(root, "images", name))
        cid = 1 if i < 30 else (2 if i < 60 else 3)
        m.images[i + 1] = (name, cid, np.eye(3), np.zeros(3))
        m.image_raw[i + 1] = (np.array([1.0, 0, 0, 0]), np.zeros(3), np.array([[10.5, 7.25]]), np.array([-1]))
    mvs.write_sparse_bin(os.path.join(root, "sparse"), m)

    writes = {{}}
    real = mvs._write_file
    def counted(path, data):
        writes[path] = writes.get(path, 0) + 1
        real(path, data)
    mvs._write_file = counted

    def sizes(out):
        got = {{}}
        model = mvs.read_sparse(os.path.join(out, "sparse"))
        for iid, (name, cid, _, _) in model.images.items():
            if not os.path.exists(os.path.join(out, "images", name)):
                continue
            data = open(os.path.join(out, "images", name), "rb").read()
            if data.startswith(b"MOCKJPEG"):
                wh = [int(v) for v in data.split()[1:]]
            else:
                a = pb._core.debug_decode_png(data) if name.endswith(".png") else np.asarray(Image.open(io.BytesIO(data)))
                wh = [a.shape[1], a.shape[0]]
            cam = model.cameras[cid]
            got[name] = [wh, [cam[1], cam[2]], int(cam[0]), os.path.islink(os.path.join(out, "images", name))]
        return got

    out = {{}}
    pb.undistort_images(os.path.join(root, "a"), os.path.join(root, "sparse"), os.path.join(root, "images"),
                        copy_policy="soft-link")
    out["a"] = dict(sizes=sizes(os.path.join(root, "a")), writes=writes.copy())
    writes.clear()
    pb.undistort_images(os.path.join(root, "b"), os.path.join(root, "sparse"), os.path.join(root, "images"),
                        image_list=[f"v{{i:03d}}.png" for i in range(61, 70, 2)], copy_policy="soft-link",
                        undistort_options=dict(roi_min_x=0.1, roi_max_y=0.8))
    out["b"] = dict(sizes=sizes(os.path.join(root, "b")), writes=writes.copy(),
                    cfg=open(os.path.join(root, "b", "stereo", "fusion.cfg")).read().split())
    print("RESULT", json.dumps(out))
""")


@pytest.fixture(scope="module")
def mock_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("mock_undistort"))
    oracle_dir = os.path.join(ROOT, "oracle")
    subprocess.check_call(["make", "-C", oracle_dir, "-s"])
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-o",
                           os.path.join(out, "libb200match.so"), os.path.join(HERE, "helpers", "mock_b200match.cpp"),
                           os.path.join(HERE, "helpers", "mock_undistort.cpp"), "-L", oracle_dir, "-loracle",
                           f"-Wl,-rpath,{oracle_dir}"])
    return out


def test_undistort_images_through_the_host_module(mock_lib, tmp_path):
    log = tmp_path / "undistort.log"
    env = dict(os.environ, LD_LIBRARY_PATH=mock_lib + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""),
               B2M_MOCK_UNDISTORT_LOG=str(log))
    r = subprocess.run([sys.executable, "-c", SCRIPT.format(root=ROOT), str(tmp_path / "ws")], env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "RESULT" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(r.stdout.split("RESULT", 1)[1])
    calls = [ln for ln in log.read_text().splitlines() if ln.startswith("CALL")]
    items = [dict(kv.split("=") for kv in ln.split()[1:]) for ln in log.read_text().splitlines() if ln.startswith("ITEM")]

    # run a: the 60 SIMPLE_RADIAL (k = 0) and OPENCV images go to the device in chunks of 32; the PINHOLE ones are linked
    # run b: with an ROI every image is warped, PINHOLE included: one call of 5
    assert calls == ["CALL 32", "CALL 28", "CALL 5"]
    a_items, b_items = items[:60], items[60:]
    assert [it["model"] for it in a_items] == ["2"] * 30 + ["4"] * 30
    assert [it["output"] for it in a_items] == ["0", "1"] * 30  # JPEG for .jpg names, pixels for .png
    assert [it["source"] for it in a_items] == ["0", "1"] * 30  # JPEG files whole, PNG files decoded on the host
    assert all(it["camera"] == "40x30" for it in items)
    assert [it["model"] for it in b_items] == ["1"] * 5

    for run, n_written in (("a", 60), ("b", 5)):
        writes = res[run]["writes"]
        assert len(writes) == n_written and set(writes.values()) == {1}, run
        assert len(res[run]["sizes"]) == (70 if run == "a" else 5)
        for name, (wh, cam_wh, model, link) in res[run]["sizes"].items():
            assert wh == cam_wh and model == 1, (run, name, wh, cam_wh)
    a = res["a"]["sizes"]
    assert a["v000.jpg"][1] == [39, 29]  # SIMPLE_RADIAL with k = 0 is not the input's pinhole camera: warped
    assert all(v[3] == (int(k[1:4]) >= 60) for k, v in a.items())  # only the PINHOLE images are links
    b = res["b"]
    assert b["cfg"] == [f"v{i:03d}.png" for i in range(61, 70, 2)]
    from oracle import undistort as U
    want = U.undistort_camera(dict(roi_min_x=0.1, roi_max_y=0.8),
                              dict(model=1, width=40, height=30, params=[35.0, 36.0, 20.0, 15.0]))
    assert all(not b["sizes"][n][3] and b["sizes"][n][1] == [want["width"], want["height"]] != [40, 30]
               for n in b["cfg"])

"""CPU: patch_match_stereo through the host module against a CPU stand-in for the PatchMatch entry points
(tests/helpers/mock_patch_match.cpp, built with tests/helpers/mock_b200match.cpp into a temporary directory and put in
front of the real library): options and problems reach the C ABI, pass order, image ids, resume, output names."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

SCRIPT = textwrap.dedent("""
    import sys
    sys.path.insert(0, {root!r})
    import numpy as np
    import pycolmap_b200 as pb
    from pycolmap_b200 import mvs, synthetic as syn
    ws = sys.argv[1]
    syn.write_dense_workspace(ws, syn.planar_scene(np.random.default_rng(1), 4, 64, 48), sources="__auto__, 2",
                              points_per_view=100)
    pb.patch_match_stereo(ws, options=dict(num_iterations=3, window_radius=4))
    for i in range(4):
        for kind in ("photometric", "geometric"):
            d = mvs.read_array(mvs.map_paths(ws, f"view_{{i:03d}}.png", kind)[0])
            n = mvs.read_array(mvs.map_paths(ws, f"view_{{i:03d}}.png", kind)[1])
            print("MAP", i, kind, d.shape, float(d[0, 0]), float(n[0, 0, 2]))
    pb.patch_match_stereo(ws, options=dict(num_iterations=3, window_radius=4))
    print("MOCK-PM-OK")
""")


@pytest.fixture(scope="module")
def mock_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("mock_pm"))
    oracle_dir = os.path.join(ROOT, "oracle")
    subprocess.check_call(["make", "-C", oracle_dir, "-s"])
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-o",
                           os.path.join(out, "libb200match.so"), os.path.join(HERE, "helpers", "mock_b200match.cpp"),
                           os.path.join(HERE, "helpers", "mock_patch_match.cpp"), "-L", oracle_dir, "-loracle",
                           f"-Wl,-rpath,{oracle_dir}"])
    return out


def test_patch_match_stereo_through_the_host_module(mock_lib, tmp_path):
    log = tmp_path / "pm.log"
    env = dict(os.environ, LD_LIBRARY_PATH=mock_lib + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""),
               B2M_MOCK_PM_LOG=str(log))
    r = subprocess.run([sys.executable, "-c", SCRIPT.format(root=ROOT), str(tmp_path / "ws")], env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "MOCK-PM-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
    lines = log.read_text().splitlines()
    # two device calls: the photometric pass without filter, then the geometric pass with it; nothing on the resume
    batches = [ln for ln in lines if ln.startswith("BATCH")]
    assert batches == ["BATCH 4 geom=0 filter=0 iters=3 radius=4", "BATCH 4 geom=1 filter=1 iters=3 radius=4"]
    sets = [ln.split() for ln in lines if ln.startswith("SET")]
    assert len(sets) == 2 and all(e.startswith("64x48:0:") for e in sets[0][2:])
    assert all(e.startswith("64x48:1:") for e in sets[1][2:])  # every source has its photometric depth map
    probs = [ln.split() for ln in lines if ln.startswith("PROBLEM")]
    ids = [int(p[2].split("=")[1]) for p in probs]
    assert ids == [1, 2, 3, 4, 1, 2, 3, 4]  # the workspace image ids key the random numbers
    assert [p[3] for p in probs] == ["n_src=2"] * 8
    assert [p[4] for p in probs] == ["init=0"] * 4 + ["init=1"] * 4
    maps = [ln.split() for ln in r.stdout.splitlines() if ln.startswith("MAP")]
    assert len(maps) == 8
    for m in maps:
        assert m[3:5] == ["(48,", "64)"] and float(m[6]) == -1.0
    # depth = depth_min + image id: the map of view i went to view i's files
    for i in range(4):
        d = [float(m[5]) for m in maps if m[1] == str(i)]
        assert all(v - (i + 1) > 0 for v in d)

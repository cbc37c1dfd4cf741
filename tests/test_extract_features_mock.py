"""CPU: the host pipeline of extract_features (reader thread, camera assignment, device calls of up to 32 images,
writer thread, skips) against a CPU stand-in for the extraction entry points (tests/helpers/mock_extract.cpp, built
with tests/helpers/mock_b200match.cpp into a temporary directory and put in front of the real library)."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

SCRIPT = textwrap.dedent("""
    import sys
    import numpy as np
    sys.path.insert(0, {root!r})
    import pycolmap_b200 as nat
    db, imgs = sys.argv[1], sys.argv[2]
    nat.extract_features(db, imgs, reader_options={{"camera_mask_path": imgs + "/../no_such_mask.png"}})
    with nat.Database(db) as d:
        for iid, name, cid in d.read_all_images():
            cam = d.read_camera(cid)
            kp, de = d.read_keypoints(iid), d.read_descriptors(iid)
            print("ROW", name, cam["width"], cam["height"], kp.shape[0], kp.shape[1], float(kp.sum()), int(de.sum()))
    print("MOCK-EXTRACT-OK")
""")


@pytest.fixture(scope="module")
def mock_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("mock_extract"))
    oracle_dir = os.path.join(ROOT, "oracle")
    subprocess.check_call(["make", "-C", oracle_dir, "-s"])
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-o",
                           os.path.join(out, "libb200match.so"), os.path.join(HERE, "helpers", "mock_b200match.cpp"),
                           os.path.join(HERE, "helpers", "mock_extract.cpp"), "-L", oracle_dir, "-loracle",
                           f"-Wl,-rpath,{oracle_dir}"])
    return out


def _mock_rows(w, h):
    """What mock_extract.cpp writes for a decoded w x h image: keypoints, descriptor sums."""
    nf = 1 + (w + h) % 4
    kp_sum = sum(k + 0.5 + w / 2.0 + 2.0 for k in range(nf))
    de_sum = sum((w * 7 + k + d) & 255 for k in range(nf) for d in range(128))
    return nf, kp_sum, de_sum


def test_extract_features_control_flow(mock_lib, tmp_path):
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    sizes = {}
    for k in range(40):  # two device calls (32 + 8)
        w, h = 20 + k, 16
        name = f"{k:03d}.{'png' if k % 3 == 0 else 'jpg'}"
        img = Image.fromarray(np.full((h, w, 3), 3 * k, np.uint8))
        img.save(imgs / name)
        sizes[name] = (w, h)
    (imgs / "010.txt").write_text("not an image")              # skipped by the host reader
    for k, tag in ((5, b"MOCKBAD"), (31, b"MOCKBAD"), (34, b"MOCKSIZE")):  # skipped after the device call
        p = imgs / f"{k:03d}.jpg"
        p.write_bytes(p.read_bytes() + tag)
    log = tmp_path / "opts.log"
    env = dict(os.environ, LD_LIBRARY_PATH=mock_lib + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""),
               B2M_MOCK_EXTRACT_LOG=str(log))
    r = subprocess.run([sys.executable, "-c", SCRIPT.format(root=ROOT), str(tmp_path / "m.db"), str(imgs)], env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "MOCK-EXTRACT-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
    rows = [line.split()[1:] for line in r.stdout.splitlines() if line.startswith("ROW")]
    skipped = {"005.jpg", "031.jpg", "034.jpg"}
    want = [n for n in sorted(sizes) if n not in skipped]
    assert [row[0] for row in rows] == want
    for name, cw, ch, n, cols, kp_sum, de_sum in rows:
        w, h = sizes[name]
        nf, ks, ds = _mock_rows(w, h)
        assert (int(cw), int(ch), int(n), int(cols), int(de_sum)) == (w, h, nf, 6, ds), name
        assert float(kp_sum) == pytest.approx(ks, abs=1e-4), name
    for name, why in (("010.txt", "not a JPEG or PNG file"), ("005.jpg", "mock: does not decode"),
                      ("031.jpg", "mock: does not decode"), ("034.jpg", "decodes to a size other than its header's")):
        assert f"{name}: {why}, skipped" in r.stderr, (name, r.stderr[-3000:])
    # an unreadable camera mask is reported and extraction goes on without it, as upstream's controller does
    assert "no_such_mask.png" in r.stderr and "No mask is going to be used." in r.stderr
    # two device calls, the sources of each: the 32 loaded files minus the host skip, then the 9 left; the options
    # are the C++ SiftExtractionOptions defaults, not Sift()'s
    calls = [line.split() for line in log.read_text().splitlines()]
    assert [int(c[0]) for c in calls] == [31, 9]
    assert all((int(c[1]), float(c[2]), int(c[3]), int(c[4])) == (-1, 0.02 / 3, 3200, 8192) for c in calls)

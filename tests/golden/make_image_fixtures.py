"""Writes the JPEG fixtures of the extraction tests (tests/golden/images/), the grey images Pillow (libjpeg) decodes
from them under FreeImage's Rec709 rule (tests/golden/images/pillow_grey.npz), and a rendered homography pair with
its planted homography.  Run from the repository root:
    python tests/golden/make_image_fixtures.py"""
import io
import os
import sys

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import image_io as O  # noqa: E402
from pycolmap_b200 import synthetic as syn  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "images")


def colour(rng, w, h):
    a, b, _ = syn.homography_pair(rng, w, h, 256)
    return np.stack([a, b, np.roll(a, 5, 1)], -1)


def exif_block():
    from PIL.TiffImagePlugin import IFDRational
    e = Image.Exif()
    ifd = e.get_ifd(0x8769)
    ifd[0x920A] = IFDRational(415, 100)  # FocalLength, mm ("4.2 mm" as FreeImage prints it)
    ifd[0xA002] = 160             # PixelXDimension
    ifd[0xA20E] = IFDRational(160, 3)  # FocalPlaneXResolution: 160 pixels per 3 cm -> a sensor 3 cm wide
    ifd[0xA210] = 3               # FocalPlaneResolutionUnit: cm
    return e.tobytes()


def main():
    os.makedirs(OUT, exist_ok=True)
    rng = np.random.default_rng(11)
    rgb = colour(rng, 160, 120)
    files = {
        "baseline_420.jpg": dict(img=Image.fromarray(rgb), quality=90, subsampling=2),
        "baseline_444.jpg": dict(img=Image.fromarray(rgb), quality=90, subsampling=0),
        "progressive.jpg": dict(img=Image.fromarray(rgb), quality=90, progressive=True),
        "grey.jpg": dict(img=Image.fromarray(O.to_grey(rgb)), quality=90),
        "exif_focal.jpg": dict(img=Image.fromarray(rgb), quality=90, exif=exif_block()),
    }
    grey = {}
    for name, kw in files.items():
        img = kw.pop("img")
        buf = io.BytesIO()
        img.save(buf, "JPEG", **kw)
        with open(os.path.join(OUT, name), "wb") as f:
            f.write(buf.getvalue())
        dec = Image.open(io.BytesIO(buf.getvalue()))
        grey[name] = np.asarray(dec) if dec.mode == "L" else O.to_grey(np.asarray(dec.convert("RGB")))
    np.savez_compressed(os.path.join(OUT, "pillow_grey.npz"), **grey)
    # two rendered views of a plane related by a planted homography (view 0 -> view 1), for the end-to-end test
    a, b, H = syn.homography_pair(np.random.default_rng(21), 1024, 768, 1024)
    for k, img in enumerate((a, b)):
        Image.fromarray(img).save(os.path.join(OUT, f"homography_view{k}.jpg"), quality=95)
    np.save(os.path.join(OUT, "homography_H.npy"), H)


if __name__ == "__main__":
    main()

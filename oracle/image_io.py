"""Test-only numpy restatement of what COLMAP's feature extraction does to an image around SIFT (SURVEY.md rows U1-U6):
FreeImage's grey conversion and bilinear rescale, ImageResizerThread's target size, FeatureKeypoint's 6 columns with
ScaleKeypoints and MaskKeypoints, Bitmap::ExifFocalLength's rules on tag values, and a PNG decoder.  The device path
(pycolmap_b200/csrc/image_io.cu) and the host reader (pycolmap_b200/host/image_reader.cc) are held against it."""
import struct
import zlib

import numpy as np


def to_grey(rgb):
    """FreeImage ConvertToGreyscale: (BYTE)(0.2126f r + 0.7152f g + 0.0722f b + 0.5f), fp32 rounded per operation, in
    that order; alpha ignored.  A 2-D array passes through."""
    rgb = np.asarray(rgb)
    if rgb.ndim == 2:
        return rgb.astype(np.uint8)
    f = rgb[..., :3].astype(np.float32)
    v = np.float32(0.2126) * f[..., 0] + np.float32(0.7152) * f[..., 1]
    v = v + np.float32(0.0722) * f[..., 2]
    return (v + np.float32(0.5)).astype(np.uint8)


def target_size(w, h, max_image_size):
    """ImageResizerThread: (int)(w * s) x (int)(h * s), s = max_image_size / max(w, h), when max(w, h) exceeds it."""
    if w <= max_image_size and h <= max_image_size:
        return w, h
    s = max_image_size / max(w, h)
    return int(w * s), int(h * s)


def bilinear_table(dst, src):
    """CWeightsTable(CBilinearFilter, dst, src): per destination pixel (left, weights), fp64, normalised, null weights
    at the right discarded."""
    scale = dst / src
    width, fscale = (1.0 / scale, scale) if scale < 1.0 else (1.0, 1.0)
    offset = 0.5 / scale
    out = []
    for u in range(dst):
        center = u / scale + offset
        left = max(0, int(center - width + 0.5))
        right = min(int(center + width + 0.5), src)
        w = []
        for s in range(left, right):
            d = abs(fscale * (s + 0.5 - center))
            w.append(fscale * (1.0 - d if d < 1.0 else 0.0))
        total = 0.0
        for v in w:
            total += v
        if total > 0 and total != 1:
            w = [v / total for v in w]
        while right > left and w[right - left - 1] == 0:
            right -= 1
        out.append((left, w[:right - left]))
    return out


def _filter_rows(img, table):
    """horizontalFilter: each row through the table, fp64 sums in weight order, (BYTE)clamp((int)(v + 0.5))."""
    h = img.shape[0]
    out = np.empty((h, len(table)), np.uint8)
    src = img.astype(np.float64)
    for x, (left, w) in enumerate(table):
        v = np.zeros(h, np.float64)
        for k, wk in enumerate(w):
            v = v + wk * src[:, left + k]
        out[:, x] = np.clip((v + 0.5).astype(np.int64), 0, 255)
    return out


def rescale(grey, w_new, h_new):
    """FreeImage_Rescale(FILTER_BILINEAR) of an 8-bit grey image: horizontal pass first when
    dst_w * src_h <= dst_h * src_w, else vertical first; the intermediate is 8-bit."""
    h, w = grey.shape
    tx, ty = bilinear_table(w_new, w), bilinear_table(h_new, h)
    if w_new * h <= h_new * w:
        tmp = _filter_rows(grey, tx)
        return _filter_rows(tmp.T, ty).T.copy()
    tmp = _filter_rows(grey.T, ty).T
    return _filter_rows(tmp, tx)


def keypoints6(kp4, scale_x=None, scale_y=None):
    """FeatureKeypoint(x, y, scale, orientation) -> (x, y, a11, a12, a21, a22), then FeatureKeypoint::Rescale(sx, sy)
    (x, a11, a21 by sx; y, a12, a22 by sy), all fp32."""
    kp4 = np.asarray(kp4, np.float32)
    x, y, s, o = (kp4[:, k] for k in range(4))
    c = s * np.cos(o.astype(np.float64)).astype(np.float32)
    sn = s * np.sin(o.astype(np.float64)).astype(np.float32)
    out = np.stack([x, y, c, -sn, sn, c], 1).astype(np.float32)
    if scale_x is not None:
        sx, sy = np.float32(scale_x), np.float32(scale_y)
        out *= np.array([sx, sy, sx, sy, sx, sy], np.float32)
    return out


def mask_keep(kp6, mask):
    """MaskKeypoints: kept iff the integer pixel ((int)x, (int)y), truncated towards zero as GetPixel's int arguments
    are, is inside the mask and the mask is nonzero there."""
    px, py = np.trunc(kp6[:, 0]).astype(np.int64), np.trunc(kp6[:, 1]).astype(np.int64)
    inside = (px >= 0) & (py >= 0) & (px < mask.shape[1]) & (py < mask.shape[0])
    keep = np.zeros(len(kp6), bool)
    keep[inside] = mask[py[inside], px[inside]] != 0
    return keep


def exif_focal(width, height, f35=None, focal=None, pixel_x_dim=None, focal_plane_x_res=None, unit=None):
    """Bitmap::ExifFocalLength on tag values (rationals as (num, den)); None when it finds no focal length.  FreeImage
    prints FocalLength as "%.1f mm" and COLMAP parses the string back; FocalPlaneXResolution prints as "num/den" unless
    it is an integer, which then does not parse; units 2 = inches, 3 = cm."""
    max_size = float(max(width, height))
    if f35 is not None and f35 > 0:
        return f35 / 35.0 * max_size
    if focal is None or focal[1] == 0:
        return None
    focal_mm = float("%.1f" % (focal[0] / focal[1]))
    if pixel_x_dim is None or focal_plane_x_res is None or unit is None:
        return None
    num, den = focal_plane_x_res
    if num == 0 or den == 0 or num % den == 0:
        return None
    ccd_width = (den / num) * pixel_x_dim
    if not (ccd_width > 0 and focal_mm > 0):
        return None
    if unit == 3:
        return focal_mm / (ccd_width * 10.0) * max_size
    if unit == 2:
        return focal_mm / (ccd_width * 25.4) * max_size
    return None


def decode_png(data):
    """8-bit non-interlaced PNG -> uint8 array (H, W) grey, (H, W, 2) grey + alpha, (H, W, 3) RGB (palette expanded),
    (H, W, 4) RGBA.  Raises ValueError for anything else."""
    if data[:8] != b"\x89PNG\r\n\x1a\n":
        raise ValueError("not a PNG")
    pos, idat, plte, ihdr = 8, b"", None, None
    while pos + 12 <= len(data):
        (n,) = struct.unpack(">I", data[pos:pos + 4])
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        if zlib.crc32(kind + body) != struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0]:
            raise ValueError("bad CRC")
        if kind == b"IHDR":
            ihdr = struct.unpack(">IIBBBBB", body)
        elif kind == b"PLTE":
            plte = np.frombuffer(body, np.uint8).reshape(-1, 3)
        elif kind == b"IDAT":
            idat += body
        elif kind == b"IEND":
            break
        pos += 12 + n
    w, h, depth, ctype, _, _, interlace = ihdr
    if depth != 8 or interlace != 0 or ctype not in (0, 2, 3, 4, 6):
        raise ValueError("unsupported PNG")
    spp = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype]
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, w * spp + 1)
    out = np.zeros((h, w * spp), np.int32)
    for y in range(h):
        f, s = raw[y, 0], raw[y, 1:].astype(np.int32)
        up = out[y - 1] if y else np.zeros(w * spp, np.int32)
        row = out[y]
        for x in range(w * spp):
            a = row[x - spp] if x >= spp else 0
            b = up[x]
            c = up[x - spp] if x >= spp else 0
            if f == 0:
                p = 0
            elif f == 1:
                p = a
            elif f == 2:
                p = b
            elif f == 3:
                p = (a + b) >> 1
            elif f == 4:
                q = a + b - c
                pa, pb, pc = abs(q - a), abs(q - b), abs(q - c)
                p = a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)
            else:
                raise ValueError("bad filter")
            row[x] = (s[x] + p) & 255
    img = out.astype(np.uint8).reshape(h, w, spp)
    if ctype == 3:
        return plte[img[..., 0]]
    return img[..., 0] if spp == 1 else img

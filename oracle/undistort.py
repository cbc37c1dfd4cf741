"""Test-only numpy (fp64) restatement of COLMAP's image undistortion, the specification K10 (csrc/undistort.cu) is held
to.  Recalled from upstream COLMAP 3.9.1 (its source is not part of the reference), DESIGN.md section 4 K10:

  undistort_camera   <- U:image/undistortion.cc UndistortCamera, Camera::Rescale(scale)
  warp               <- U:image/warp.cc WarpImageBetweenCameras, U:sensor/bitmap.cc Bitmap::InterpolateBilinear,
                        BitmapColor<float>::Cast<uint8_t>, Bitmap::Rescale (FreeImage FILTER_BILINEAR)
  undistort_points   <- U:image/undistortion.cc UndistortReconstruction (the 2-D points)

Camera models are oracle/ransac.py's; the polynomial models' ImgFromCam is restated here in the operation order of
csrc/camera_models.h, so that the warp's coordinate map is the device's bit for bit.  The rescale is
oracle/image_io.py's, per channel.
"""
import numpy as np

from . import image_io as IO
from . import ransac as R

PINHOLE = 1
DEFAULTS = dict(blank_pixels=0.0, min_scale=0.2, max_scale=2.0, max_image_size=-1, roi_min_x=0.0, roi_min_y=0.0,
                roi_max_x=1.0, roi_max_y=1.0)


def check_options(o):
    """UndistortCameraOptions' checks, in upstream's order; ValueError names the failed one."""
    for ok, expr in ((o["blank_pixels"] >= 0, "blank_pixels >= 0"), (o["blank_pixels"] <= 1, "blank_pixels <= 1"),
                     (o["min_scale"] > 0, "min_scale > 0"), (o["min_scale"] <= o["max_scale"], "min_scale <= max_scale"),
                     (o["max_image_size"] != 0, "max_image_size != 0"),
                     (o["roi_min_x"] >= 0, "roi_min_x >= 0"), (o["roi_min_y"] >= 0, "roi_min_y >= 0"),
                     (o["roi_max_x"] <= 1, "roi_max_x <= 1"), (o["roi_max_y"] <= 1, "roi_max_y <= 1"),
                     (o["roi_min_x"] < o["roi_max_x"], "roi_min_x < roi_max_x"),
                     (o["roi_min_y"] < o["roi_max_y"], "roi_min_y < roi_max_y")):
        if not ok:
            raise ValueError(f"Check Failed: {expr}")


def _intr(cam):
    model, f, c, k = R._intrinsics(cam)
    return model, f[0], f[1], c[0], c[1], k


def img_from_cam(cam, u, v):
    """Camera::ImgFromCam on arrays of normalised coordinates.  The pinhole and polynomial models (0-4, 6) follow the
    operation order of csrc/camera_models.h; the models with atan / tan go through oracle/ransac.py."""
    model, fx, fy, cx, cy, k = _intr(cam)
    u = np.asarray(u, np.float64)
    v = np.asarray(v, np.float64)
    if model in (5, 7, 8, 9, 10):
        xy = R.img_from_cam(cam, np.stack([u.ravel(), v.ravel()], 1))
        return xy[:, 0].reshape(u.shape), xy[:, 1].reshape(u.shape)
    du = dv = 0.0
    if model != 0 and model != 1:
        u2, v2 = u * u, v * v
        r2 = u2 + v2
        if model == 2:
            radial = k[0] * r2
            du, dv = u * radial, v * radial
        elif model == 3:
            radial = k[0] * r2 + k[1] * r2 * r2
            du, dv = u * radial, v * radial
        elif model == 4:
            uv = u * v
            radial = k[0] * r2 + k[1] * r2 * r2
            du = u * radial + 2.0 * k[2] * uv + k[3] * (r2 + 2.0 * u2)
            dv = v * radial + 2.0 * k[3] * uv + k[2] * (r2 + 2.0 * v2)
        else:  # FULL_OPENCV
            uv, r4 = u * v, r2 * r2
            r6 = r4 * r2
            radial = (1.0 + k[0] * r2 + k[1] * r4 + k[4] * r6) / (1.0 + k[5] * r2 + k[6] * r4 + k[7] * r6)
            du = u * radial + 2.0 * k[2] * uv + k[3] * (r2 + 2.0 * u2) - u
            dv = v * radial + 2.0 * k[3] * uv + k[2] * (r2 + 2.0 * v2) - v
    return fx * (u + du) + cx, fy * (v + dv) + cy


def _pinhole(fx, fy, cx, cy, width, height):
    return dict(model=PINHOLE, width=int(width), height=int(height), params=[fx, fy, cx, cy])


def rescale_camera(cam, scale):
    """Camera::Rescale(scale) of a PINHOLE camera: size round(scale * size), parameters by the per-axis ratio the
    rounding gives."""
    fx, fy, cx, cy = cam["params"]
    w, h = cam["width"], cam["height"]
    sx = round(scale * w) / w
    sy = round(scale * h) / h
    return _pinhole(sx * fx, sy * fy, sx * cx, sy * cy, round(scale * w), round(scale * h))


def undistort_camera(options, cam):
    """UndistortCamera: the PINHOLE camera of the undistorted image (dict(model, width, height, params))."""
    o = dict(DEFAULTS, **(options or {}))
    check_options(o)
    model, fx, fy, cx, cy, _ = _intr(cam)
    W, H = int(cam["width"]), int(cam["height"])
    ux, uy, w, h = cx, cy, W, H
    rx0, ry0, rx1, ry1 = 0, 0, W, H
    roi = o["roi_min_x"] > 0 or o["roi_min_y"] > 0 or o["roi_max_x"] < 1 or o["roi_max_y"] < 1
    if roi:
        rx0, ry0 = int(round(o["roi_min_x"] * w)), int(round(o["roi_min_y"] * h))
        rx1, ry1 = int(round(o["roi_max_x"] * w)), int(round(o["roi_max_y"] * h))
        rx0, ry0 = min(rx0, w - 1), min(ry0, h - 1)
        rx1, ry1 = max(rx1, rx0 + 1), max(ry1, ry0 + 1)
        w, h = rx1 - rx0, ry1 - ry0
        ux, uy = ux - rx0, uy - ry0
    if roi or model not in (0, 1):
        ys = np.arange(ry0, ry1) + 0.5
        xs = np.arange(rx0, rx1) + 0.5

        def proj(px, py):  # distorted CamFromImg, then the undistorted pinhole ImgFromCam
            uv = R.cam_from_img(cam, np.stack([px, py], 1))
            return fx * uv[:, 0] + ux, fy * uv[:, 1] + uy

        left = proj(np.full(len(ys), 0.5), ys)[0]
        right = proj(np.full(len(ys), W - 0.5), ys)[0]
        top = proj(xs, np.full(len(xs), 0.5))[1]
        bottom = proj(xs, np.full(len(xs), H - 0.5))[1]
        min_sx = min(ux / (ux - left.min()), (w - 0.5 - ux) / (right.max() - ux))
        min_sy = min(uy / (uy - top.min()), (h - 0.5 - uy) / (bottom.max() - uy))
        max_sx = max(ux / (ux - left.max()), (w - 0.5 - ux) / (right.min() - ux))
        max_sy = max(uy / (uy - top.max()), (h - 0.5 - uy) / (bottom.min() - uy))
        b = o["blank_pixels"]
        sx = min(max(1.0 / (min_sx * b + max_sx * (1.0 - b)), o["min_scale"]), o["max_scale"])
        sy = min(max(1.0 / (min_sy * b + max_sy * (1.0 - b)), o["min_scale"]), o["max_scale"])
        w0, h0 = w, h
        w, h = int(max(1.0, sx * w)), int(max(1.0, sy * h))
        ux = ux * float(w) / float(w0)
        uy = uy * float(h) / float(h0)
    out = _pinhole(fx, fy, ux, uy, w, h)
    if o["max_image_size"] > 0:
        s = min(o["max_image_size"] / float(w), o["max_image_size"] / float(h))
        if s < 1.0:
            out = rescale_camera(out, s)
    return out


def to_rgb(img):
    """The 24-bit RGB bitmap Bitmap::Read(path, as_rgb=true) makes: grey replicated, alpha dropped."""
    img = np.asarray(img, np.uint8)
    if img.ndim == 2:
        img = img[:, :, None]
    if img.shape[2] == 1:
        return np.repeat(img, 3, 2)
    return np.ascontiguousarray(img[:, :, :3])


def interpolate_bilinear(img, x, y):
    """Bitmap::InterpolateBilinear on an (H, W, 3) uint8 image at arrays x, y: fp64 on FreeImage's bottom-up scan lines
    (line y0 is image row H - 1 - y0), then BitmapColor<float> and Cast<uint8_t> (rounded half away from zero,
    clamped).  Outside (x0 < 0, x0 + 1 >= W, y0 < 0, y0 + 1 >= H, or NaN): black."""
    H, W = img.shape[:2]
    inv_y = float(H - 1) - y
    with np.errstate(invalid="ignore"):
        fx0, fy0 = np.floor(x), np.floor(inv_y)
        ok = (fx0 >= 0) & (fx0 + 1 < W) & (fy0 >= 0) & (fy0 + 1 < H)
    x0 = np.where(ok, fx0, 0).astype(np.int64)
    y0 = np.where(ok, fy0, 0).astype(np.int64)
    dx, dy = x - x0, inv_y - y0
    dx_1, dy_1 = 1.0 - dx, 1.0 - dy
    r0 = H - 1 - y0
    r1 = np.maximum(r0 - 1, 0)
    x1 = np.minimum(x0 + 1, W - 1)
    out = np.zeros(x.shape + (3,), np.uint8)
    for c in range(3):
        p = img[:, :, c].astype(np.float64)
        v0 = dx_1 * p[r0, x0] + dx * p[r0, x1]
        v1 = dx_1 * p[r1, x0] + dx * p[r1, x1]
        f = (dy_1 * v0 + dy * v1).astype(np.float32).astype(np.float64)
        val = np.clip(np.floor(f + 0.5), 0, 255)  # std::round of a non-negative value
        out[..., c] = np.where(ok, val, 0).astype(np.uint8)
    return out


def warp(img, distorted, undistorted):
    """WarpImageBetweenCameras(distorted, undistorted) of an image read as RGB: warped at the source size with the
    target camera rescaled to it (Camera::Rescale(w, h)), then Bitmap::Rescale to the undistorted size."""
    rgb = to_rgb(img)
    H, W = rgb.shape[:2]
    if (W, H) != (distorted["width"], distorted["height"]):
        raise ValueError(f"image {W} x {H} is not its camera's size")
    fx, fy, cx, cy = undistorted["params"]
    uw, uh = undistorted["width"], undistorted["height"]
    if (uw, uh) != (W, H):
        sx, sy = float(W) / float(uw), float(H) / float(uh)
        fx, fy, cx, cy = sx * fx, sy * fy, sx * cx, sy * cy
    ys, xs = np.mgrid[0:H, 0:W]
    u = (xs + 0.5 - cx) / fx
    v = (ys + 0.5 - cy) / fy
    sx_, sy_ = img_from_cam(distorted, u, v)
    out = interpolate_bilinear(rgb, sx_ - 0.5, sy_ - 0.5)
    if (uw, uh) != (W, H):
        out = np.stack([IO.rescale(out[:, :, c], uw, uh) for c in range(3)], -1)
    return out


def undistort_image(options, img, distorted):
    """UndistortImage: (undistorted RGB image, undistorted camera)."""
    und = undistort_camera(options, distorted)
    return warp(img, distorted, und), und


def undistort_points(distorted, undistorted, xy):
    """UndistortReconstruction's 2-D points: undistorted.ImgFromCam(distorted.CamFromImg(xy))."""
    uv = R.cam_from_img(distorted, np.asarray(xy, np.float64).reshape(-1, 2))
    fx, fy, cx, cy = undistorted["params"]
    return np.stack([fx * uv[:, 0] + cx, fy * uv[:, 1] + cy], 1)


def is_undistorted(cam):
    """Camera::IsUndistorted: every extra (distortion) parameter within 1e-8 of zero."""
    _, _, _, _, _, k = _intr(cam)
    return all(abs(v) <= 1e-8 for v in k)


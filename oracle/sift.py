"""Numpy restatement of SIFT feature extraction as COLMAP 3.9.1's SiftCPUFeatureExtractor computes it (VLFeat's
vl_sift on the non-covariant path; SURVEY.md rows X1-X8).  It is the specification the GPU extractor
(csrc/sift.cu) is held to, not a CPU baseline.

Arithmetic follows VLFeat's types: the pyramid, gradients and descriptor histograms in fp32, the keypoint refinement,
orientation histogram and Gaussian table in fp64, with float and double mixed where VLFeat mixes them.  Every fp32
sum is accumulated in VLFeat's order.  np.float32 arithmetic has no fused multiply-add, which matches VLFeat built for
plain x86-64.

extract(image, opts) -> dict(keypoints [N x 4] (x, y, scale, orientation), descriptors [N x 128] uint8, octave, level,
margin) in COLMAP's output order."""
import math

import numpy as np

f32 = np.float32
EPS_F = f32(1.19209290e-07)
TWO_PI_F = f32(2 * math.pi)
EXPN_SZ, EXPN_MAX = 256, 25.0
# the table of VLFeat's fast_expn, with libm's exp like VLFeat (math.exp, not numpy's SIMD exp)
EXPN_TAB = np.array([math.exp(-k * (EXPN_MAX / EXPN_SZ)) for k in range(EXPN_SZ + 1)] + [0.0])
UBC_Q = np.array([0, 7, 6, 5, 4, 3, 2, 1])


def defaults(**kw):
    """SiftExtractionOptions' C++ defaults (U:feature/sift.h), overridden by `kw`."""
    o = dict(max_image_size=3200, max_num_features=8192, first_octave=-1, num_octaves=4, octave_resolution=3,
             peak_threshold=0.02 / 3, edge_threshold=10.0, max_num_orientations=2, upright=False, normalization="L1_ROOT")
    o.update(kw)
    return o


def pycolmap_defaults(**kw):
    """pycolmap.Sift()'s defaults (R:pycolmap/feature/sift.h:99-102)."""
    return defaults(**{"peak_threshold": 0.01, "first_octave": 0, "max_image_size": 7000, **kw})


# ---- VLFeat's fast math (X6) -------------------------------------------------------------------------------------
def fast_expn(x):
    """exp(-x) from a 257-entry table with linear interpolation, 0 above 25 (fp64)."""
    x = np.asarray(x, np.float64)
    out = np.zeros(x.shape)
    m = x <= EXPN_MAX
    xs = x[m] * (EXPN_SZ / EXPN_MAX)
    i = np.floor(xs).astype(np.int64)
    r = xs - i
    a, b = EXPN_TAB[i], EXPN_TAB[i + 1]
    out[m] = a + r * (b - a)
    return out


def fast_atan2_f(y, x):
    """vl_fast_atan2_f: a cubic in r, |error| < 6.5e-3 rad (fp32)."""
    y = np.asarray(y, f32)
    x = np.asarray(x, f32)
    ay = np.abs(y) + EPS_F
    pos = x >= 0
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(pos, (x - ay) / (x + ay), (x + ay) / (ay - x)).astype(f32)
    ang = np.where(pos, f32(math.pi / 4), f32(3 * math.pi / 4)).astype(f32)
    ang = (ang + ((f32(0.1821) * r * r - f32(0.9675)) * r)).astype(f32)
    return np.where(y < 0, -ang, ang).astype(f32)


def fast_sqrt_f(x):
    """vl_fast_sqrt_f: x * (two Newton steps of the 0x5f3759df inverse square root), 0 below 1e-8 (fp32)."""
    x = np.asarray(x, f32)
    xhalf = f32(0.5) * x
    i = np.int32(0x5F3759DF) - (x.view(np.int32) >> 1)
    y = i.view(f32)
    y = y * (f32(1.5) - xhalf * y * y)
    y = y * (f32(1.5) - xhalf * y * y)
    return np.where(x.astype(np.float64) < 1e-8, f32(0), x * y).astype(f32)


def mod_2pi_f(x):
    """vl_mod_2pi_f on fp32 values."""
    x = np.asarray(x, f32).copy()
    for _ in range(4):
        x = np.where(x > TWO_PI_F, x - TWO_PI_F, x).astype(f32)
        x = np.where(x < 0, x + TWO_PI_F, x).astype(f32)
    return x


# ---- scale space (X2) ---------------------------------------------------------------------------------------------
def gauss_filter(sigma):
    """_vl_sift_smooth's normalised kernel: half-width max(ceil(4 sigma), 1), fp32 taps."""
    W = max(int(math.ceil(4.0 * sigma)), 1)
    d = (np.arange(2 * W + 1) - W).astype(f32) / f32(sigma)
    g = np.array([math.exp(-0.5 * float(v)) for v in (d * d)], dtype=f32)
    acc = f32(0)
    for v in g:
        acc = f32(acc + v)
    return (g / acc).astype(f32)


def _conv_axis0(img, g):
    """Sum over the taps in VLFeat's order with a replicated border, along axis 0 (fp32 product, then fp32 add)."""
    W = (len(g) - 1) // 2
    h = img.shape[0]
    idx = np.arange(h)
    acc = np.zeros(img.shape, f32)
    for k in range(2 * W + 1):
        acc = (acc + img[np.clip(idx - W + k, 0, h - 1)] * g[k]).astype(f32)
    return acc


def smooth(img, sigma):
    """vl_imconvcol_vf twice: along y first, then along x."""
    g = gauss_filter(sigma)
    return _conv_axis0(_conv_axis0(img, g).T, g).T.copy()


def _upsample_rows(a):
    """copy_and_upsample_rows without its transpose: [h, w] -> [h, 2w]."""
    h, w = a.shape
    out = np.empty((h, 2 * w), f32)
    out[:, 0::2] = a
    out[:, 1::2] = ((a + a[:, np.minimum(np.arange(w) + 1, w - 1)]) * f32(0.5)).astype(f32)
    return out


def octave_dims(W, H, o):
    return (W << -o, H << -o) if o < 0 else (W >> o, H >> o)


def sigma_constants(S):
    sigmak = 2.0 ** (1.0 / S)
    sigma0 = 1.6 * sigmak
    dsigma0 = sigma0 * math.sqrt(1.0 - 1.0 / (sigmak * sigmak))
    return sigmak, sigma0, dsigma0


def first_level_sigma(S, o_min):
    sigmak, sigma0, _ = sigma_constants(S)
    sa, sb = sigma0 * sigmak ** -1, 0.5 * 2.0 ** (-o_min)
    return math.sqrt(sa * sa - sb * sb) / 2.0 ** o_min if sa > sb else 0.0


def level_sigma(S, s):
    sigmak, _, dsigma0 = sigma_constants(S)
    return dsigma0 * sigmak ** s


def octaves(image_f, opts):
    """Yields (o, gaussian levels s = -1 .. S + 1 as [S + 3, h, w]) per octave with at least 3 x 3 samples."""
    S, o_min, O = opts["octave_resolution"], opts["first_octave"], opts["num_octaves"]
    H, W = image_f.shape
    if o_min < 0:
        base = image_f
        for _ in range(-o_min):
            base = _upsample_rows(_upsample_rows(base).T).T.copy()
    else:
        d = 1 << o_min
        base = image_f[::d, ::d][: H >> o_min, : W >> o_min].copy()
    s1 = first_level_sigma(S, o_min)
    if s1 > 0:
        base = smooth(base, s1)
    for o in range(o_min, o_min + O):
        w, h = octave_dims(W, H, o)
        if w < 3 or h < 3:
            return
        if o > o_min:
            base = G[S][::2, ::2][:h, :w].copy()  # level S - 1 (index S from s = -1); sa == sb: no smoothing
        G = [base]
        for s in range(0, S + 2):
            G.append(smooth(G[-1], level_sigma(S, s)))
        yield o, np.stack(G)


# ---- detection and refinement (X3) -------------------------------------------------------------------------------
def detect(dog, o, opts):
    """Candidates in VLFeat's scan order (level, y, x), refined; returns keypoint dicts of this octave."""
    S = opts["octave_resolution"]
    pt, et = float(opts["peak_threshold"]), float(opts["edge_threshold"])
    nL, h, w = dog.shape  # levels s = -1 .. S
    c = dog[1:S + 1, 1:h - 1, 1:w - 1]
    cd = c.astype(np.float64)
    is_max = cd >= 0.8 * pt
    is_min = cd <= -0.8 * pt
    for ds in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                if ds == dy == dx == 0:
                    continue
                n = dog[1 + ds:S + 1 + ds, 1 + dy:h - 1 + dy, 1 + dx:w - 1 + dx]
                is_max &= c > n
                is_min &= c < n
    out = []
    xper = 2.0 ** o
    sigmak, sigma0, _ = sigma_constants(S)
    for (si, yi, xi) in np.argwhere(is_max | is_min):
        k = refine(dog, int(xi) + 1, int(yi) + 1, int(si), w, h, S, pt, et)
        if k is None:
            continue
        x, y, s, sn, b, margin = k
        # extremum margin: the closest of the 26 neighbours and the 0.8 peak threshold
        v = float(dog[si + 1, yi + 1, xi + 1])
        nb = dog[si:si + 3, yi:yi + 3, xi:xi + 3].astype(np.float64).ravel()
        nb = np.delete(nb, 13)
        ext = min(np.min(np.abs(v - nb)), abs(abs(v) - 0.8 * pt)) / max(abs(v), 1e-30)
        out.append(dict(o=o, ix=x, iy=y, is_=s, x=f32((x + b[0]) * xper), y=f32((y + b[1]) * xper),
                        s=f32(sn), sigma=f32(sigma0 * 2.0 ** (sn / S) * xper), margin=min(margin, ext)))
    return out


def refine(dog, x, y, s, w, h, S, pt, et):
    """VLFeat's refinement loop (up to 5 quadratic fits, one-pixel steps while |offset| > 0.6), fp64 with fp32
    differences where VLFeat subtracts floats.  `s` indexes DoG levels from s_min + 1 = 0, i.e. dog[s + 1]."""
    def at(dx, dy, ds):
        return dog[s + 1 + ds, y + dy, x + dx]

    dx = dy = 0
    step_margin = math.inf
    for _ in range(5):
        x += dx
        y += dy
        Dx = 0.5 * float(at(1, 0, 0) - at(-1, 0, 0))
        Dy = 0.5 * float(at(0, 1, 0) - at(0, -1, 0))
        Ds = 0.5 * float(at(0, 0, 1) - at(0, 0, -1))
        Dxx = float(at(1, 0, 0) + at(-1, 0, 0)) - 2.0 * float(at(0, 0, 0))
        Dyy = float(at(0, 1, 0) + at(0, -1, 0)) - 2.0 * float(at(0, 0, 0))
        Dss = float(at(0, 0, 1) + at(0, 0, -1)) - 2.0 * float(at(0, 0, 0))
        Dxy = 0.25 * float(at(1, 1, 0) + at(-1, -1, 0) - at(-1, 1, 0) - at(1, -1, 0))
        Dxs = 0.25 * float(at(1, 0, 1) + at(-1, 0, -1) - at(-1, 0, 1) - at(1, 0, -1))
        Dys = 0.25 * float(at(0, 1, 1) + at(0, -1, -1) - at(0, -1, 1) - at(0, 1, -1))
        b = solve3([[Dxx, Dxy, Dxs], [Dxy, Dyy, Dys], [Dxs, Dys, Dss]], [-Dx, -Dy, -Ds])
        step_margin = min(step_margin, abs(abs(b[0]) - 0.6), abs(abs(b[1]) - 0.6))
        dx = (1 if (b[0] > 0.6 and x < w - 2) else 0) + (-1 if (b[0] < -0.6 and x > 1) else 0)
        dy = (1 if (b[1] > 0.6 and y < h - 2) else 0) + (-1 if (b[1] < -0.6 and y > 1) else 0)
        if dx == 0 and dy == 0:
            break
    val = float(at(0, 0, 0)) + 0.5 * (Dx * b[0] + Dy * b[1] + Ds * b[2])
    det = Dxx * Dyy - Dxy * Dxy
    tr2 = (Dxx + Dyy) * (Dxx + Dyy)
    score = tr2 / det if det != 0 else (math.inf if tr2 > 0 else math.nan)
    thr = (et + 1) * (et + 1) / et
    xn, yn, sn = x + b[0], y + b[1], (s) + b[2]
    good = (abs(val) > pt and score < thr and score >= 0 and abs(b[0]) < 1.5 and abs(b[1]) < 1.5 and abs(b[2]) < 1.5
            and 0 <= xn <= w - 1 and 0 <= yn <= h - 1 and -1 <= sn <= S + 1)
    if not good:
        return None
    margin = min(abs(abs(val) - pt) / pt, abs(score - thr) / thr if math.isfinite(score) else math.inf, step_margin)
    return x, y, s, sn, b, margin


def solve3(A, b):
    """VLFeat's Gauss elimination with partial pivoting; a pivot below 1e-10f gives b = 0."""
    A = [row[:] for row in A]
    b = b[:]
    tiny = float(f32(1e-10))
    for j in range(3):
        maxa = maxabsa = 0.0
        maxi = -1
        for i in range(j, 3):
            a = A[i][j]
            if abs(a) > maxabsa:
                maxa, maxabsa, maxi = a, abs(a), i
        if maxabsa < tiny:
            b = [0.0, 0.0, 0.0]
            break
        i = maxi
        for jj in range(j, 3):
            A[i][jj], A[j][jj] = A[j][jj], A[i][jj]
            A[j][jj] /= maxa
        b[j], b[i] = b[i], b[j]
        b[j] /= maxa
        for ii in range(j + 1, 3):
            xx = A[ii][j]
            for jj in range(j, 3):
                A[ii][jj] -= xx * A[j][jj]
            b[ii] -= xx * b[j]
    for i in range(2, 0, -1):
        xx = b[i]
        for ii in range(i - 1, -1, -1):
            b[ii] -= xx * A[ii][i]
    return b


# ---- gradients, orientation (X4) and descriptor (X5) --------------------------------------------------------------
def gradients(G, S):
    """update_gradient: (modulus, angle in [0, 2 pi]) of levels s = 0 .. S - 1, fp32, one-sided at the border."""
    out = []
    for s in range(S):
        L = G[s + 1]
        gx = np.empty_like(L)
        gy = np.empty_like(L)
        gx[:, 1:-1] = f32(0.5) * (L[:, 2:] - L[:, :-2])
        gx[:, 0] = L[:, 1] - L[:, 0]
        gx[:, -1] = L[:, -1] - L[:, -2]
        gy[1:-1] = f32(0.5) * (L[2:] - L[:-2])
        gy[0] = L[1] - L[0]
        gy[-1] = L[-1] - L[-2]
        mod = fast_sqrt_f((gx * gx + gy * gy).astype(f32))
        ang = mod_2pi_f((fast_atan2_f(gy, gx).astype(np.float64) + 2 * math.pi).astype(f32))
        out.append((mod, ang))
    return out


def orientations(grad, k, o, w, h, margins=None):
    """vl_sift_calc_keypoint_orientations with bilinear binning: up to 4 angles in bin order, fp64."""
    xper = 2.0 ** o
    x, y, sigma = float(k["x"]) / xper, float(k["y"]) / xper, float(k["sigma"]) / xper
    xi, yi, si = int(x + 0.5), int(y + 0.5), k["is_"]
    sigmaw = 1.5 * sigma
    W = int(max(math.floor(3.0 * sigmaw), 1))
    if xi < 0 or xi > w - 1 or yi < 0 or yi > h - 1:
        return []
    mod, ang = grad[si]
    ys = np.arange(max(-W, -yi), min(W, h - 1 - yi) + 1)
    xs = np.arange(max(-W, -xi), min(W, w - 1 - xi) + 1)
    YS, XS = np.meshgrid(ys, xs, indexing="ij")
    dx = (xi + XS).astype(np.float64) - x
    dy = (yi + YS).astype(np.float64) - y
    r2 = dx * dx + dy * dy
    m = r2 < W * W + 0.6
    wgt = fast_expn(r2[m] / (2 * sigmaw * sigmaw))
    md = mod[yi + YS[m], xi + XS[m]].astype(np.float64)
    fbin = 36 * ang[yi + YS[m], xi + XS[m]].astype(np.float64) / (2 * math.pi)
    b = np.floor(fbin - 0.5).astype(np.int64)
    rbin = fbin - b - 0.5
    idx = np.stack([(b + 36) % 36, (b + 1) % 36], 1).ravel()
    val = np.stack([(1 - rbin) * md * wgt, rbin * md * wgt], 1).ravel()
    hist = np.zeros(36)
    np.add.at(hist, idx, val)
    for _ in range(6):
        prev, first = hist[35], hist[0]
        for i in range(35):
            newh = (prev + hist[i] + hist[i + 1]) / 3.0
            prev = hist[i]
            hist[i] = newh
        hist[35] = (prev + hist[35] + first) / 3.0
    maxh = max(0.0, hist.max())
    angles = []
    pm = math.inf
    for i in range(36):
        h0, hm, hp = hist[i], hist[(i - 1) % 36], hist[(i + 1) % 36]
        if h0 > hm and h0 > hp:
            pm = min(pm, abs(h0 - 0.8 * maxh) / max(maxh, 1e-300))
        if h0 > 0.8 * maxh and h0 > hm and h0 > hp:
            di = -0.5 * (hp - hm) / (hp + hm - 2 * h0)
            angles.append(2 * math.pi * (i + di + 0.5) / 36)
            if len(angles) == 4:
                break
    if margins is not None:
        margins.append(pm)
    return angles


def descriptor(grad, k, o, w, h, angle0):
    """vl_sift_calc_keypoint_descriptor: 4 x 4 x 8 float histogram (VLFeat layout), L2-normalised, clamped at 0.2,
    renormalised.  All-zero when VLFeat's bounds check skips the keypoint."""
    xper = 2.0 ** o
    x, y, sigma = float(k["x"]) / xper, float(k["y"]) / xper, float(k["sigma"]) / xper
    xi, yi, si = int(x + 0.5), int(y + 0.5), k["is_"]
    st0, ct0 = math.sin(angle0), math.cos(angle0)
    SBP = 3.0 * sigma + 2.220446049250313e-16
    W = int(math.floor(math.sqrt(2.0) * SBP * 5 / 2.0 + 0.5))
    desc = np.zeros(128, f32)
    if xi < 0 or xi >= w or yi < 0 or yi >= h - 1:
        return desc
    mod, ang = grad[si]
    ys = np.arange(max(-W, 1 - yi), min(W, h - yi - 2) + 1)
    xs = np.arange(max(-W, 1 - xi), min(W, w - xi - 2) + 1)
    if len(ys) and len(xs):
        YS, XS = np.meshgrid(ys, xs, indexing="ij")
        YS, XS = YS.ravel(), XS.ravel()
        md = mod[yi + YS, xi + XS]
        th = mod_2pi_f((ang[yi + YS, xi + XS].astype(np.float64) - angle0).astype(f32))
        dx = ((xi + XS).astype(np.float64) - x).astype(f32).astype(np.float64)
        dy = ((yi + YS).astype(np.float64) - y).astype(f32).astype(np.float64)
        nx = ((ct0 * dx + st0 * dy) / SBP).astype(f32)
        ny = ((-st0 * dx + ct0 * dy) / SBP).astype(f32)
        nt = (8.0 * th.astype(np.float64) / (2 * math.pi)).astype(f32)
        win = fast_expn((nx * nx + ny * ny).astype(f32).astype(np.float64) / 8.0).astype(f32)
        binx = np.floor((nx.astype(np.float64) - 0.5).astype(f32)).astype(np.int64)
        biny = np.floor((ny.astype(np.float64) - 0.5).astype(f32)).astype(np.int64)
        bint = np.floor(nt).astype(np.int64)
        rbinx = (nx.astype(np.float64) - (binx + 0.5)).astype(f32)
        rbiny = (ny.astype(np.float64) - (biny + 0.5)).astype(f32)
        rbint = (nt - bint.astype(f32)).astype(f32)
        wm = (win * md).astype(f32)
        idx, val = [], []
        for dbx in (0, 1):
            for dby in (0, 1):
                for dbt in (0, 1):
                    ok = (binx + dbx >= -2) & (binx + dbx < 2) & (biny + dby >= -2) & (biny + dby < 2)
                    wt = (wm * np.abs(f32(1 - dbx) - rbinx) * np.abs(f32(1 - dby) - rbiny)
                          * np.abs(f32(1 - dbt) - rbint)).astype(f32)
                    i = (biny + dby + 2) * 32 + (binx + dbx + 2) * 8 + (bint + dbt) % 8
                    idx.append(np.where(ok, i, -1))
                    val.append(wt)
        idx = np.stack(idx, 1).ravel()
        val = np.stack(val, 1).ravel()
        keep = idx >= 0
        np.add.at(desc, idx[keep], val[keep])
    _normalize(desc)
    desc[desc.astype(np.float64) > 0.2] = f32(0.2)
    _normalize(desc)
    return desc


def _normalize(d):
    n = f32(0)
    for v in d:
        n = f32(n + v * v)
    n = f32(fast_sqrt_f(n) + EPS_F)
    d /= n


def to_u8(desc, normalization):
    """COLMAP's L1_ROOT (L1-normalise, sqrt) or L2, then min(255, round(512 x)), then the VLFeat -> UBC layout."""
    d = desc.astype(f32)
    if normalization == "L1_ROOT":
        s = f32(0)
        for v in np.abs(d):
            s = f32(s + v)
        d = np.sqrt((d / s).astype(f32)).astype(f32)
    else:
        s = f32(0)
        for v in d:
            s = f32(s + v * v)
        d = (d / np.sqrt(s)).astype(f32) if s > 0 else d
    v = (f32(512) * d).astype(f32)
    r = np.trunc(v)
    r = r + ((v - r) >= 0.5)
    u8 = np.minimum(r, 255).astype(np.uint8)
    out = np.empty_like(u8)
    for c in range(16):
        out[8 * c + UBC_Q] = u8[8 * c: 8 * c + 8]
    return out


# ---- the whole extractor (X7, X8) ---------------------------------------------------------------------------------
def image_to_float(image):
    """uint8 -> float / 255; float32 -> (x * 255) truncated to uint8 first (R:pycolmap/feature/sift.h:82-85)."""
    if image.dtype == np.float32:
        image = (image * f32(255)).astype(np.uint8)
    return (image.astype(f32) / f32(255)).astype(f32)


def extract(image, opts=None):
    opts = defaults() if opts is None else opts
    S = opts["octave_resolution"]
    img = image_to_float(np.asarray(image))
    levels = []  # per (octave, level) run: list of keypoints (with their octave's gradients)
    grads = {}
    for o, G in octaves(img, opts):
        dog = (G[1:] - G[:-1]).astype(f32)
        kps = detect(dog, o, opts)
        if not kps:
            continue
        grads[o] = (gradients(G, S), G.shape[2], G.shape[1])
        for k in kps:
            if not levels or levels[-1][0] != (o, k["is_"]):
                levels.append(((o, k["is_"]), []))
            levels[-1][1].append(k)
    # max_num_features: keep levels from the coarsest down; the level that passes the limit is kept whole
    first, n = 0, 0
    for i in range(len(levels) - 1, -1, -1):
        n += len(levels[i][1])
        if n > opts["max_num_features"]:
            first = i
            break
    kp_out, desc_out, octv, lev, marg = [], [], [], [], []
    for _, ks in levels[first:]:
        for k in ks:
            o = k["o"]
            grad, w, h = grads[o]
            om = []
            angles = [0.0] if opts["upright"] else orientations(grad, k, o, w, h, om)
            m = min(k["margin"], om[0]) if om else k["margin"]
            for a in angles[:opts["max_num_orientations"]]:
                af = f32(a)
                sc = f32(k["sigma"])
                a11, a21 = f32(sc * np.cos(af)), f32(sc * np.sin(af))
                a12, a22 = f32(-sc * np.sin(af)), f32(sc * np.cos(af))
                scale = f32((np.sqrt(f32(a11 * a11 + a21 * a21)) + np.sqrt(f32(a12 * a12 + a22 * a22))) / f32(2))
                kp_out.append([f32(k["x"] + f32(0.5)), f32(k["y"] + f32(0.5)), scale, np.arctan2(a21, a11)])
                desc_out.append(to_u8(descriptor(grad, k, o, w, h, a), opts["normalization"]))
                octv.append(o)
                lev.append(k["is_"])
                marg.append(m)
    return dict(keypoints=np.array(kp_out, f32).reshape(-1, 4), descriptors=np.array(desc_out, np.uint8).reshape(-1, 128),
                octave=np.array(octv, np.int32), level=np.array(lev, np.int32), margin=np.array(marg))

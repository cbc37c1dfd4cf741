"""Numpy (float32) restatement of K8, the PatchMatch stereo kernels of pycolmap_b200/csrc/patch_match.cu.

It restates the schedule the device runs -- start hypotheses, four sweeps per iteration (down, up, right, left), the
backward and forward messages of the visibility chain along each sweep, the candidate set (current, propagated, random,
perturbed), the Monte Carlo source draws from posterior visibility times the priors,
the bilaterally weighted NCC through the plane-induced homography, the geometric term and the filter -- with the same
counter-based random numbers, vectorised over the scan lines of a sweep.  It is meant for tiny images.

Like oracle/sift.py, it restates a recollection of upstream COLMAP's PatchMatch (U:mvs/patch_match_cuda.cu; Schoenberger
et al., ECCV 2016) and is not pinned to upstream: the recalled points are listed in SURVEY.md (rows M1-M9).  The window
sums are added in a different order than the device's warp butterfly, so costs agree to float32 rounding, not bit for
bit.
"""
import numpy as np

MASK64 = np.uint64(0xFFFFFFFFFFFFFFFF)
INIT_SWEEP = 4


def _mix64(z):
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def uniform(seed, image, pixel, it, sweep, draw):
    """The device's pm_uniform: a float32 in [0, 1) keyed by (seed, image, pixel, iteration, sweep, draw)."""
    pixel = np.asarray(pixel, np.int64).astype(np.uint64)
    h = _mix64(np.uint64(seed) ^ np.uint64(image & 0xFFFFFFFF) + np.zeros_like(pixel))
    h = _mix64(h ^ pixel)
    h = _mix64(h ^ ((np.uint64(it & 0xFFFFFFFF) << np.uint64(8)) | np.uint64(sweep)))
    h = _mix64(h ^ np.uint64(draw & 0xFFFFFFFF))
    return (h >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def defaults(**kw):
    """The options of b2m_patch_match_opts_default, with overrides."""
    o = dict(window_radius=5, window_step=1, num_samples=15, num_iterations=5, geom_consistency=False, filter=True,
             filter_min_num_consistent=2, sigma_spatial=-1.0, sigma_color=0.2, ncc_sigma=0.6, min_triangulation_angle=1.0,
             incident_angle_sigma=0.9, geom_consistency_regularizer=0.3, geom_consistency_max_cost=3.0,
             filter_min_ncc=0.1, filter_min_triangulation_angle=3.0, filter_geom_consistency_max_cost=1.0)
    o.update(kw)
    return o


def _f(v):
    return np.float32(v)


class Problem:
    """One reference image and its sources.  images: grey uint8 arrays; cams: (fx, fy, cx, cy, R (3x3), t (3)) per image,
    cam_from_world; ref / src: indices; depth maps (geometric pass): per image or None."""

    def __init__(self, images, cams, ref, src, depth_min, depth_max, depth_maps=None, image_id=None):
        self.images, self.ref, self.src = images, ref, list(src)
        self.key = ref if image_id is None else image_id  # the key of the problem's random numbers
        self.dmin, self.dmax = _f(depth_min), _f(depth_max)
        self.K = [tuple(_f(v) for v in c[:4]) for c in cams]
        self.dmaps = depth_maps
        Rr, tr = np.asarray(cams[ref][4], np.float64), np.asarray(cams[ref][5], np.float64)
        self.Rs, self.ts = [], []
        for s in self.src:
            Rc, tc = np.asarray(cams[s][4], np.float64), np.asarray(cams[s][5], np.float64)
            R = Rc @ Rr.T
            self.Rs.append(R.astype(np.float32))
            self.ts.append((tc - R @ tr).astype(np.float32))
        self.H, self.W = images[ref].shape


class Params:
    def __init__(self, o):
        self.r, self.step = o["window_radius"], o["window_step"]
        side = 2 * self.r // self.step + 1
        k = np.arange(side * side)
        self.dy = -self.r + (k // side) * self.step
        self.dx = -self.r + (k % side) * self.step
        ss = _f(o["sigma_spatial"]) if o["sigma_spatial"] > 0 else _f(self.r)
        self.inv_2ss = _f(1.0) / (_f(2.0) * ss * ss)
        sc = _f(o["sigma_color"])
        self.inv_2sc = _f(1.0) / (_f(2.0) * sc * sc)
        ns = _f(o["ncc_sigma"])
        self.inv_2ncc = _f(1.0) / (_f(2.0) * ns * ns)
        deg = _f(3.14159265358979) / _f(180.0)
        self.min_tri = max(_f(o["min_triangulation_angle"]) * deg, _f(1e-6))
        si = _f(o["incident_angle_sigma"])
        self.inv_2inc = _f(1.0) / (_f(2.0) * si * si)
        self.num_samples = o["num_samples"]
        self.geom = bool(o["geom_consistency"])
        self.reg, self.gmax = _f(o["geom_consistency_regularizer"]), _f(o["geom_consistency_max_cost"])
        self.filter_max_cost = _f(1.0) - _f(o["filter_min_ncc"])
        self.filter_min_tri = _f(o["filter_min_triangulation_angle"]) * deg
        self.filter_geom_max = _f(o["filter_geom_consistency_max_cost"])
        self.min_consistent = o["filter_min_num_consistent"]


def _pix(img, x, y):
    H, W = img.shape
    ok = (x >= 0) & (y >= 0) & (x < W) & (y < H)
    v = img[np.clip(y, 0, H - 1), np.clip(x, 0, W - 1)].astype(np.float32) * _f(1.0 / 255.0)
    return np.where(ok, v, _f(0.0))


def bilinear(img, u, v):
    """Bilinear sample at COLMAP coordinates (pixel centres at +0.5), zero outside the image."""
    x, y = u - _f(0.5), v - _f(0.5)
    good = (np.abs(x) < _f(1e6)) & (np.abs(y) < _f(1e6))
    x, y = np.where(good, x, _f(0)), np.where(good, y, _f(0))
    fx, fy = np.floor(x), np.floor(y)
    x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
    ax, ay = x - fx, y - fy
    top = (_f(1) - ax) * _pix(img, x0, y0) + ax * _pix(img, x0 + 1, y0)
    bot = (_f(1) - ax) * _pix(img, x0, y0 + 1) + ax * _pix(img, x0 + 1, y0 + 1)
    return np.where(good, (_f(1) - ay) * top + ay * bot, _f(0))


def _ray(K, x, y):
    fx, fy, cx, cy = K
    return ((x.astype(np.float32) + _f(0.5) - cx) / fx, (y.astype(np.float32) + _f(0.5) - cy) / fy)


def _window(P, pr, x, y):
    """Per-sample reference values and bilateral weights, [L, S], with the validity mask."""
    img = pr.images[pr.ref]
    xx, yy = x[:, None] + P.dx[None], y[:, None] + P.dy[None]
    ok = (xx >= 0) & (yy >= 0) & (xx < pr.W) & (yy < pr.H)
    r = _pix(img, xx, yy)
    c0 = _pix(img, x, y)[:, None]
    dc = r - c0
    sd = (P.dx * P.dx + P.dy * P.dy).astype(np.float32)[None]
    w = np.exp(-sd * P.inv_2ss - dc * dc * P.inv_2sc).astype(np.float32)
    w = np.where(ok, w, _f(0))
    return xx, yy, r, w, ok


def photo_cost(P, pr, s, x, y, d, n, win=None):
    """1 - weighted NCC of hypotheses (d [L], n [L, 3]) at pixels (x, y) [L] against source slot s, in [0, 2]."""
    xx, yy, r, w, ok = win if win is not None else _window(P, pr, x, y)
    K = pr.K[pr.ref]
    rx, ry = _ray(K, x, y)
    dn = d * (n[:, 0] * rx + n[:, 1] * ry + n[:, 2] * _f(1))
    Rs, ts = pr.Rs[s], pr.ts[s]
    with np.errstate(all="ignore"):
        M = Rs[None] + ts[None, :, None] * n[:, None, :] / dn[:, None, None]  # [L, 3, 3]
        q0 = (xx.astype(np.float32) + _f(0.5) - K[2]) / K[0]
        q1 = (yy.astype(np.float32) + _f(0.5) - K[3]) / K[1]
        Y0 = M[:, 0, 0, None] * q0 + M[:, 0, 1, None] * q1 + M[:, 0, 2, None]
        Y1 = M[:, 1, 0, None] * q0 + M[:, 1, 1, None] * q1 + M[:, 1, 2, None]
        Y2 = M[:, 2, 0, None] * q0 + M[:, 2, 1, None] * q1 + M[:, 2, 2, None]
        Ks = pr.K[pr.src[s]]
        sv = bilinear(pr.images[pr.src[s]], Ks[0] * (Y0 / Y2) + Ks[2], Ks[1] * (Y1 / Y2) + Ks[3])
        sv = np.where((Y2 > 0) & ok, sv, _f(0))
        sw, swr, swrr = w.sum(1), (w * r).sum(1), (w * r * r).sum(1)
        sws, swss, swrs = (w * sv).sum(1), (w * sv * sv).sum(1), (w * r * sv).sum(1)
        inv = _f(1) / sw
        mr, ms = swr * inv, sws * inv
        vr, vs = swrr * inv - mr * mr, swss * inv - ms * ms
        cv = swrs * inv - mr * ms
        ncc = cv / np.sqrt(vr * vs)
        c = np.clip(_f(1) - ncc, _f(0), _f(2))
    bad = ~(vr > _f(1e-5)) | ~(vs > _f(1e-5)) | ~(np.abs(dn) > 0)
    return np.where(bad, _f(2), c).astype(np.float32)


def geom_error(P, pr, s, x, y, d, n):
    """Forward-backward reprojection error through the source's depth map, at most geom_consistency_max_cost."""
    K = pr.K[pr.ref]
    rx, ry = _ray(K, x, y)
    X = np.stack([d * rx, d * ry, d], 1)
    Rs, ts = pr.Rs[s], pr.ts[s]
    Y = X @ Rs.T + ts
    Ks = pr.K[pr.src[s]]
    dm = pr.dmaps[pr.src[s]]
    Hs, Ws = dm.shape
    cap = P.gmax
    with np.errstate(all="ignore"):
        u, v = Ks[0] * (Y[:, 0] / Y[:, 2]) + Ks[2], Ks[1] * (Y[:, 1] / Y[:, 2]) + Ks[3]
        inside = (Y[:, 2] > 0) & (u >= 0) & (v >= 0) & (u < Ws) & (v < Hs)
        su = np.where(inside, u, 0).astype(np.int64)
        sv = np.where(inside, v, 0).astype(np.int64)
        ds = dm[sv, su].astype(np.float32)
        Z = np.stack([ds * ((su.astype(np.float32) + _f(0.5) - Ks[2]) / Ks[0]) - ts[0],
                      ds * ((sv.astype(np.float32) + _f(0.5) - Ks[3]) / Ks[1]) - ts[1], ds - ts[2]], 1)
        B = Z @ Rs
        ex = K[0] * (B[:, 0] / B[:, 2]) + K[2] - (x.astype(np.float32) + _f(0.5))
        ey = K[1] * (B[:, 1] / B[:, 2]) + K[3] - (y.astype(np.float32) + _f(0.5))
        e = np.minimum(np.sqrt(ex * ex + ey * ey), cap)
    return np.where(inside & (ds > 0) & (B[:, 2] > 0), e, cap).astype(np.float32)


def view_angles(pr, s, x, y, d, n):
    K = pr.K[pr.ref]
    rx, ry = _ray(K, x, y)
    X = np.stack([d * rx, d * ry, d], 1)
    Rs, ts = pr.Rs[s], pr.ts[s]
    C = -(Rs.T @ ts)
    v = X - C
    nx, nv = np.linalg.norm(X, axis=1), np.linalg.norm(v, axis=1)
    return (X * v).sum(1) / (nx * nv), -(n * v).sum(1) / nv


def propagated_depth(K, x, y, d, n, x2, y2):
    """Depth at pixel (x2, y2) of the plane through the hypothesis point of (x, y)."""
    rx, ry = _ray(K, x, y)
    qx, qy = _ray(K, x2, y2)
    num = d * (n[:, 0] * rx + n[:, 1] * ry + n[:, 2])
    with np.errstate(all="ignore"):
        return num / (n[:, 0] * qx + n[:, 1] * qy + n[:, 2])


def _face(n, rx, ry):
    flip = (n[:, 0] * rx + n[:, 1] * ry + n[:, 2]) > 0
    return np.where(flip[:, None], -n, n)


def random_hyp(seed, image, pixel, it, sweep, draw, dmin, dmax, rx, ry):
    u0 = uniform(seed, image, pixel, it, sweep, draw)
    u1 = uniform(seed, image, pixel, it, sweep, draw + 1)
    u2 = uniform(seed, image, pixel, it, sweep, draw + 2)
    z = _f(2) * u1 - _f(1)
    phi = _f(6.2831853) * u2
    rxy = np.sqrt(np.maximum(_f(1) - z * z, _f(0)))
    n = np.stack([rxy * np.cos(phi), rxy * np.sin(phi), z], 1).astype(np.float32)
    return (dmin + u0 * (dmax - dmin)).astype(np.float32), _face(n, rx, ry)


STAY = _f(0.999)
UNIFORM = _f(0.5)


def hmm_predict(m):
    return m * STAY + (_f(1) - m) * (_f(1) - STAY)


def hmm_update(P, pred, cost):
    z1 = pred * np.exp(-cost * cost * P.inv_2ncc)
    z0 = (_f(1) - pred) * UNIFORM
    return (z1 / (z0 + z1)).astype(np.float32)


def hmm_posterior(f, b):
    v, o = f * b, (_f(1) - f) * (_f(1) - b)
    return (v / (v + o)).astype(np.float32)


def _select_prob(P, post, cos_tri, cos_inc):
    tri = np.arccos(np.clip(cos_tri, -1, 1)).astype(np.float32)
    prior_tri = np.where(tri < P.min_tri, (tri / P.min_tri) ** 2, _f(1))
    om = _f(1) - cos_inc
    prior_inc = np.where(cos_inc > 0, np.exp(-om * om * P.inv_2inc), _f(0))
    return (post * prior_tri * prior_inc).astype(np.float32)


def run(problem, options, seed=0, init=None):
    """Depth [H, W] and normal [H, W, 3] maps of `problem` (filtered pixels 0) as K8 computes them."""
    P = Params(options)
    pr = problem
    H, W, ns = pr.H, pr.W, len(pr.src)
    ys, xs = np.mgrid[0:H, 0:W]
    xs, ys = xs.ravel(), ys.ravel()
    pix = ys * W + xs
    rx, ry = _ray(pr.K[pr.ref], xs, ys)
    d, n = random_hyp(seed, pr.key, pix, 0, INIT_SWEEP, 0, pr.dmin, pr.dmax, rx, ry)
    if init is not None:
        d0, n0 = init[0].ravel(), init[1].reshape(-1, 3)
        use = d0 > 0
        d = np.where(use, d0, d).astype(np.float32)
        n = np.where(use[:, None], n0, n).astype(np.float32)
    depth, normal = d.reshape(H, W), n.reshape(H, W, 3)

    def eval_all(x, y, dd, nn, win):
        c = np.stack([photo_cost(P, pr, s, x, y, dd, nn, win) for s in range(ns)])
        g = np.stack([geom_error(P, pr, s, x, y, dd, nn) for s in range(ns)]) if P.geom else np.zeros_like(c)
        return c, g

    def line_pixels(vertical, j, lines):
        line = np.arange(lines)
        return (line, np.full(lines, j)) if vertical else (np.full(lines, j), line)

    def backward(vertical, forward, length, lines):
        """Predicted backward message [position along the line][source, line] from the current hypotheses."""
        out = np.zeros((length, ns, lines), np.float32)
        b = np.full((ns, lines), 0.5, np.float32)
        for i in range(length - 1, -1, -1):
            j = i if forward else length - 1 - i
            x, y = line_pixels(vertical, j, lines)
            pred = hmm_predict(b)
            out[j] = pred
            c, _ = eval_all(x, y, depth[y, x], normal[y, x], _window(P, pr, x, y))
            b = hmm_update(P, pred, c)
        return out

    for it in range(options["num_iterations"]):
        perturb = _f(2.0 ** -it)
        for sw in range(4):
            vertical, forward = sw < 2, sw % 2 == 0
            length, lines = (H, W) if vertical else (W, H)
            bpred = backward(vertical, forward, length, lines)
            fwd = np.full((ns, lines), 0.5, np.float32)
            prev = None
            for i in range(length):
                j = i if forward else length - 1 - i
                line = np.arange(lines)
                x, y = (line, np.full(lines, j)) if vertical else (np.full(lines, j), line)
                pixel = y * W + x
                crx, cry = _ray(pr.K[pr.ref], x, y)
                cd, cn = depth[y, x].copy(), normal[y, x].copy()
                win = _window(P, pr, x, y)
                c, g = eval_all(x, y, cd, cn, win)
                ang = [view_angles(pr, s, x, y, cd, cn) for s in range(ns)]
                fwd = hmm_update(P, hmm_predict(fwd), c)
                post = hmm_posterior(fwd, bpred[j])
                prob = np.stack([_select_prob(P, post[s], ang[s][0], ang[s][1]) for s in range(ns)])
                cum = np.cumsum(prob, 0, dtype=np.float32)
                total = cum[-1]
                uni = ~(total > _f(1e-20))
                count = np.zeros((ns, lines), np.int64)
                for q in range(P.num_samples):
                    u = uniform(seed, pr.key, pixel, it, sw, q)
                    t = u * total
                    lo = cum - prob
                    hit = (prob > 0) & (t >= lo) & ((t < cum) | (np.arange(ns)[:, None] == ns - 1))
                    first = np.where(hit.any(0), hit.argmax(0), -1)
                    pick = np.where(uni, np.minimum((u * ns).astype(np.int64), ns - 1), first)
                    for s in range(ns):
                        count[s] += pick == s
                inv_n = _f(1.0 / P.num_samples)

                def total_cost(cc, gg):
                    return (count.astype(np.float32) * (cc + P.reg * gg)).sum(0).astype(np.float32) * inv_n

                best_c = total_cost(c, g)
                bd, bn = cd.copy(), cn.copy()
                cands = []
                if i > 0:
                    pd, pn = prev
                    px = x if vertical else (x - 1 if forward else x + 1)
                    py = (y - 1 if forward else y + 1) if vertical else y
                    dp = propagated_depth(pr.K[pr.ref], px, py, pd, pn, x, y)
                    dp = np.where((dp > 0) & np.isfinite(dp), dp, pd)
                    cands.append((np.clip(dp, pr.dmin, pr.dmax).astype(np.float32), pn))
                q0 = P.num_samples
                cands.append(random_hyp(seed, pr.key, pixel, it, sw, q0, pr.dmin, pr.dmax, crx, cry))
                u = [uniform(seed, pr.key, pixel, it, sw, q0 + 3 + k) for k in range(4)]
                pd = cd * (_f(1) + _f(0.05) * perturb * (_f(2) * u[0] - _f(1)))
                m = np.stack([cn[:, k] + _f(0.5) * perturb * (_f(2) * u[k + 1] - _f(1)) for k in range(3)], 1)
                m = (m * (_f(1) / np.sqrt((m * m).sum(1)))[:, None]).astype(np.float32)
                back = (m[:, 0] * crx + m[:, 1] * cry + m[:, 2]) > 0
                m = np.where(back[:, None], cn, m)
                cands.append((np.clip(pd, pr.dmin, pr.dmax).astype(np.float32), m))
                for dd, nn in cands:
                    cc, gg = eval_all(x, y, dd, nn, win)
                    tc = total_cost(cc, gg)
                    better = tc < best_c
                    best_c = np.where(better, tc, best_c)
                    bd = np.where(better, dd, bd)
                    bn = np.where(better[:, None], nn, bn)
                depth[y, x], normal[y, x] = bd, bn
                prev = (bd, bn)
    if options["filter"]:
        bpred = backward(True, True, H, W)
        fwd = np.full((ns, W), 0.5, np.float32)
        drop = np.zeros((H, W), bool)
        for yy in range(H):
            x, y = line_pixels(True, yy, W)
            dd, nn = depth[y, x], normal[y, x]
            c, g = eval_all(x, y, dd, nn, _window(P, pr, x, y))
            fwd = hmm_update(P, hmm_predict(fwd), c)
            post = hmm_posterior(fwd, bpred[yy])
            ok = np.zeros(W, np.int64)
            for s in range(ns):
                tri = np.arccos(np.clip(view_angles(pr, s, x, y, dd, nn)[0], -1, 1))
                good = (post[s] >= 0.5) & (c[s] <= P.filter_max_cost) & (tri >= P.filter_min_tri)
                if P.geom:
                    good &= g[s] <= P.filter_geom_max
                ok += good
            drop[yy] = ok < P.min_consistent
        depth[drop] = 0
        normal[drop] = 0
    return depth, normal

"""Second, independent restatement of the hot path in pure Python (numpy scalars), written from
SURVEY.md Appendix A/B rather than from oracle/gg_oracle.cpp, so that a typo in either shows
up as a bit mismatch in tests/test_oracle_vs_pyref.py.  Small inputs only (pure-Python loops).

Type discipline mirrors the C++ promotions of the reference: every value is an explicit
np.float32 / np.float64 scalar (NumPy 2 treats bare Python floats as "weak", so doubles are
always wrapped in f64()).
Reference: src/GroundSegmentation.cpp:50-197,200-311,314-340,343-395,398-465.
"""
import math

import numpy as np

f32 = np.float32
f64 = np.float64
FLT_MIN = f32(np.finfo(np.float32).tiny)
FLT_MAX = f32(np.finfo(np.float32).max)

DEFAULT_CFG = dict(
    point_count_cell_variance_threshold=10,
    max_ring=1024,
    groundpatch_detection_minimum_threshold=0.01,
    distance_factor=0.0001,
    minimum_distance_factor=0.0005,
    miminum_point_height_threshold=0.3,
    minimum_point_height_obstacle_threshold=0.1,
    outlier_tolerance=0.1,
    ground_patch_detection_minimum_point_count_threshold=0.25,
    patch_size_change_distance=20.0,
    occupied_cells_decrease_factor=5.0,
    occupied_cells_point_count_factor=20.0,
    min_outlier_detection_ground_confidence=1.25,
    thread_count=8,
)


def tree_sum(e):
    """Eigen 3.3.7 redux_novec_unroller order (binary split, column-major block order)."""
    n = len(e)
    if n == 1:
        return e[0]
    h = n // 2
    return f32(tree_sum(e[:h]) + tree_sum(e[h:]))


def block(m, r0, c0, S):
    return [m[r0 + k % S, c0 + k // S] for k in range(S * S)]


class Geo:
    def __init__(self, length_m, res_f32, px, py):
        self.res = f64(f32(res_f32))
        self.n = int(round(float(f64(length_m) / self.res)))
        self.len = f64(self.n) * self.res
        self.px = f64(px)
        self.py = f64(py)

    def index(self, x, y):
        half = f64(0.5) * self.len
        vx = (f64(x) - half - self.px) / self.res
        vy = (f64(y) - half - self.py) / self.res
        return -int(vx), -int(vy)

    def inside(self, x, y):
        half = f64(0.5) * self.len
        tx = -(f64(x) - self.px - half)
        ty = -(f64(y) - self.py - half)
        return bool(tx >= 0.0 and ty >= 0.0 and tx < self.len and ty < self.len)


def filter_cloud(points, origin, base_z, G, C, E, geo, cfg=None, stop_after=0):
    """points: structured array with x,y,z,ring; G, C: float32 (n,n) arrays [i,j], modified in place.
    Returns dict(labels=..., layers...)."""
    cfg = dict(DEFAULT_CFG, **(cfg or {}))
    N = geo.n
    ox, oy, oz = f32(origin[0]), f32(origin[1]), f32(origin[2])
    z = lambda: np.zeros((N, N), np.float32)
    cnt, m2, mean, gc, pdist, raw = z(), z(), z(), z(), z(), z()
    minh = np.full((N, N), FLT_MAX, np.float32)
    maxh = np.full((N, N), FLT_MIN, np.float32)
    kept, ignored, outliers = [], [], []
    npts = len(points)

    for i in range(npts):
        x, y, zz, ring = f32(points["x"][i]), f32(points["y"][i]), f32(points["z"][i]), int(points["ring"][i])
        dxo = f32(x - ox)
        dyo = f32(y - oy)
        sqdist = f32(f64(dxo) * f64(dxo) + f64(dyo) * f64(dyo))
        if not (math.isfinite(float(x)) and math.isfinite(float(y))):
            continue
        gi = geo.index(x, y)
        if not geo.inside(x, y):
            continue
        if gi[0] < 0 or gi[1] < 0 or gi[0] >= N or gi[1] >= N:
            continue
        raw[gi] = f32(raw[gi] + f32(1.0))
        if ring > cfg["max_ring"] or sqdist < f32(12.0):
            ignored.append((i, gi))
            continue
        skip = False
        if f64(zz) < f64(G[gi]) - f64(0.2):
            vx, vy, vz = dxo, dyo, f32(zz - oz)
            ln = np.sqrt(f32(f32(f32(vx * vx) + f32(vy * vy)) + f32(vz * vz)))
            ln = f32(ln)
            with np.errstate(all="ignore"):
                vx, vy, vz = f32(vx / ln), f32(vy / ln), f32(vz / ln)
            step = 3
            while True:
                sx, sy, sz = f32(f32(step) * vx), f32(f32(step) * vy), f32(f32(step) * vz)
                lhs = f64(sx) * f64(sx) + f64(sy) * f64(sy) + f64(sz) * f64(sz)
                if not (lhs < f64(ln) * f64(ln) and vz < f32(-0.01)):
                    break
                I = geo.index(f32(sx + ox), f32(sy + oy))
                if not (I[0] <= 0 or I[1] <= 0 or I[0] >= N - 1 or I[1] >= N - 1):
                    bs = tree_sum(block(C, max(I[0] - 1, 2), max(I[1] - 1, 2), 3))
                    if (f64(bs) > f64(cfg["min_outlier_detection_ground_confidence"]) and C[I] > f32(0.01)
                            and f64(G[I]) >= f64(f32(sz + oz)) + f64(cfg["outlier_tolerance"])):
                        outliers.append(i)
                        skip = True
                        break
                step += 1
        if skip:
            continue
        kept.append((i, gi))
        n = cnt[gi]
        pd = f32(zz - oz)
        gc[gi] = f32(f64(f32(zz + f32(n * gc[gi]))) / (f64(n) + f64(1.0)))
        if mean[gi] == 0.0:
            mean[gi] = pd
        if not math.isnan(float(pd)):
            delta = f32(pd - mean[gi])
            mean[gi] = f32(mean[gi] + f32(delta / f32(n + f32(1.0))))
            pdist[gi] = f32(f64(f32(pd + f32(n * pdist[gi]))) / (f64(n) + f64(1.0)))
            m2[gi] = f32(m2[gi] + f32(delta * f32(pd - mean[gi])))
        maxh[gi] = max(maxh[gi], zz)
        minh[gi] = min(minh[gi], f32(zz - f32(0.0001)))
        cnt[gi] = f32(n + f32(1.0))

    var = np.zeros((N, N), np.float32)
    out = dict(kept=kept, ignored=ignored, outliers=outliers, count=cnt.copy(), m2=m2, minGroundHeight=minh,
               maxGroundHeight=maxh, meanVariance=mean, groundCandidates=gc, planeDist=pdist, pointsRaw=raw, variance=var)
    if stop_after == 1:
        return out

    # ---- detect_ground_patches (A.3 / A.4)
    with np.errstate(all="ignore"):
        var[...] = m2 / (cnt + FLT_MIN)
    res_f = f32(geo.res)
    for i in range(2, N - 2):
        for j in range(2, N - 2):
            detect_cell(cnt, var, minh, G, C, E, i, j, patch_size(N, res_f, cfg, i, j), cfg, res_f)
    if stop_after == 2:
        return out

    # ---- spiral (A.5)
    c = N // 2 - 1
    C[c, c] = f32(1.0)
    G[c, c] = f32(f64(base_z))
    res2 = geo.res * geo.res

    def visit(x, y):
        Cb = block(C, x - 1, y - 1, 3)
        Gb = block(G, x - 1, y - 1, 3)
        s = f32(tree_sum(Cb) + FLT_MIN)
        avg = f32(tree_sum([f32(a * b) for a, b in zip(Cb, Gb)]) / s)
        occ = C[x, y]
        G[x, y] = f32(f32(f32(f32(1.0) - occ) * avg) + f32(occ * G[x, y]))
        fx = f32(f32(x) - f32(c))
        fy = f32(f32(y) - f32(c))
        if (f64(fx) * f64(fx) + f64(fy) * f64(fy)) * res2 > f64(12.0):
            C[x, y] = f32(max(f64(occ) - f64(occ) / f64(cfg["occupied_cells_decrease_factor"]), f64(0.001)))

    for p in range(c - 1, 0, -1):
        Ls = (c - p) * 2
        for side in range(2):
            for pos in range(p, p + Ls):
                visit(pos if side else p, p if side else pos)
        q = p + Ls
        for side in range(2):
            for pos in range(q, q - Ls - 1, -1):
                visit(pos if side else q, q if side else pos)
    if stop_after == 3:
        return out

    # ---- labels (A.6)
    labels = np.zeros(npts, np.uint8)
    obst = z()
    order = []
    mdf5 = f64(cfg["minimum_distance_factor"]) * f64(5)
    thr = f64(cfg["miminum_point_height_threshold"])
    othr = f64(cfg["minimum_point_height_obstacle_threshold"])
    for (i, gi) in kept + ignored:
        if N <= gi[0] + 3 or N <= gi[1] + 3:
            continue
        x, y, zz = f32(points["x"][i]), f32(points["y"][i]), f32(points["z"][i])
        dxo, dyo = f32(x - ox), f32(y - oy)
        dist = f32(np.sqrt(f64(dxo) * f64(dxo) + f64(dyo) * f64(dyo)))
        with np.errstate(all="ignore"):
            a = (mdf5 * f64(dist)) / f64(var[gi]) * thr
        t = thr if thr < a else a          # std::min(a, b) = (b < a) ? b : a
        t = othr if t < othr else t        # std::max(a, b) = (a < b) ? b : a
        if t + f64(G[gi]) < f64(zz):
            labels[i] = 99
            obst[gi] = f32(obst[gi] + f32(1.0))
        else:
            labels[i] = 49
        order.append(i)
    for i in outliers:
        labels[i] = 49
        order.append(i)
    out.update(labels=labels, order=np.array(order, np.uint32), points=obst)
    return out


def patch_size(N, res_f, cfg, i, j):
    """3 or 5: the window detect_ground_patches picks for cell (i, j) (:332-337)."""
    di = f64(i) - f64(N) / f64(2.0)
    dj = f64(j) - f64(N) / f64(2.0)
    sqd = f32((di * di + dj * dj) * (f64(res_f) * f64(res_f)))
    return 3 if f64(sqd) <= f64(cfg["patch_size_change_distance"]) ** 2 else 5


def variance_threshold(N, res_f, cfg, i, j):
    """varThresholdsq of cell (i, j) (:369)."""
    di = f64(i) - f64(N) / f64(2.0)
    dj = f64(j) - f64(N) / f64(2.0)
    sqd = f32((di * di + dj * dj) * (f64(res_f) * f64(res_f)))
    dfac = f64(cfg["distance_factor"])
    mdf = f64(cfg["minimum_distance_factor"])
    return f32(min(max(f64(sqd) * (dfac * dfac), mdf * mdf), (mdf * f64(10)) * (mdf * f64(10))))


def min_point_count(cfg, S, e):
    """The early-skip bound of :364, a double (NaN stays NaN: std::max(NaN, 3.0) is NaN)."""
    x = f64(cfg["ground_patch_detection_minimum_point_count_threshold"]) * f64(S) * f64(e)
    x = f64(math.floor(x)) if math.isfinite(x) else x
    return f64(3.0) if x < 3.0 else x


def detect_cell(cnt, var, minh, G, C, E, i, j, S, cfg, res_f):
    """GroundSegmentation::detect_ground_patch<S>(map, i, j) (A.4, :343-395) on the planes as stored: updates G, C in place
    and returns which way the cell went: "need" (skipped, too few points, :364), "upward" (skipped, known high confidence
    estimate not raised, :379), "confident" (:382-388), "localmin" (:389-394) or "unchanged"."""
    N = cnt.shape[0]
    cfg = dict(DEFAULT_CFG, **(cfg or {}))
    h = S // 2
    Pb = block(cnt, i - h, j - h, S)
    psum = tree_sum(Pb)
    e = E[i, j]
    oc, og = C[i, j], G[i, j]
    if f64(psum) < min_point_count(cfg, S, e):
        return "need"
    vt = variance_threshold(N, res_f, cfg, i, j)
    Vb = block(var, i - h, j - h, S)
    Mb = block(minh, i - h, j - h, S)
    variance = var[i, j]
    localmin = Mb[0]
    for t in Mb[1:]:                     # minCoeff: column by column, the first strict minimum (a NaN only from element 0)
        if t < localmin:
            localmin = t
    with np.errstate(all="ignore"):
        if cnt[i, j] >= f32(cfg["point_count_cell_variance_threshold"]):
            maxVar = variance
        else:
            maxVar = f32(tree_sum([f32(p * v) for p, v in zip(Pb, Vb)]) / psum)
        groundlevel = f32(tree_sum([f32(p * m) for p, m in zip(Pb, Mb)]) / psum)
        gd = f32(f32(groundlevel - og) * f32(f32(2.0) * oc))
        groundDiff = f32(1.0) if gd < f32(1.0) else gd
        if f64(oc) > 0.5 and f64(groundlevel) >= f64(og) + f64(cfg["outlier_tolerance"]):
            return "upward"
        factor = f64(cfg["occupied_cells_point_count_factor"])
        gp = f64(cfg["ground_patch_detection_minimum_point_count_threshold"])
        if (f64(vt) > f64(maxVar) * f64(maxVar) and maxVar > 0
                and f64(psum) > f64(f32(f32(groundDiff * e) * f32(S))) * gp):
            q = f64(psum) / factor
            nc = f32(f64(1.0) if f64(1.0) < q else q)
            num = f32(f32(groundlevel * nc) + f32(f32(oc * og) * f32(2)))
            den = f32(nc + f32(oc * f32(2)))
            G[i, j] = f32(num / den)
            c = (f64(psum) / (factor * f64(2.0)) + f64(oc)) / f64(2.0)
            C[i, j] = f32(f64(1.0) if f64(1.0) < c else c)
            return "confident"
        if localmin < og:
            G[i, j] = localmin
            t = f32(oc + f32(0.1))
            C[i, j] = f32(0.5) if f32(0.5) < t else t
            return "localmin"
    return "unchanged"

"""Priors and rays for the outlier test of k_rasterize (insert_cloud :243-272): the pre-test against the prior "ground",
then the occlusion ray-march over the prior "groundpatch" / "ground".  Synthetic scans only reach it with smooth
confidences and rays of a few dozen steps; a caller can import any float into both planes (gg_set_layer /
gg_set_layers_from_device) and send rays of any length.  Each case here plants one ray on one decision of the march,
on both sides of it (the float or double neighbour):

  pretest      z against (double) G[cell] - 0.2, and G NaN, +-inf, -0, a denormal, +-FLT_MAX
  direction    vz against -0.01f: the adjacent floats z whose vz fall on either side of it
  loop_end     the occluding cell met at the last step the loop runs (lhs < len2), or at the first it does not
  cell         C == 0.01f and above; the 3x3 sum at the threshold (1.25, representable; 0.6, not); Eigen's tree sum and the
               sequential sum on opposite sides of it; G at the height bound fl(fl(s * vz) + oz) + tol and one float
               below; NaN, +-inf, inf - inf, FLT_MAX sums, -0 and denormals in the block
  geometry     occluders at ix / iy = 0, 1, 2, 3, N-2, N-1 (rows 1 .. 3 share the clamped block at row 2), rays entering
               and leaving the interior, an origin outside the map, origins on cell edges
  config       min_outlier_detection_ground_confidence <= 0 and large; outlier_tolerance < 0, 0, > 0
  long         steep rays whose first occluding cell lies just before / after step 2^20 (the step cap the march once
               had), and around step 4096 (where k_rasterize hands a ray to its exact walk); |z - oz| up to 3e7; an
               origin 2e6 m outside the map whose ray enters it

The march itself is restated here with numpy (march(): float32 / float64 arrays, chunk by chunk, for rays of any
length); tests/test_outlier_rays.py checks that every case lands where its name says, and the oracle against it.
"""
from dataclasses import dataclass, field

import numpy as np

import pyref

f32, f64 = np.float32, np.float64
FLT_MAX = f32(np.finfo(np.float32).max)
DENORMAL = f32(1e-40)
OLD_CAP = 1 << 20       # the step cap k_rasterize's march once had
WALK_FROM = 4096        # gg_internal.h:RAY_WALK_FROM
INT_END = 1 << 31       # the reference counts in int: the march ends after step INT_MAX
GEOMETRY = {100: (33.0, 0.33), 101: (33.0, float(np.float32(33.0 / 101.0))), 300: (99.0, 0.33)}
FAR = (1.2e5 + 0.37, -3.4e5 - 0.11)
BACKGROUND_G = f32(-1000.0)   # no cell occludes unless planted
POINT_RING = 10


def up(x, n=1):
    x = f32(x)
    for _ in range(n):
        x = np.nextafter(x, f32(np.inf))
    return x


def down(x, n=1):
    x = f32(x)
    for _ in range(n):
        x = np.nextafter(x, f32(-np.inf))
    return x


@dataclass
class Case:
    name: str
    n: int
    position: tuple
    G: np.ndarray
    C: np.ndarray
    origin: np.ndarray          # float32 (3,)
    point: np.ndarray           # float32 (3,): the one point of the cloud
    cfg: dict = field(default_factory=dict)
    regime: str = ""            # what the case is planted on (checked by tests/test_outlier_rays.py)
    want: object = None         # (outlier, step): the numpy march's answer, step of the hit or None

    @property
    def dim(self):
        return GEOMETRY[self.n][0]

    @property
    def res(self):
        return GEOMETRY[self.n][1]

    def geo(self):
        return pyref.Geo(self.dim, self.res, *self.position)

    def thr(self):
        return f64(dict(pyref.DEFAULT_CFG, **self.cfg)["min_outlier_detection_ground_confidence"])

    def tol(self):
        return f64(dict(pyref.DEFAULT_CFG, **self.cfg)["outlier_tolerance"])

    def cloud(self):
        from oracle import POINT_DTYPE

        pts = np.zeros(1, POINT_DTYPE)
        pts["x"], pts["y"], pts["z"], pts["ring"] = self.point[0], self.point[1], self.point[2], POINT_RING
        return pts


# ---- the march, restated over arrays of steps -------------------------------------------------------------------------
@dataclass
class Ray:
    ox: np.float32
    oy: np.float32
    oz: np.float32
    vx: np.float32
    vy: np.float32
    vz: np.float32
    len2: np.float64


def ray(origin, point):
    """The unit direction and len^2 of insert_cloud :250-257 (pyref's arithmetic)."""
    ox, oy, oz = (f32(v) for v in origin)
    vx, vy, vz = f32(f32(point[0]) - ox), f32(f32(point[1]) - oy), f32(f32(point[2]) - oz)
    ln = f32(np.sqrt(f32(f32(f32(vx * vx) + f32(vy * vy)) + f32(vz * vz))))
    with np.errstate(all="ignore"):
        return Ray(ox, oy, oz, f32(vx / ln), f32(vy / ln), f32(vz / ln), f64(ln) * f64(ln))


def _trunc(q):
    """(int) of the quotient, clamped at +-1e9 like k_rasterize's trunc_index (outside the map either way)."""
    q = np.where(np.isnan(q), 1e9, np.clip(q, -1e9, 1e9))
    return np.trunc(q).astype(np.int64)


def at(r, geo, steps):
    """lhs, ix, iy and fl(fl(fs * vz) + oz) of the given steps (int64 array)."""
    fs = np.asarray(steps, np.int64).astype(np.float32)
    sx, sy, sz = fs * r.vx, fs * r.vy, fs * r.vz
    lhs = (sx.astype(f64) * sx.astype(f64) + sy.astype(f64) * sy.astype(f64)) + sz.astype(f64) * sz.astype(f64)
    half = f64(0.5) * geo.len
    with np.errstate(all="ignore"):
        ix = -_trunc((((sx + r.ox).astype(f64) - half) - geo.px) / geo.res)
        iy = -_trunc((((sy + r.oy).astype(f64) - half) - geo.py) / geo.res)
    return lhs, ix, iy, (sz + r.oz).astype(np.float32)


def tree9_blocks(C):
    """tree9 of the clamped block of every cell (rows / columns max(i - 1, 2) .. + 2); NaN where there is none."""
    n = C.shape[0]
    out = np.full((n, n), np.nan, np.float32)
    r = np.maximum(np.arange(1, n - 1) - 1, 2)
    e = [C[np.ix_(r + q % 3, r + q // 3)] for q in range(9)]
    with np.errstate(all="ignore"):
        out[1:n - 1, 1:n - 1] = ((e[0] + e[1]) + (e[2] + e[3])) + ((e[4] + e[5]) + (e[6] + (e[7] + e[8])))
    return out


def march(c, start=3, chunk=1 << 20, end=INT_END):
    """The occlusion march of case c from step `start`: (outlier, step of the hit or None, loop end S)."""
    geo = c.geo()
    r = ray(c.origin, c.point)
    if not r.vz < f32(-0.01):
        return False, None, None
    n = c.n
    BS = tree9_blocks(c.C)
    thr, tol = c.thr(), c.tol()
    s0 = start
    while s0 < end:
        steps = np.arange(s0, min(s0 + chunk, end), dtype=np.int64)
        lhs, ix, iy, hz = at(r, geo, steps)
        run = lhs < r.len2
        stop = int(np.argmin(run)) if not run.all() else len(steps)
        inner = (ix > 0) & (iy > 0) & (ix < n - 1) & (iy < n - 1)
        i, j = np.where(inner, ix, 1), np.where(inner, iy, 1)
        with np.errstate(all="ignore"):
            hit = (inner & (BS[i, j].astype(f64) > thr) & (c.C[i, j] > f32(0.01))
                   & (c.G[i, j].astype(f64) >= hz.astype(f64) + tol))[:stop]
        if hit.any():
            return True, int(steps[int(np.argmax(hit))]), None
        if stop < len(steps):
            return False, None, int(steps[stop])
        s0 += chunk
    return False, None, end


def trace(c):
    """Steps 3 .. S-1 of a short ray: (steps, ix, iy, hz)."""
    geo = c.geo()
    r = ray(c.origin, c.point)
    steps = np.arange(3, 1 << 16, dtype=np.int64)
    lhs, ix, iy, hz = at(r, geo, steps)
    S = int(np.argmin(lhs < r.len2))
    assert S > 0
    return steps[:S], ix[:S], iy[:S], hz[:S]


def pretest(c):
    """The pre-test of :244 for the point of c: z < (double) G[cell] - 0.2."""
    i, j = c.geo().index(c.point[0], c.point[1])
    return bool(f64(c.point[2]) < f64(c.G[i, j]) - f64(0.2))


def outcome(c):
    """(outlier, step of the hit): the pre-test and the march."""
    if not pretest(c):
        return False, None
    hit, step, _ = march(c)
    return hit, step


# ---- building blocks ----------------------------------------------------------------------------------------------------
def blank(n):
    return np.full((n, n), BACKGROUND_G, np.float32), np.zeros((n, n), np.float32)


def centre(n, position, dx=0.37, dy=-0.21, z=1.8):
    return np.array([position[0] + dx, position[1] + dy, z], np.float32)


def make(name, n, position, origin, point, regime, cfg=None, G=None, C=None):
    if G is None:
        G, C = blank(n)
    c = Case(name, n, position, G, C, np.asarray(origin, np.float32), np.asarray(point, np.float32), dict(cfg or {}), regime)
    i, j = c.geo().index(c.point[0], c.point[1])
    if c.G[i, j] == BACKGROUND_G:
        c.G[i, j] = 0.0   # the point's own cell passes the pre-test
    return c


def last_steps(c):
    """Interior cells of a short ray in march order, with the last step the ray spends in each: [(i, j, step, hz)]."""
    steps, ix, iy, hz = trace(c)
    n = c.n
    out = []
    for k in range(len(steps)):
        if not (0 < ix[k] < n - 1 and 0 < iy[k] < n - 1):
            continue
        if k + 1 < len(steps) and ix[k + 1] == ix[k] and iy[k + 1] == iy[k]:
            continue
        out.append((int(ix[k]), int(iy[k]), int(steps[k]), hz[k]))
    return out


def block_cells(i, j):
    r0, c0 = max(i - 1, 2), max(j - 1, 2)
    return [(r0 + q % 3, c0 + q // 3) for q in range(9)]


def plant(c, i, j, conf=1.0, block=None, G=None):
    """Cell (i, j) occludes: confidence conf, the rest of its clamped block `block` (8 values in block order without the
    cell, or one value for all), height G (default: far above the ray)."""
    cells = [b for b in block_cells(i, j) if b != (i, j)]
    vals = [f32(1.0)] * len(cells) if block is None else (list(block) if np.ndim(block) else [f32(block)] * len(cells))
    for (a, b), v in zip(cells, vals):
        c.C[a, b] = v
    c.C[i, j] = conf
    c.G[i, j] = f32(1e6) if G is None else G
    return c


def height_bound(c, hz):
    """fl(fl(s * vz) + oz) + tol in double, and the float at / above it and the one below."""
    h = f64(hz) + c.tol()
    g = f32(h)
    if f64(g) < h:
        g = up(g)
    return h, g, down(g)


def planted_short(name, n, position, regime, cfg=None, pick=0.5, offset=(9.0, 4.0, -5.0), **kw):
    """A ray from near the map centre to `offset`, one occluder at the pick-th interior cell it visits."""
    o = centre(n, position)
    p = o + np.array(offset, np.float32)
    c = make(name, n, position, o, p, regime, cfg)
    cells = last_steps(c)
    i, j, step, hz = cells[int(pick * (len(cells) - 1))]
    return c, (i, j, step, hz)


# ---- the cases --------------------------------------------------------------------------------------------------------
def pretest_cases(n, position):
    out = []
    # z at the floats right below and right above (double) G - 0.2 (for |G| < 2^51 that double is never a float itself);
    # the march behind the pre-test always finds an occluder
    g = f32(0.75)
    bound = f64(g) - f64(0.2)
    zb = f32(bound) if f64(f32(bound)) < bound else down(f32(bound))
    for tag, z in (("just below", zb), ("two below", down(zb)), ("just above", up(zb))):
        c, (i, j, step, hz) = planted_short(f"pretest/{tag}", n, position, "pretest")
        c.point[2] = z
        c.G[c.geo().index(c.point[0], c.point[1])] = g
        cells = last_steps(c)
        plant(c, *cells[len(cells) // 2][:2])
        out.append(c)
    for tag, g in (("nan", f32(np.nan)), ("+inf", f32(np.inf)), ("-inf", f32(-np.inf)), ("-0", f32(-0.0)), ("denormal", DENORMAL),
                   ("+max", FLT_MAX), ("-max", -FLT_MAX)):
        c, (i, j, step, hz) = planted_short(f"pretest/G {tag}", n, position, "pretest")
        c.G[c.geo().index(c.point[0], c.point[1])] = g
        plant(c, i, j)
        out.append(c)
    return out


def direction_cases(n, position):
    """vz == -0.01f: z searched in float32 (pyref's arithmetic) for a fixed horizontal offset of 10 m."""
    o = centre(n, position)
    lo, hi = f32(o[2] - 1.0), f32(o[2])
    vz = lambda z: ray(o, (o[0] + f32(10.0), o[1], z)).vz
    while up(lo) < hi:   # vz grows with z: the smallest z with vz >= -0.01f
        mid = f32((f64(lo) + f64(hi)) / 2)
        mid = up(lo) if mid <= lo else mid
        if vz(mid) >= f32(-0.01):
            hi = mid
        else:
            lo = mid
    z0 = hi if vz(hi) == f32(-0.01) else lo
    out = []
    for tag, z in (("-0.01f", z0), ("above", up(z0)), ("below", down(z0))):
        c = make(f"direction/{tag}", n, position, o, (o[0] + f32(10.0), o[1], z), "direction")
        c.G[c.geo().index(c.point[0], c.point[1])] = f32(10.0)
        cells = last_steps(c) if ray(o, c.point).vz < f32(-0.01) else last_steps_any(c)
        i, j = cells[len(cells) // 2][:2]
        plant(c, i, j)
        out.append(c)
    return out


def last_steps_any(c):
    """last_steps of the same ray with the direction test ignored (for rays that do not march)."""
    d = Case(c.name, c.n, c.position, c.G, c.C, c.origin, c.point.copy(), c.cfg)
    d.point[2] = down(d.point[2], 4)
    return last_steps(d)


def loop_end_cases(n, position):
    """Integral lengths ((3, 4, -12) -> 13, (4, 4, -7) -> 9, (6, 2, -3) -> 7) and their float perturbations: the occluder
    at the cell of the loop's last step, or at the cell of the first step it does not run."""
    out = []
    o = centre(n, position)
    for off in ((3.0, 4.0, -12.0), (4.0, 4.0, -7.0), (6.0, 2.0, -3.0)):
        for pert in (0, 1, -1):
            p = o + np.array(off, np.float32)
            p[2] = up(p[2], pert) if pert > 0 else down(p[2], -pert)
            c = make(f"loop_end/{off}{pert:+d}", n, position, o, p, "loop_end")
            steps, ix, iy, hz = trace(c)
            S = int(steps[-1]) + 1
            _, jx, jy, _ = at(ray(o, p), c.geo(), np.array([S]))
            last = (int(ix[-1]), int(iy[-1]))
            beyond = (int(jx[0]), int(jy[0]))
            if beyond != last and 0 < beyond[0] < n - 1 and 0 < beyond[1] < n - 1:
                d = make(f"loop_end/{off}{pert:+d} beyond", n, position, o, p, "loop_end beyond")
                plant(d, *beyond)
                if d.G[d.geo().index(p[0], p[1])] != 0.0 and beyond != d.geo().index(p[0], p[1]):
                    pass
                out.append(d)
            if 0 < last[0] < n - 1 and 0 < last[1] < n - 1:
                plant(c, *last)
                out.append(c)
    return out


def eigen_vs_sequential(thr, seed):
    """Nine fractional confidences whose tree sum is above thr while the sequential sum is not (or the other way)."""
    rng = np.random.default_rng(seed)
    for _ in range(2000):
        e = rng.uniform(0.0, 2.0 * thr / 9, 9).astype(np.float32)
        e[8] = f32(f64(thr) - e[:8].astype(f64).sum())
        for k in range(-40, 41):   # the last value walked through the floats around the one that makes the sum thr
            e2 = e.copy()
            e2[8] = up(e[8], k) if k > 0 else down(e[8], -k)
            t = pyref.tree_sum(list(e2))
            s = f32(0.0)
            for v in e2:
                s = f32(s + v)
            if (f64(t) > f64(thr)) != (f64(s) > f64(thr)):
                return e2
    raise AssertionError("no block found")


def cell_cases(n, position):
    out = []
    # the confidence gate C > 0.01f
    for tag, v in (("C=0.01f", f32(0.01)), ("C above 0.01f", up(f32(0.01)))):
        c, (i, j, _, _) = planted_short(f"cell/{tag}", n, position, "cell C")
        out.append(plant(c, i, j, conf=v, block=f32(1.0)))
    # the block sum at the threshold
    for thr, tag in ((1.25, "1.25"), (0.6, "0.6")):
        for side, delta in (("at", 0), ("above", 1), ("below", -1)):
            c, (i, j, _, _) = planted_short(f"cell/sum {tag} {side}", n, position, "cell sum", cfg=dict(min_outlier_detection_ground_confidence=thr))
            total = up(f32(thr), delta) if delta > 0 else down(f32(thr), -delta)   # the float block sum
            conf, rest = (f32(1.0), f32(f64(total) - 1.0)) if thr > 1 else (total, f32(0.0))
            out.append(plant(c, i, j, conf=conf, block=[rest] + [f32(0.0)] * 7))
    for thr, seed in ((1.25, 1), (0.6, 2)):
        e = eigen_vs_sequential(thr, seed)
        c, (i, j, _, _) = planted_short(f"cell/tree vs sequential {thr}", n, position, "cell tree", cfg=dict(min_outlier_detection_ground_confidence=thr))
        cells = block_cells(i, j)
        for (a, b), v in zip(cells, e):
            c.C[a, b] = v
        c.G[i, j] = f32(1e6)
        out.append(c)
    # the height bound, at the cell's last step, for tol 0.1, 0 and -0.3
    for tol in (0.1, 0.0, -0.3):
        for side in ("at", "below"):
            c, (i, j, step, hz) = planted_short(f"cell/G {side} bound tol {tol}", n, position, "cell G", cfg=dict(outlier_tolerance=tol))
            _, g_at, g_below = height_bound(c, hz)
            out.append(plant(c, i, j, G=g_at if side == "at" else g_below))
    # non-finite and edge values in the block / the cell
    specials = {
        "G nan": dict(G=f32(np.nan)), "G +inf": dict(G=f32(np.inf)), "G -inf": dict(G=f32(-np.inf)),
        "C nan": dict(conf=f32(np.nan)), "C +inf": dict(conf=f32(np.inf)), "C -inf": dict(conf=f32(-np.inf)),
        "block +inf": dict(block=[f32(np.inf)] + [f32(0.0)] * 7),
        "block -inf": dict(block=[f32(-np.inf)] + [f32(1.0)] * 7),
        "block +inf -inf": dict(block=[f32(np.inf), f32(-np.inf)] + [f32(1.0)] * 6),
        "block nan": dict(block=[f32(np.nan)] + [f32(1.0)] * 7),
        "block FLT_MAX overflow": dict(block=[FLT_MAX, FLT_MAX] + [f32(0.0)] * 6),
        "block -FLT_MAX overflow": dict(conf=f32(1.0), block=[-FLT_MAX, -FLT_MAX] + [f32(0.0)] * 6),
        "block -0 denormal": dict(conf=f32(1.25), block=[f32(-0.0), DENORMAL] + [f32(0.0)] * 6),
        "block denormal above": dict(conf=f32(1.25), block=[DENORMAL, DENORMAL] + [f32(0.0)] * 6),
    }
    for tag, kw in specials.items():
        c, (i, j, _, _) = planted_short(f"cell/{tag}", n, position, "cell special")
        out.append(plant(c, i, j, **kw))
    return out


def geometry_cases(n, position):
    """Occluders at rows / columns 0, 1, 2, 3, N-2, N-1 of rays toward the map's edges (ix grows toward -x: index 0 is at the
    +x edge), a ray that leaves the interior and one that enters it from an origin outside the map, origins on cell
    edges."""
    out = []
    geo = pyref.Geo(*GEOMETRY[n], *position)
    half = float(0.5 * geo.len)
    for axis in (0, 1):
        for k in (0, 1, 2, 3, n - 2, n - 1):
            # a ray from the centre toward the edge where index k lies, ending in the edge row
            sgn = 1.0 if k < n // 2 else -1.0
            o = centre(n, position)
            for t in range(200):   # the first origin beyond that edge whose ray has a step in row k
                p = o.copy()
                o = o.copy()
                o[axis] = f32(float(position[axis]) + sgn * (half + 2.0 + 0.013 * t))
                o[2] = f32(6.0)
                p[axis] = f32(float(position[axis]) - sgn * 4.0)
                p[1 - axis] = f32(o[1 - axis] + 0.5)
                p[2] = f32(-4.0)
                c = make(f"geometry/{'xy'[axis]} row {k}", n, position, o, p, "geometry row")
                steps, ix, iy, _ = trace(c)
                hits = np.nonzero((ix if axis == 0 else iy) == k)[0]
                if len(hits):
                    break
            assert len(hits), (axis, k)
            s = hits[-1]
            i, j = int(ix[s]), int(iy[s])
            if not (0 <= i < n and 0 <= j < n):
                continue
            c.C[i, j] = 1.0
            c.G[i, j] = f32(1e6)
            if 0 < i < n - 1 and 0 < j < n - 1:
                plant(c, i, j)
            else:   # an edge cell: the march skips it, whatever it holds
                for a, b in block_cells(min(max(i, 1), n - 2), min(max(j, 1), n - 2)):
                    c.C[a, b] = 1.0
            out.append(c)
    # an origin outside the map (beyond the +x edge): the ray enters the interior and meets an occluder inside
    o = np.array([position[0] + half + 6.0, position[1] + 1.1, 9.0], np.float32)
    p = np.array([position[0] + half - 9.0, position[1] + 2.3, -3.0], np.float32)
    c = make("geometry/origin outside", n, position, o, p, "geometry enter")
    cells = last_steps(c)
    out.append(plant(c, *cells[len(cells) // 3][:2]))
    # an origin on a cell edge (x and y exactly on boundaries of the index arithmetic)
    ex = f32(geo.px + f64(0.5) * geo.len - f64(40) * geo.res)
    ey = f32(geo.py + f64(0.5) * geo.len - f64(45) * geo.res)
    for tag, (x0, y0) in (("edge", (ex, ey)), ("edge -ulp", (down(ex), down(ey))), ("edge +ulp", (up(ex), up(ey)))):
        o = np.array([x0, y0, 1.8], np.float32)
        p = np.array([x0 + f32(7.0), y0 + f32(5.0), -4.0], np.float32)
        c = make(f"geometry/origin on {tag}", n, position, o, p, "geometry edge origin")
        cells = last_steps(c)
        out.append(plant(c, *cells[0][:2]))
    return out


def config_cases(n, position):
    out = []
    for thr in (0.0, -1.0, 1e9):
        c, (i, j, _, _) = planted_short(f"config/threshold {thr:g}", n, position, "config", cfg=dict(min_outlier_detection_ground_confidence=thr))
        out.append(plant(c, i, j, conf=f32(0.5), block=f32(0.0)))
    for tol in (-0.5, 0.0, 0.5):
        c, (i, j, step, hz) = planted_short(f"config/tolerance {tol:g}", n, position, "config", cfg=dict(outlier_tolerance=tol))
        out.append(plant(c, i, j, G=f32(f64(hz) + 0.25)))
    return out


def confident_ring(n, position, inner, G=0.0):
    """A prior confident (C = 1, ground G) beyond `inner` metres from the map centre, unknown inside."""
    geo = pyref.Geo(*GEOMETRY[n], *position)
    idx = np.arange(n)
    half = f64(0.5) * geo.len
    cx = (geo.px + (half - f64(0.5) * geo.res)) - geo.res * idx   # grid_map cell centres
    cy = (geo.py + (half - f64(0.5) * geo.res)) - geo.res * idx
    r = np.hypot((cx - geo.px)[:, None], (cy - geo.py)[None, :])
    C = np.where(r > inner, 1.0, 0.0).astype(np.float32)
    return np.full((n, n), G, np.float32), C


def long_cases(n, position, heavy=True):
    """Steep rays whose first occluding step lies around 2^20 and around the walk's start; the rays of the cap probe
    (|z| from 1e3 to 2e7 under a prior confident beyond 8 m); an origin 2e6 m outside the map."""
    out = []
    o = np.array([position[0], position[1], 1.8], np.float32)
    for target, tag in ((OLD_CAP - 1, "2^20-1"), (OLD_CAP, "2^20"), (OLD_CAP + 1, "2^20+1"), (WALK_FROM - 1, "walk-1"), (WALK_FROM, "walk"),
                        (WALK_FROM + 1, "walk+1")):
        # the ray is ~10 m out at the target step; the confident ground lies at the height of that step
        zd = f32(-(target * 1.2 + 7))
        p = np.array([o[0] + 12.0, o[1] + 0.5, zd], np.float32)
        G, C = confident_ring(n, position, 8.0, G=0.0)
        c = make(f"long/hit at {tag}", n, position, o, p, "long", cfg=dict(outlier_tolerance=0.0), G=G, C=C)
        r = ray(o, p)
        _, _, _, hz = at(r, c.geo(), np.array([target - 1, target]))
        c.G[C > 0] = f32(f64(hz[1]) - f64(0.0))
        c.G[c.geo().index(p[0], p[1])] = f32(1e9)
        out.append(c)
    zs = (-1e3, -1e5, -1e6, -3e6, -2e7) if heavy else (-1e3, -3e6)
    for z in zs:
        G, C = confident_ring(n, position, 8.0)
        p = np.array([o[0] + 12.0, o[1] + 0.5, z], np.float32)
        out.append(make(f"long/cap probe z {z:g}", n, position, o, p, "long probe", G=G, C=C))
    G, C = confident_ring(n, position, 8.0)
    far_o = np.array([position[0] - 2e6, position[1] + 0.5, 3e6], np.float32)
    p = np.array([position[0] + 12.0, position[1] + 0.5, -100.0], np.float32)
    out.append(make("long/origin 2e6 m outside", n, position, far_o, p, "long enter", G=G, C=C))
    return out


def cases(n=100, position=(0.0, 0.0), heavy=True):
    out = (pretest_cases(n, position) + direction_cases(n, position) + loop_end_cases(n, position) + cell_cases(n, position)
           + geometry_cases(n, position) + config_cases(n, position) + long_cases(n, position, heavy))
    for c in out:
        c.want = outcome(c)
    return out

"""Imported planes for patch detection (GroundSegmentation.cpp:314-395), with cells planted on every branch and edge.

CPU only.  A case is one map: its geometry (N, dimension, resolution), a configuration, and the planes a caller can
import with gg_set_layer / gg_set_layers_from_device before calling the detection on its own -- "points", "m2",
"minGroundHeight", "ground", "groundpatch" and a stale "variance" (detect_ground_patches replaces it by
m2 / (points + FLT_MIN) first, :323; detect_ground_patch<S> reads it as stored).  Every case also lists its planted
cells: (i, j, S, outcome), S the window detect_ground_patches picks there and outcome the branch the cell is built to
take ("need", "upward", "confident", "localmin", "unchanged"; None where only parity with the reference is asked).

The generators:
  random      integer counts (mostly 0 .. 40, a few up to 8 192), variances around sqrt(vt), minimum heights on both
              sides of ground +- outlier_tolerance, confidences 0, 0.5 and nextafter(0.5, 1)
  boundaries  isolated windows on each boundary of the decision: psum == need and need - 1, centre count == and one
              below point_count_cell_variance_threshold, groundlevel == ground + outlier_tolerance (in double) and its
              float neighbours at confidence 0.5 and nextafter(0.5, 1), maxVar^2 just above and below vt, maxVar 0, -0
              and a denormal, psum == occupied_cells_point_count_factor, localmin == ground
  nonfinite   NaN, +-inf, -0, FLT_MAX and a denormal in each plane, at element 0 of a window, at the head of a later
              column (with the strict minimum further down that column), at the centre and at the last element
  fractional  non-integer and negative counts, windows whose sums pass 2^24
  cap         ground_patch_detection_minimum_point_count_threshold = 1e6, outside GroundGrid.cfg's range: bounds of :364
              above 2^24, with window sums just below and at the bound
  ring        resolution 0.5 (1.0 for odd N, sqdist stays exact): cells with sqdist == patch_size_change_distance^2,
              with that distance and its two double neighbours (ring, ring+, ring-)
Every case also carries one isolated window per outcome and window size, wherever the map has room for them.
"""
import math

import numpy as np

import pyref

f32, f64 = np.float32, np.float64
FLT_MIN = f32(np.finfo(np.float32).tiny)
FLT_MAX = f32(np.finfo(np.float32).max)
DENORM = f32(1e-40)
HALF_UP = np.nextafter(f32(0.5), f32(1.0))
OUTCOMES = ("need", "upward", "confident", "localmin", "unchanged")
PLANES = ("points", "m2", "minGroundHeight", "ground", "groundpatch", "variance")

# Both ends of every GroundGrid.cfg range the detection reads (cfg/GroundGrid.cfg:8-21), except
# minimum_distance_factor = 0 (vt = 0 there: no cell can take the confident branch) and patch_size_change_distance,
# which each case sets from its geometry so that both window sizes occur (the ring cases put cells on it).
CONFIGS = {
    "default": {},
    "low": dict(point_count_cell_variance_threshold=0, distance_factor=0.0, minimum_distance_factor=0.01, outlier_tolerance=-0.5,
                ground_patch_detection_minimum_point_count_threshold=0.01, occupied_cells_point_count_factor=1.0),
    "high": dict(point_count_cell_variance_threshold=30, distance_factor=0.01, minimum_distance_factor=1e-5, outlier_tolerance=0.5,
                 ground_patch_detection_minimum_point_count_threshold=1.0, occupied_cells_point_count_factor=50.0),
    "cap": dict(ground_patch_detection_minimum_point_count_threshold=1e6),
}
CASES = [("random", "default"), ("random", "low"), ("random", "high"), ("boundaries", "default"), ("boundaries", "low"),
         ("boundaries", "high"), ("nonfinite", "default"), ("nonfinite", "low"), ("fractional", "default"),
         ("fractional", "high"), ("cap", "cap"), ("ring", "default"), ("ring+", "default"), ("ring-", "default")]


def cells_per_side(dim, res):
    """GroundSegmentation::init / grid_map: round(float(dimension) / resolution) in float."""
    return int(math.floor(float(f32(dim) / f32(res)) + 0.5))


def geometry(n, ring=False):
    """(dimension, resolution) of an N x N map: an integer dimension (the reference's init takes it as size_t) near
    0.33 m cells, or the exact resolutions of the ring cases."""
    if ring:
        res = 0.5 if n % 2 == 0 else 1.0
        return n * res, res
    for d in range(max(1, round(n * 0.33)), 10 * n):
        res = float(f32(d / n))
        if cells_per_side(d, res) == n:
            return float(d), res
    raise ValueError(n)


_EXPECTED = {}


def expected_points(n):
    """GroundSegmentation::init's table (it depends on N only), from the oracle port."""
    if n not in _EXPECTED:
        from oracle import Oracle

        dim, res = geometry(n)
        _EXPECTED[n] = Oracle(dim, res).expected_points()
    return _EXPECTED[n]


def quotient(m2, points):
    """m2 / (points + FLT_MIN) (:323) in float."""
    with np.errstate(all="ignore"):
        return (np.asarray(m2, np.float32) / (np.asarray(points, np.float32) + FLT_MIN)).astype(np.float32)


def pow2_at_least(x):
    return float(2.0 ** max(0, math.ceil(math.log2(max(float(x), 1.0)))))


class Case:
    def __init__(self, kind, cfg_name, n):
        self.kind, self.cfg_name, self.n = kind, cfg_name, n
        self.dim, self.res = geometry(n, ring=kind.startswith("ring"))
        self.res_f = f32(self.res)
        self.cfg = dict(pyref.DEFAULT_CFG, **CONFIGS[cfg_name])
        self.cfg["patch_size_change_distance"] = min(50.0, 0.3 * n * float(self.res_f))
        self.E = expected_points(n)
        z = lambda v=0.0: np.full((n, n), v, np.float32)   # noqa: E731
        self.planes = dict(points=z(), m2=z(), minGroundHeight=z(FLT_MAX), ground=z(), groundpatch=z(), variance=z())
        self.planted = []
        self.taken = np.zeros((n, n), bool)
        self.hi = 2 * (n // 2) - 2      # detect_ground_patches visits i in [2, hi), j in [2, N - 2) (:325-328)

    @property
    def config(self):
        """The fields of the configuration that differ from GroundGrid.cfg's defaults."""
        return {k: v for k, v in self.cfg.items() if pyref.DEFAULT_CFG.get(k) != v}

    def size(self, i, j):
        return pyref.patch_size(self.n, self.res_f, self.cfg, i, j)

    def vt(self, i, j):
        return pyref.variance_threshold(self.n, self.res_f, self.cfg, i, j)

    def need(self, i, j, S):
        return pyref.min_point_count(self.cfg, S, self.E[i, j])

    def inner(self, i, j):
        return 2 <= i < self.hi and 2 <= j < self.n - 2

    def claim(self, i, j):
        """Reserves the 5 x 5 block around (i, j) if it is free (windows of planted cells never overlap)."""
        if not self.inner(i, j):
            return False
        blk = self.taken[i - 2:i + 3, j - 2:j + 3]
        if blk.any():
            return False
        blk[...] = True
        return True

    def slots(self, S=None):
        """Free centres of the 5-cell lattice, optionally of one window size."""
        for i in range(2, self.hi, 5):
            for j in range(2, self.n - 2, 5):
                if (S is None or self.size(i, j) == S) and not self.taken[i - 2:i + 3, j - 2:j + 3].any() and self.inner(i, j):
                    yield i, j

    def window(self, i, j, S):
        """Cells of the S x S window in Eigen's column-major order: element k = block(k % S, k / S)."""
        h = S // 2
        return [(i - h + k % S, j - h + k // S) for k in range(S * S)]

    # ---- the design window: counts only at the centre (psum, groundlevel and maxVar are then exact) ----------------
    def design(self, i, j, S, outcome, og=None, P=None):
        """Plants the isolated window of cell (i, j) so that it takes `outcome`; returns the centre's count."""
        p = self.planes
        sv = math.sqrt(float(self.vt(i, j)))
        e = float(self.E[i, j])
        og = f32(0.05 * ((i * 7 + j * 3) % 11) - 0.2) if og is None else f32(og)
        gp = self.cfg["ground_patch_detection_minimum_point_count_threshold"]
        if P is None:
            P = pow2_at_least(max(float(self.need(i, j, S)), self.cfg["point_count_cell_variance_threshold"], math.floor(gp * S * e) + 1))
        w = self.window(i, j, S)
        for c in w:
            p["points"][c] = 0.0
            p["m2"][c] = 0.0
            p["variance"][c] = f32(3.0 * sv)
            p["minGroundHeight"][c] = FLT_MAX
        p["ground"][i, j] = og
        tol = abs(self.cfg["outlier_tolerance"])
        q, oc, mc = f32(2.0 * sv), f32(0.25), og + f32(0.5)
        low = None
        if outcome == "need":
            P = 0.0
        elif outcome == "upward":
            oc, mc = f32(0.75), f32(og + f32(tol + 1.0))
        elif outcome == "confident":
            q, oc, mc = f32(0.5 * sv), f32(0.0), og - f32(0.2)
        elif outcome == "localmin":
            low = og - f32(1.0)
        p["points"][i, j] = P
        p["m2"][i, j] = f32(q * f32(P))
        p["minGroundHeight"][i, j] = mc
        if low is not None:
            p["minGroundHeight"][w[0]] = low
        p["groundpatch"][i, j] = oc
        return P

    def plant(self, i, j, outcome, S=None):
        self.planted.append((i, j, self.size(i, j) if S is None else S, outcome))

    def base_lattice(self):
        """One isolated window per outcome and window size, where the map has room."""
        for S in (3, 5):
            free = self.slots(S)
            for outcome in OUTCOMES:
                ij = next(free, None)
                if ij is None:
                    break
                self.claim(*ij)
                self.design(*ij, S, outcome)
                self.plant(*ij, outcome)

    def free_slots(self):
        for ij in list(self.slots()):
            if self.claim(*ij):
                yield ij


# ---- generators ------------------------------------------------------------------------------------------------------
def _random_background(c, rng):
    n = c.n
    p = c.planes
    P = rng.integers(0, 41, (n, n)).astype(np.float32)
    P[rng.uniform(size=(n, n)) < 0.3] = 0.0
    big = rng.uniform(size=(n, n)) < 0.01
    P[big] = rng.integers(41, 8193, big.sum())
    ii, jj = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    di = ii - n / 2.0
    dj = jj - n / 2.0
    sqd = ((di * di + dj * dj) * (float(c.res_f) ** 2)).astype(np.float32).astype(np.float64)
    dfac, mdf = c.cfg["distance_factor"], c.cfg["minimum_distance_factor"]
    vt = np.minimum(np.maximum(sqd * (dfac * dfac), mdf * mdf), (mdf * 10) * (mdf * 10)).astype(np.float32)
    q = (np.sqrt(vt) * 2.0 ** rng.uniform(-1.5, 1.5, (n, n))).astype(np.float32)
    p["points"][...] = P
    p["m2"][...] = q * P
    p["variance"][...] = (q * 2.0 ** rng.uniform(-2, 2, (n, n))).astype(np.float32)
    G = rng.normal(0.0, 0.3, (n, n)).astype(np.float32)
    tol = c.cfg["outlier_tolerance"]
    p["ground"][...] = G
    p["minGroundHeight"][...] = (G + tol * rng.choice([-1.0, 1.0], (n, n)) + rng.normal(0.0, 0.02 + 0.05 * abs(tol), (n, n))).astype(np.float32)
    C = rng.choice(np.array([0.0, 0.5, HALF_UP], np.float32), (n, n))
    u = rng.uniform(size=(n, n)) < 0.2
    C[u] = rng.uniform(0.0, 1.0, u.sum())
    p["groundpatch"][...] = C


def gen_random(c, rng):
    _random_background(c, rng)
    c.base_lattice()


def _equal_after_tol(tol):
    """A float og for which og + tol (double) is a float again: (og, that float)."""
    for k in range(-4, 80):
        og = f32(1.5 * 2.0 ** k)
        t = f64(og) + f64(tol)
        if math.isfinite(t) and f64(f32(t)) == t:
            return og, f32(t)
    raise ValueError(tol)


def _sq_neighbours(vt):
    """The largest float q with q^2 < vt and the smallest with q^2 > vt (squares in double, as :382 takes them)."""
    q = f32(math.sqrt(float(vt)))
    while f64(q) * f64(q) >= f64(vt):
        q = np.nextafter(q, f32(0))
    lo = q
    q = np.nextafter(lo, f32(np.inf))
    while f64(q) * f64(q) <= f64(vt):
        q = np.nextafter(q, f32(np.inf))
    return lo, q


def gen_boundaries(c, rng):
    c.base_lattice()
    p = c.planes
    free = c.free_slots()
    T = c.cfg["point_count_cell_variance_threshold"]
    tol = c.cfg["outlier_tolerance"]
    gp = c.cfg["ground_patch_detection_minimum_point_count_threshold"]
    factor = c.cfg["occupied_cells_point_count_factor"]

    def nxt():
        return next(free, None)

    # psum == need (not skipped) and need - 1 (skipped)
    for d, outcome in ((0, "localmin"), (-1, "need")):
        ij = nxt()
        if ij is None:
            return
        S = c.size(*ij)
        c.design(*ij, S, "localmin", P=float(c.need(*ij, S)) + d)
        c.plant(*ij, outcome)
    # centre count == threshold (its own variance, small: confident) and one below (the window's, large: not)
    for d, outcome in ((0, "confident"), (-1, "localmin")):
        ij = nxt()
        if ij is None:
            return
        i, j = ij
        S = c.size(i, j)
        sv = math.sqrt(float(c.vt(i, j)))
        c.design(i, j, S, "confident")
        K = math.ceil((max(float(c.need(i, j, S)), gp * S * float(c.E[i, j])) + 2) / (S * S - 1))
        for cell in c.window(i, j, S):
            p["points"][cell] = K
            p["m2"][cell] = f32(10.0 * sv) * f32(K)
            p["minGroundHeight"][cell] = p["ground"][i, j] - f32(0.2)
        p["points"][i, j] = T + d
        p["m2"][i, j] = f32(0.5 * sv) * f32(T + d) if T + d != 0 else f32(0.5 * sv) * FLT_MIN
        c.plant(i, j, outcome)
    # groundlevel == ground + outlier_tolerance (double) and its float neighbours, at confidence 0.5 and just above
    og, gl0 = _equal_after_tol(tol)
    for gl in (gl0, np.nextafter(gl0, f32(np.inf)), np.nextafter(gl0, f32(-np.inf))):
        for oc in (f32(0.5), HALF_UP):
            ij = nxt()
            if ij is None:
                return
            S = c.size(*ij)
            c.design(*ij, S, "unchanged", og=og)
            p["minGroundHeight"][ij] = gl
            p["groundpatch"][ij] = oc
            if f64(oc) > 0.5 and f64(gl) >= f64(og) + f64(tol):
                outcome = "upward"
            else:
                outcome = "localmin" if gl < og else "unchanged"
            c.plant(*ij, outcome)
    # maxVar^2 just below / above vt; maxVar 0, -0, denormal
    for which in ("below", "above", "zero", "negzero", "denormal"):
        ij = nxt()
        if ij is None:
            return
        S = c.size(*ij)
        P = c.design(*ij, S, "confident")
        lo, hi = _sq_neighbours(c.vt(*ij))
        q = dict(below=lo, above=hi, zero=f32(0.0), negzero=f32(-0.0), denormal=DENORM)[which]
        p["m2"][ij] = f32(q * f32(P))
        c.plant(*ij, "confident" if which in ("below", "denormal") else "localmin")
    # psum == occupied_cells_point_count_factor: the nc = 1 shortcut of the confident branch
    if f64(f32(factor)) == f64(factor):
        for ij in list(c.slots()):
            S = c.size(*ij)
            if factor >= c.need(*ij, S) and factor > gp * S * float(c.E[ij]) and c.claim(*ij):
                c.design(*ij, S, "confident", P=factor)
                c.plant(*ij, "confident")
                break
    # localmin == ground: no update
    ij = nxt()
    if ij is None:
        return
    S = c.size(*ij)
    c.design(*ij, S, "unchanged")
    p["minGroundHeight"][c.window(*ij, S)[0]] = p["ground"][ij]
    c.plant(*ij, "unchanged")


def gen_nonfinite(c, rng):
    c.base_lattice()
    p = c.planes
    free = c.free_slots()
    # a NaN heading a later column with the strict minimum further down it: the minimum counts (:373); one at
    # element 0: the window minimum is that NaN
    for head in (1, 0):
        for ij in (next(free, None), ):
            if ij is None:
                return
            i, j = ij
            S = c.size(i, j)
            c.design(i, j, S, "unchanged")
            w = c.window(i, j, S)
            p["minGroundHeight"][w[head * S]] = np.nan
            p["minGroundHeight"][w[(S - 1) * S + 2 if head == 0 else S + 2]] = p["ground"][i, j] - f32(1.0)
            c.plant(i, j, "localmin" if head else "unchanged")
    values = (f32(np.nan), f32(np.inf), f32(-np.inf), f32(-0.0), FLT_MAX, DENORM)
    k = 0
    for plane in ("minGroundHeight", "points", "m2", "ground", "groundpatch", "variance"):
        for v in values:
            for where in ("first", "head", "centre", "last"):
                ij = next(free, None)
                if ij is None:
                    return
                i, j = ij
                S = c.size(i, j)
                c.design(i, j, S, ("confident", "localmin", "upward")[k % 3])
                k += 1
                w = c.window(i, j, S)
                if plane in ("ground", "groundpatch"):
                    cell = (i, j)
                else:
                    cell = w[dict(first=0, head=S, centre=S * S // 2, last=S * S - 1)[where]]
                    if where == "head" and plane == "minGroundHeight":
                        p["minGroundHeight"][w[S + 1]] = p["ground"][i, j] - f32(0.5)
                p[plane][cell] = v
                c.plant(i, j, None)


def gen_fractional(c, rng):
    c.base_lattice()
    p = c.planes
    odd = np.array([0.5, 0.25, 1.75, -2.5, -0.75, 3.3, 1e7 + 0.5, 2.0 ** 24, 2.0 ** 24 + 2, 3 * 2.0 ** 23, 1.0, 1.0], np.float32)
    for k, ij in enumerate(c.free_slots()):
        if k >= 60:
            break
        i, j = ij
        S = c.size(i, j)
        c.design(i, j, S, "confident")
        sv = math.sqrt(float(c.vt(i, j)))
        for cell in c.window(i, j, S):
            P = odd[rng.integers(0, len(odd))] if rng.uniform() < 0.7 else f32(rng.uniform(-3, 40))
            p["points"][cell] = P
            p["m2"][cell] = f32(f32(rng.uniform(0.2, 0.6) * sv) * P)
            p["minGroundHeight"][cell] = p["ground"][i, j] - f32(rng.uniform(-0.3, 0.3))
        c.plant(i, j, None)


def gen_cap(c, rng):
    """Early-skip bounds above 2^24: a window summing to a float just below the bound is skipped, one summing to the
    bound rounded up to float is not."""
    c.base_lattice()
    for ij in list(c.slots()):
        S = c.size(*ij)
        need = float(c.need(*ij, S))
        if not 2.0 ** 24 + 4 < need < 2.0 ** 30 or not c.claim(*ij):
            continue
        up = float(np.nextafter(f32(need), f32(np.inf))) if float(f32(need)) < need else float(f32(need))
        below = float(np.nextafter(f32(need), f32(0))) if float(f32(need)) >= need else float(f32(need))
        P = below if len([p for p in c.planted if p[3] == "need"]) % 2 == 0 else up
        c.design(*ij, S, "localmin", P=P)
        c.plant(*ij, "need" if P < need else "localmin")
        if len(c.planted) >= 20:
            break


def _ring_distance(c):
    """A target cell about 0.3 N from the centre and a distance whose double square equals its sqdist exactly."""
    n = c.n
    for off in range(max(1, int(0.3 * n)), 1, -1):
        i, j = n // 2 + off, n // 2 + off // 3
        if not c.inner(i, j):
            continue
        di, dj = f64(i) - f64(n) / 2.0, f64(j) - f64(n) / 2.0
        t = f64(f32((di * di + dj * dj) * (f64(c.res_f) * f64(c.res_f))))
        psc = math.sqrt(t)
        for _ in range(8):
            if psc * psc == t:
                return t, psc
            psc = math.nextafter(psc, math.inf if psc * psc < t else -math.inf)
    return None, None


def gen_ring(c, rng, shift):
    t, psc = _ring_distance(c)
    if t is not None:
        c.cfg["patch_size_change_distance"] = {0: psc, 1: math.nextafter(psc, math.inf), -1: math.nextafter(psc, -math.inf)}[shift]
        p = c.planes
        n = c.n
        for i in range(2, c.hi):
            for j in range(2, n - 2):
                di, dj = f64(i) - f64(n) / 2.0, f64(j) - f64(n) / 2.0
                if f64(f32((di * di + dj * dj) * (f64(c.res_f) * f64(c.res_f)))) != t or not c.claim(i, j):
                    continue
                S = c.size(i, j)
                c.design(i, j, 5, "localmin", P=0.0)
                need5 = float(c.need(i, j, 5))
                for cell in c.window(i, j, 5):
                    if max(abs(cell[0] - i), abs(cell[1] - j)) == 2:   # the outer ring only: a 3 x 3 window sees none
                        p["points"][cell] = math.ceil(need5 / 16.0) + 1
                c.plant(i, j, "need" if S == 3 else "localmin", S)
    c.base_lattice()


GENERATORS = {"random": gen_random, "boundaries": gen_boundaries, "nonfinite": gen_nonfinite, "fractional": gen_fractional, "cap": gen_cap,
              "ring": lambda c, r: gen_ring(c, r, 0), "ring+": lambda c, r: gen_ring(c, r, 1), "ring-": lambda c, r: gen_ring(c, r, -1)}


def make_case(kind, cfg_name, n, seed=0):
    c = Case(kind, cfg_name, n)
    GENERATORS[kind](c, np.random.default_rng(1000 * n + 17 * seed + CASES.index((kind, cfg_name))))
    return c


def cases(n):
    for kind, cfg_name in CASES:
        yield make_case(kind, cfg_name, n)


def window_limit_cells(n):
    """(S, i, j) at the limits detect_ground_patch<S> accepts: i or j = S / 2 and N - S / 2 - 1."""
    out = []
    for S in (3, 5):
        h = S // 2
        lo, hi, mid = h, n - h - 1, n // 2
        for i, j in ((lo, lo), (lo, hi), (hi, lo), (hi, hi), (lo, mid), (mid, hi)):
            out.append((S, i, j))
    return out


def outcome(c, i, j, S, planes=None):
    """The branch pyref's one-cell restatement takes at (i, j) on the case's planes, with the variance
    detect_ground_patches computes first; (outcome, ground, groundpatch) of the cell afterwards."""
    p = c.planes if planes is None else planes
    G = p["ground"].copy()
    C = p["groundpatch"].copy()
    var = quotient(p["m2"], p["points"])
    r = pyref.detect_cell(p["points"], var, p["minGroundHeight"], G, C, c.E, i, j, S, c.cfg, c.res_f)
    return r, G[i, j], C[i, j]

"""Point orders, cell densities, non-finite heights and far map positions for the rasteriser's order recovery.

k_rasterize turns the kept points of a warp (32 consecutive input points) that share a cell into one run, k_scatter
files the runs of a cell in arrival order and k_cell_stats has to put them back into input order before the fp32
Welford recurrence, whose last bits depend on that order.  groundgrid_b200/synth.py only emits ring-major clouds; the
generators here re-order such clouds, or build clouds from the cell centres of the map under test, so that a cell gets a
chosen number of runs and points.  run_profile() counts what a cloud really feeds (plain numpy, no GPU), and the tests
assert the regime with it before they compare anything.

Re-orderings return (cloud, perm) with cloud == points[perm]; constructed clouds return (cloud, origin, targets).
"""
import numpy as np

from groundgrid_b200 import synth

POINT_DTYPE = synth.POINT_DTYPE
FIELDS = ("x", "y", "z", "intensity", "ring")
RUNS_LADDER = (1, 2, 7, 8, 9, 10, 11, 22, 23, 24, 56, 57, 58, 59, 120)
COUNT_LADDER = (1, 31, 32, 33, 40, 63, 64, 65, 255, 256, 1000, 8192)
MAX_POINTS_PER_CELL, MAX_RUNS_PER_CELL = 8192, 2048   # nothing here goes beyond: one thread walks one cell
RUN_BANDS = ((1, 1), (2, 8), (9, 23), (24, 57), (58, None))
COUNT_BANDS = ((1, 32), (33, 6143), (6144, None))


def take(points, perm):
    """points[perm] as 32-byte records (fancy indexing keeps the padded dtype, the copy makes it contiguous)."""
    out = np.zeros(len(perm), POINT_DTYPE)
    for f in FIELDS:
        out[f] = points[f][perm]
    return out


# ---- the map's arithmetic, as grid_map does it (fp64 on the widened float resolution) --------------------------------
def cell_index(points, n, res, position):
    """Flat cell (i + j * n) of every point, n * n for a point outside the map or with a non-finite x / y."""
    r = float(np.float32(res))
    length, half = n * r, 0.5 * (n * r)
    x, y = points["x"].astype(np.float64), points["y"].astype(np.float64)
    with np.errstate(invalid="ignore"):
        tx, ty = -(x - position[0] - half), -(y - position[1] - half)
        inside = (tx >= 0.0) & (ty >= 0.0) & (tx < length) & (ty < length)
        vi = np.where(inside, np.trunc((x - half - position[0]) / r), 1.0)
        vj = np.where(inside, np.trunc((y - half - position[1]) / r), 1.0)
    i, j = -vi.astype(np.int64), -vj.astype(np.int64)
    inside &= (i >= 0) & (j >= 0) & (i < n) & (j < n)
    return np.where(inside, i + j * n, n * n)


def cell_centre(i, j, n, res, position):
    r = float(np.float32(res))
    off = 0.5 * (n * r) - 0.5 * r
    return (position[0] + off) + r * -np.asarray(i, np.float64), (position[1] + off) + r * -np.asarray(j, np.float64)


def kept_mask(points, origin, n, res, position, max_ring=1024):
    """Points the rasteriser accumulates, short of the outlier ray-march (none on a fresh map): inside, ring within
    max_ring, at least sqrt(12) m from the origin."""
    dx = (points["x"] - np.float32(origin[0])).astype(np.float64)
    dy = (points["y"] - np.float32(origin[1])).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        far = (dx * dx + dy * dy).astype(np.float32) >= np.float32(12.0)
    return (cell_index(points, n, res, position) < n * n) & (points["ring"].astype(np.int64) <= max_ring) & far


class Profile:
    """count[cell], runs[cell]; per run its length and whether its lanes are not consecutive ones."""

    def __init__(self, count, runs, run_len, run_cell, run_first_lane, run_split):
        self.count, self.runs = count, runs
        self.run_len, self.run_cell, self.run_first_lane, self.run_split = run_len, run_cell, run_first_lane, run_split

    def bands(self):
        def band(a, bounds):
            return {f"{lo}" + ("" if hi == lo else f"-{hi}" if hi else "+"): int(((a >= lo) & (a <= (hi or a.max() + 1))).sum())
                    for lo, hi in bounds}

        return {"runs": band(self.runs, RUN_BANDS), "points": band(self.count, COUNT_BANDS)}

    def __str__(self):
        b = self.bands()
        return (f"cells by runs {b['runs']}, by points {b['points']}; max {self.runs.max()} runs, {self.count.max()} points; "
                f"{int(self.run_split.sum())} of {len(self.run_len)} runs on non-consecutive lanes, {int((self.run_len == 32).sum())} full-warp runs")


def run_profile(points, origin, n, res, position, max_ring=1024, kept=None):
    """Per cell the number of kept points and of runs: groups of (point index >> 5, cell).  `kept` overrides the
    kept_mask() approximation (e.g. when the scan has outliers)."""
    if kept is None:
        kept = kept_mask(points, origin, n, res, position, max_ring)
    idx = np.nonzero(kept)[0]
    cell = cell_index(points, n, res, position)[idx]
    assert (cell < n * n).all()
    key = (idx >> 5) * (n * n) + cell            # ascending idx inside a key: the sort below is stable
    order = np.argsort(key, kind="stable")
    ks = key[order]
    first = np.nonzero(np.r_[True, ks[1:] != ks[:-1]])[0] if len(ks) else np.zeros(0, np.int64)
    length = np.diff(np.r_[first, len(ks)])
    lane = (idx & 31)[order]
    run_cell = (ks[first] % (n * n)).astype(np.int64)
    first_lane = lane[first]
    split = (lane[first + length - 1] - first_lane + 1) != length if len(first) else np.zeros(0, bool)
    return Profile(np.bincount(cell, minlength=n * n), np.bincount(run_cell, minlength=n * n), length, run_cell, first_lane, split)


# ---- re-orderings of an existing cloud --------------------------------------------------------------------------
def firing(points, origin):
    """Azimuth-major with the ring fastest: the order in which a spinning sensor's driver emits its returns."""
    with np.errstate(invalid="ignore"):
        az = np.arctan2(points["y"].astype(np.float64) - origin[1], points["x"].astype(np.float64) - origin[0])
    perm = np.lexsort((points["ring"], az))
    return take(points, perm), perm


def shuffled(points, seed):
    perm = np.random.default_rng(seed).permutation(len(points))
    return take(points, perm), perm


def reversed_order(points):
    perm = np.arange(len(points))[::-1].copy()
    return take(points, perm), perm


def _rank_in_cell(cell, order):
    """Position of every point among the points of its cell, in input order (order = stable argsort of cell)."""
    cs = cell[order]
    first = np.nonzero(np.r_[True, cs[1:] != cs[:-1]])[0]
    rank = np.empty(len(cell), np.int64)
    rank[order] = np.arange(len(cell)) - np.repeat(first, np.diff(np.r_[first, len(cs)]))
    return rank


def cell_sorted(points, n, res, position):
    """All points of a cell next to each other (points outside the map last): the fewest runs a cloud can have."""
    perm = np.argsort(cell_index(points, n, res, position), kind="stable")
    return take(points, perm), perm


def cell_round_robin(points, n, res, position):
    """The points of a cell dealt to different warps, one each, so that every run has length 1 and a cell has as many
    runs as points.  Needs no cell with more points than the cloud has full warps."""
    cell = cell_index(points, n, res, position)
    order = np.argsort(cell, kind="stable")
    warps = len(points) // 32
    assert np.bincount(cell[cell < n * n]).max() <= warps
    cs = cell[order]
    tail = np.nonzero(np.r_[True, cs[1:] != cs[:-1]])[0][:len(points) - 32 * warps]   # the last, partial warp: one point of as many cells
    body = np.delete(order, tail)
    t = np.arange(32 * warps)
    perm = np.r_[body[np.lexsort((t // warps, t % warps))], order[tail]]
    return take(points, perm), perm


def two_cell_alternation(points, n, res, position):
    """Cells paired by size, the points of a pair interleaved A B A B ..: every run sits on every second lane."""
    cell = cell_index(points, n, res, position)
    order = np.argsort(cell, kind="stable")
    rank = _rank_in_cell(cell, order)
    ids, inv, counts = np.unique(cell, return_inverse=True, return_counts=True)
    by_size = np.empty(len(ids), np.int64)
    by_size[np.argsort(-counts, kind="stable")] = np.arange(len(ids))
    place = by_size[inv]                       # 0 = the largest cell
    pair, side = place // 2, place % 2
    partner = np.minimum(place | 1, len(ids) - 1)
    b = counts[np.argsort(-counts, kind="stable")][partner]   # size of the pair's smaller cell (B)
    sub = np.where(rank < b, 2 * rank + side, b + rank)
    perm = np.lexsort((sub, pair))
    return take(points, perm), perm


REORDERINGS = ("firing", "shuffled", "reversed", "cell_sorted", "cell_round_robin", "two_cell_alternation")


def reorder(name, points, origin, n, res, position=(0.0, 0.0), seed=0):
    """(cloud, perm) of the re-ordering `name`."""
    if name == "firing":
        return firing(points, origin)
    if name == "shuffled":
        return shuffled(points, seed)
    if name == "reversed":
        return reversed_order(points)
    return {"cell_sorted": cell_sorted, "cell_round_robin": cell_round_robin,
            "two_cell_alternation": two_cell_alternation}[name](points, n, res, position)


# ---- clouds built from the cell centres of the map under test --------------------------------------------------------
def _origin(position):
    return np.array([position[0], position[1], synth.SENSOR_HEIGHT], np.float32)


def _target_cells(count, n, res, rng):
    """`count` distinct cells, two cells apart at least, clear of the border and of the 12 m^2 disc around the centre."""
    clear = int(np.ceil(np.sqrt(12.0) / res)) + 2
    ii, jj = np.meshgrid(np.arange(4, n - 4, 2), np.arange(4, n - 4, 2), indexing="ij")
    ok = (np.abs(ii - n // 2) >= clear) | (np.abs(jj - n // 2) >= clear)
    cand = np.stack([ii[ok], jj[ok]], 1)
    assert len(cand) >= count, "map too small for the ladder"
    return cand[rng.permutation(len(cand))[:count]]


def _heights(count, oz, rng):
    """Heights whose Welford result depends on the order (magnitudes alternate over three decades, signs are random);
    about one in nine equals the origin's z, where the recurrence restarts its mean."""
    mag = np.where(np.arange(count) % 2 == 0, rng.uniform(0.5, 3.0, count), rng.uniform(1e-3, 5e-3, count))
    pd = (mag * rng.choice([-1.0, 1.0], count)).astype(np.float32)
    z = (np.float32(oz) + pd).astype(np.float32)
    z[rng.uniform(size=count) < 0.11] = np.float32(oz)
    if count > 2:
        z[0] = z[2] = np.float32(oz)          # a restart at the head of the cell and one in the middle
    return z


def _assemble(slots, cells, n, res, position, seed):
    """slots[p] = index into `cells` of record p (-1: a filler outside the map, which no phase keeps)."""
    rng = np.random.default_rng(seed + 1)
    org = _origin(position)
    pts = np.zeros(len(slots), POINT_DTYPE)
    r = float(np.float32(res))
    pts["x"] = np.float32(position[0] + n * r)         # fillers: half a map length beyond the edge
    pts["y"] = np.float32(position[1])
    pts["z"] = rng.uniform(-1.0, 1.0, len(slots)).astype(np.float32)
    pts["intensity"] = rng.uniform(size=len(slots)).astype(np.float32)
    pts["ring"] = rng.integers(0, 64, len(slots))
    used = slots >= 0
    cx, cy = cell_centre(cells[slots[used], 0], cells[slots[used], 1], n, res, position)
    pts["x"][used], pts["y"][used] = cx.astype(np.float32), cy.astype(np.float32)
    for t in range(len(cells)):
        mine = np.nonzero(slots == t)[0]
        pts["z"][mine] = _heights(len(mine), org[2], rng)
    flat = cells[:, 0] + cells[:, 1] * n
    assert len(set(flat.tolist())) == len(flat)
    assert np.array_equal(cell_index(pts, n, res, position)[used], flat[slots[used]]), "a rounded cell centre left its cell"
    return pts, org, flat


def runs_ladder(n, res, position=(0.0, 0.0), seed=0, warps=256):
    """One target cell per entry of RUNS_LADDER with exactly that many runs (its points sit in that many distinct
    warps), plus cells made of full-warp (32) and 31-point runs.  Run lengths cover 1, 2, 3, 31 and 32, heads sit on lane 0,
    on lane 31 and in between, and most runs are on non-consecutive lanes.  The warps of a cell are a seeded random
    subset of all warps, so its runs are spread over the blocks and rounds of the rasteriser and do not arrive in
    ascending order.  Returns (cloud, origin, {runs: [cells]})."""
    rng = np.random.default_rng(seed)
    wide = ((2, (32, 31)), (7, (32, 31, 32, 31, 32, 31, 32)), (9, (31, 32, 31, 32, 31, 32, 31, 32, 31)))
    cells = _target_cells(len(RUNS_LADDER) + len(wide), n, res, rng)
    slots = np.full((warps, 32), -1, np.int64)
    free_warps = list(rng.permutation(warps))
    targets = {}
    for t, (k, lengths) in enumerate(wide):            # whole warps first
        for length in lengths:
            w = free_warps.pop()
            slots[w, 32 - length:] = t                  # a 31-point run leaves lane 0 to another cell
        targets.setdefault(k, []).append(t)
    for q, k in enumerate(RUNS_LADDER):
        t = len(wide) + q
        assert k <= warps
        roomy = [w for w in rng.permutation(warps) if (slots[w] < 0).sum() >= 3][:k]   # not the warps of the wide runs
        assert len(roomy) == k
        for r, w in enumerate(roomy):
            length = (1, 2, 3, 1)[r % 4]
            free = np.nonzero(slots[w] < 0)[0]
            want = free[free == {0: 0, 3: 31}.get(r, -1)]
            slots[w, want if len(want) else rng.choice(free, length, replace=False)] = t
        targets.setdefault(k, []).append(t)
    pts, org, flat = _assemble(slots.ravel(), cells, n, res, position, seed)
    return pts, org, {k: [int(flat[t]) for t in ts] for k, ts in targets.items()}


def count_ladder(n, res, position=(0.0, 0.0), seed=0, scattered=False, records=40960):
    """One cell per entry of COUNT_LADDER with exactly that many points: around the 32 / 33 step of the cell worklist's
    classes, and one beyond the 6 144 points of its last class.  scattered=False: each cell one contiguous block (the
    fewest runs); True: the points of all cells dealt at random over `records` records (the 8 192-point cell then has a
    run in nearly every warp: records / 32 <= MAX_RUNS_PER_CELL).  Returns (cloud, origin, {count: cell})."""
    rng = np.random.default_rng(seed)
    assert records // 32 <= MAX_RUNS_PER_CELL and max(COUNT_LADDER) <= MAX_POINTS_PER_CELL and records >= sum(COUNT_LADDER) + 64
    cells = _target_cells(len(COUNT_LADDER), n, res, rng)
    slots = np.full(records, -1, np.int64)
    body = np.repeat(np.arange(len(COUNT_LADDER)), COUNT_LADDER)
    if scattered:
        slots[rng.permutation(records)[:len(body)]] = body
    else:
        slots[7:7 + len(body)] = body                   # off the warp boundary: blocks start on every lane
    pts, org, flat = _assemble(slots, cells, n, res, position, seed)
    return pts, org, {c: int(flat[t]) for t, c in enumerate(COUNT_LADDER)}


def nonfinite_heights(points, seed, every=1000):
    """A copy of `points` with NaN, +inf and -inf heights at seeded positions (x and y stay finite), some of them with a
    ring above any max_ring, and -inf / very low heights among points that a prior would test as outliers."""
    rng = np.random.default_rng(seed)
    out = points.copy()
    idx = rng.choice(len(out), 3 * (len(out) // every), replace=False)
    a, b, c = np.array_split(idx, 3)
    out["z"][a], out["z"][b], out["z"][c] = np.nan, np.inf, -np.inf
    low = rng.choice(len(out), len(out) // every, replace=False)
    out["z"][low] -= rng.uniform(0.25, 2.0, len(low)).astype(np.float32)     # -inf stays -inf, NaN stays NaN
    out["ring"][idx[::7]] = 2000
    return out


def far_scene(position, seed=1234, **kw):
    """synth.make_scene() moved to `position`."""
    scene = synth.make_scene(seed=seed, **kw)
    scene.boxes[:, [0, 3]] += position[0]
    scene.boxes[:, [1, 4]] += position[1]
    return scene


def coarse_far_cloud(position, seed=1234, scene_seed=1234, **kw):
    """A 64-beam scan of a scene around `position`: far from the origin float32 coordinates are coarse (0.008 m apart
    at 1.2e5, 0.5 m at 5.6e6), so many points share a coordinate pair and sit exactly on cell edges."""
    return synth.scan_64(far_scene(position, scene_seed), ego_xy=position, seed=seed, **kw)

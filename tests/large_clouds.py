"""Clouds at the sizes a handle accepts: up to 2^26 - 256 points per cloud, cells with more than 2^24 points, maps of
4094 .. 4096 cells per side.

Below these sizes some code paths never run:
  * the output scan (k_out_scan) scans 3 * nblk block counts, nblk = ceil(points / 1024), in tiles of 4096 and carries a
    running total from one tile to the next: a scan of more than TILE_EDGE = 1 397 760 points needs two tiles, one of
    more than 2 * TILE_EDGE three;
  * the reference counts "pointsRaw" and "points" up by 1.0f, which stops at 2^24; a cell past 2^24 points shows where
    the CUDA path's integer counters have to stop as well;
  * the point code keeps the cell in 24 bits: at N = 4096 that field is full, from N = 2897 on bit 23 is set.
The generators are seeded and vectorised (plain numpy, no GPU), like tests/cloud_orders.py.  Large counts only ever go
into cells of ignored points: a kept cell stays within MAX_POINTS_PER_CELL points and MAX_RUNS_PER_CELL runs, because one
thread walks one kept cell serially.  kept_cell_bounds() measures that for any cloud.
"""
import numpy as np

import cloud_orders as co
import ref_scenarios as rs
from groundgrid_b200 import synth

POINT_DTYPE = synth.POINT_DTYPE
OUT_TILE, SCAN_TILE = 1024, 4096          # points per block count of the output scan, counts per tile of its scan
TILE_EDGE = SCAN_TILE // 3 * OUT_TILE      # 1 397 760: the largest scan whose three classes' block counts fit one tile
BOUNDARY_SIZES = (TILE_EDGE, TILE_EDGE + 1, 2 * TILE_EDGE, 2 * TILE_EDGE + 1, 3_000_000)
FLOAT_STOP = 1 << 24                       # counting up by 1.0f from 0 stops here
PILE_SIZES = (FLOAT_STOP - 1, FLOAT_STOP, FLOAT_STOP + 1, FLOAT_STOP + 2, FLOAT_STOP + 3, 1 << 25)
CAPACITY = (1 << 26) - 256                 # the most points gg_create accepts per cloud
MAX_RING_IGNORED = 2000                    # a ring above the default max_ring (1024): the point is ignored
# (dimension, resolution) of the largest maps; tests check each N with gg_host_cells_per_side
WIDE_GEOMETRIES = {4096: (2048.0, 0.5), 4095: (1365.0, 1.0 / 3.0), 4094: (1351.0, 0.33)}
BOUNDARY_GEOMETRY = (99.0, 0.33)           # N = 300
PILE_GEOMETRY = (33.0, 0.33)               # N = 100
CAPACITY_GEOMETRIES = {300: (99.0, 0.33), 4096: (2048.0, 0.5)}


def out_scan_tiles(n_points):
    """Tiles the output scan of a launch whose largest scan has n_points points runs over."""
    nblk = max(1, -(-n_points // OUT_TILE))
    return -(-3 * nblk // SCAN_TILE)


def concat(parts):
    """Point arrays joined into one of 32-byte records (np.concatenate would keep the padded dtype, but copies field by
    field anyway)."""
    out = np.zeros(sum(len(p) for p in parts), POINT_DTYPE)
    at = 0
    for p in parts:
        for f in co.FIELDS:
            out[f][at:at + len(p)] = p[f]
        at += len(p)
    return out


def kept_cell_bounds(points, origin, n, res, position=(0.0, 0.0), kept=None):
    """(most points, most runs) of any kept cell.  `kept` overrides cloud_orders.kept_mask (e.g. the classes a scan
    reported, which also leave out the outliers)."""
    prof = co.run_profile(points, origin, n, res, position, kept=kept)
    return int(prof.count.max(initial=0)), int(prof.runs.max(initial=0))


# ---- the output order -------------------------------------------------------------------------------------------------
SELECT_GROUND, SELECT_NONGROUND = 1, 2
SELECTS = {"all": SELECT_GROUND | SELECT_NONGROUND, "ground": SELECT_GROUND, "nonground": SELECT_NONGROUND}


def output_order(classes, labels, select=SELECTS["all"]):
    """The input index of every output point: kept points, then ignored points, then outliers, each in input order (a
    stable 3-way partition); points in border cells and outside the map are not part of it; `select` keeps the points
    whose label it names (outliers are ground).  classes: the point classes of gg_get_point_classes (codes >> 24) or of
    the oracle's filter_cloud(want_classes=True)."""
    classes = np.asarray(classes)
    part = np.select([classes == 1, classes == 3, classes == 5], [0, 1, 2], -1)
    bit = np.where(labels == 99, SELECT_NONGROUND, SELECT_GROUND)
    part[(bit & select) == 0] = -1
    idx = np.nonzero(part >= 0)[0]
    return idx[np.argsort(part[idx], kind="stable")].astype(np.uint32)


# ---- clouds across the tile edges of the output scan ---------------------------------------------------------------------
def boundary_scene():
    return synth.make_scene(seed=2600)


def prior_scan():
    """The ordinary scan that builds the prior the boundary clouds' outliers are tested against: (points, origin)."""
    return synth.scan_64(boundary_scene(), seed=2601)


BOUNDARY_SENSORS = tuple((dx, dy, synth.SENSOR_HEIGHT, 45.0 * k) for k, (dx, dy) in
                         enumerate(((15.0, 0.0), (-15.0, 0.0), (0.0, 15.0), (0.0, -15.0),
                                    (25.0, 25.0), (-25.0, 25.0), (25.0, -25.0), (-25.0, -25.0))))


def boundary_cloud(n_points, seed=0):
    """Eight 64-beam sensors spread over the map (so that no kept cell gets too many points) scanning boundary_scene()
    with as many azimuth steps as it takes to return n_points points, cut to exactly n_points.  About 10 % of the
    points, drawn at random, get a ring above max_ring (ignored) and about 1 % are pushed below the ground (outliers on
    the prior of prior_scan()), so the three output classes are interleaved all over the cloud and each class's block
    counts cross the tile edges of the output scan.  Returns (points, origin)."""
    az = int(np.ceil(n_points / (64 * 0.9 * len(BOUNDARY_SENSORS))))
    pts, org = synth.scan_64(boundary_scene(), seed=2700 + seed, az_steps=az, sensors=BOUNDARY_SENSORS)
    assert len(pts) >= n_points, (len(pts), n_points)
    pts = co.take(pts, np.arange(n_points))
    rng = np.random.default_rng(2800 + seed)
    pts["ring"][rng.uniform(size=n_points) < 0.1] = MAX_RING_IGNORED
    rs.push_below_ground(pts, n_points // 100, 2900 + seed)
    return pts, org


# ---- piles: one inner cell with more points than a float count reaches ----------------------------------------------------
PILE_CELLS = {"ring": (20, 70), "near": (48, 47)}   # N = 100: a cell far from the centre, one within sqrt(12) m of it


def pile(count, how="ring", seed=0):
    """A small ordinary scan (a few hundred kept points) followed by `count` points in one inner cell of a
    PILE_GEOMETRY map, all of them ignored: how="ring" gives them a ring above max_ring, how="near" puts the cell
    within sqrt(12) m of the origin (their rings 0 .. 63 are then tallied by the evaluation).  All but one of the piled
    points are 3 m above the ground, so more than 2^24 of them are obstacles once count > 2^24 + 1; the one in the
    middle is 1 m below it.  Returns (points, origin, flat cell, piled non-ground count)."""
    dim, res = PILE_GEOMETRY
    n = 100
    scene = synth.make_scene(seed=3000 + seed, n_boxes=6, rmin=4.0, rmax=14.0)
    scan, org = synth.lidar_scan(scene, beams=8, az_steps=64, seed=3000 + seed)
    i, j = PILE_CELLS[how]
    cx, cy = co.cell_centre(i, j, n, res, (0.0, 0.0))
    p = np.zeros(count, POINT_DTYPE)
    p["x"], p["y"] = np.float32(cx), np.float32(cy)
    p["z"] = np.float32(3.0)
    p["z"][count // 2] = np.float32(-1.0)
    p["intensity"] = np.float32(0.25)
    if how == "ring":
        p["ring"] = MAX_RING_IGNORED
    else:
        p["ring"] = np.random.default_rng(3100 + seed).integers(0, 64, count, dtype=np.uint16)
    cloud = concat([scan, p])
    return cloud, org, i + j * n, count - 1


# ---- the largest cloud a handle takes ---------------------------------------------------------------------------------
def capacity_cloud(n, seed=0, count=CAPACITY):
    """`count` points spread at random over the inner cells of the CAPACITY_GEOMETRIES[n] map (a kept cell gets a few
    hundred points on N = 300 and a few on N = 4096; every point a run of its own at worst), with about 5 % ignored
    (ring above max_ring), heights on and 2 m above a flat ground.  Returns (points, origin)."""
    dim, res = CAPACITY_GEOMETRIES[n]
    rng = np.random.default_rng(4000 + seed)
    r = float(np.float32(res))
    half = 0.5 * n * r - 1.5 * r
    pts = np.zeros(count, POINT_DTYPE)
    pts["x"] = rng.uniform(-half, half, count).astype(np.float32)
    pts["y"] = rng.uniform(-half, half, count).astype(np.float32)
    z = rng.normal(0.0, 0.03, count).astype(np.float32)
    z[rng.uniform(size=count) < 0.15] += np.float32(2.0)
    pts["z"] = z
    del z
    pts["intensity"] = np.float32(0.5)
    ring = rng.integers(0, 64, count, dtype=np.uint16)
    ring[rng.uniform(size=count) < 0.05] = MAX_RING_IGNORED
    pts["ring"] = ring
    return pts, np.array([0.0, 0.0, synth.SENSOR_HEIGHT], np.float32)


# ---- whole-map sprinkles on the largest maps ----------------------------------------------------------------------------
def sprinkle_cells(n, seed=0, extra=20000):
    """(i, j) of the cells a sprinkle puts points into: every cell of the border rows and columns (the four corners
    with them), the last inner cell, cells whose flat index has bit 23 set (when the map has any), the last cell, and
    `extra` cells at random."""
    rng = np.random.default_rng(5000 + seed)
    k = np.arange(n)
    edge = np.concatenate([np.stack([k, np.zeros_like(k)], 1), np.stack([k, np.full_like(k, n - 1)], 1),
                           np.stack([np.zeros_like(k), k], 1), np.stack([np.full_like(k, n - 1), k], 1)])
    special = [(n - 4, n - 4), (n - 1, n - 1), (0, 0), (n - 1, 0), (0, n - 1)]
    cells = [edge, np.array(special)]
    if n * n > 1 << 23:
        flat = rng.integers(1 << 23, n * n, 2000)
        cells.append(np.stack([flat % n, flat // n], 1))
        first = 1 << 23                                      # the first cell with bit 23 set
        cells.append(np.array([[first % n, first // n]]))
    cells.append(rng.integers(0, n, (extra, 2)))
    return np.unique(np.concatenate(cells), axis=0)


def sprinkle(n, position=(0.0, 0.0), seed=0, per_cell=3):
    """per_cell points at the centre of every sprinkle_cells() cell of the WIDE_GEOMETRIES[n] map at `position`, cells in
    a seeded random order, heights mixed on and 1.5 m above the ground, a few ignored by ring.  Returns (points, origin,
    cells)."""
    dim, res = WIDE_GEOMETRIES[n]
    rng = np.random.default_rng(5100 + seed)
    cells = sprinkle_cells(n, seed)
    cells = cells[rng.permutation(len(cells))]
    ci = np.repeat(cells[:, 0], per_cell)
    cj = np.repeat(cells[:, 1], per_cell)
    cx, cy = co.cell_centre(ci, cj, n, res, position)
    pts = np.zeros(len(ci), POINT_DTYPE)
    pts["x"], pts["y"] = cx.astype(np.float32), cy.astype(np.float32)
    z = rng.normal(0.0, 0.02, len(ci)).astype(np.float32)
    z[rng.uniform(size=len(ci)) < 0.2] += np.float32(1.5)
    pts["z"] = z
    pts["intensity"] = rng.uniform(size=len(ci)).astype(np.float32)
    ring = rng.integers(0, 64, len(ci), dtype=np.uint16)
    ring[rng.uniform(size=len(ci)) < 0.03] = MAX_RING_IGNORED
    pts["ring"] = ring
    org = np.array([position[0], position[1], synth.SENSOR_HEIGHT], np.float32)
    return pts, org, cells

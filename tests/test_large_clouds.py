"""tests/large_clouds.py without a GPU: every cloud reaches the size it is named for and keeps its kept cells within the
band one thread walks; the oracle's "pointsRaw" and "points" stop at 2^24 like a float count; the numpy restatement of
the output order (a stable 3-way partition filtered by the labels a select names) is the oracle's."""
import os
import time

import numpy as np
import pytest

import cloud_orders as co
import large_clouds as lc
from groundgrid_b200 import capi
from oracle import Oracle


def host_available():
    return os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")


def need_host(nbytes, what):
    have = host_available()
    if have < nbytes:
        pytest.skip(f"{what} needs {nbytes / 2**30:.1f} GiB of host memory, {have / 2**30:.1f} GiB available "
                    f"({(nbytes - have) / 2**30:.1f} GiB short)")


def prior_oracle(n_points):
    o = Oracle(*lc.BOUNDARY_GEOMETRY)
    o.init_map(0.0, 0.0, 0.0)
    o.filter_cloud(*lc.prior_scan(), 0.0)
    return o


def block_counts(classes, n_points):
    """Per 1024-point block of the output scan, the points of each output class (kept, ignored, outlier)."""
    nblk = -(-n_points // lc.OUT_TILE)
    blk = np.arange(n_points) // lc.OUT_TILE
    return np.stack([np.bincount(blk[classes == c], minlength=nblk) for c in (1, 3, 5)])


@pytest.mark.parametrize("n_points", lc.BOUNDARY_SIZES)
def test_boundary_clouds(n_points):
    pts, org = lc.boundary_cloud(n_points)
    assert len(pts) == n_points
    assert lc.out_scan_tiles(n_points) == {lc.TILE_EDGE: 1, lc.TILE_EDGE + 1: 2, 2 * lc.TILE_EDGE: 2}.get(n_points, 3)
    o = prior_oracle(n_points)
    labels, index, _, classes = o.filter_cloud(pts, org, 0.0, want_classes=True)
    n = o.n
    # the classes the oracle found are the ones the generator aims at: ignored by ring, outliers among the pushed points
    assert np.array_equal(classes == 0, co.cell_index(pts, n, 0.33, (0.0, 0.0)) == n * n)
    assert np.array_equal(np.isin(classes, (3, 4)), (classes > 0) & ~co.kept_mask(pts, org, n, 0.33, (0.0, 0.0)))
    counts = block_counts(classes, n_points)
    assert ((counts > 0).mean(axis=1) > 0.5).all(), "each class in most blocks of the output scan"
    flat = counts.ravel()                        # the order in which k_out_scan scans them
    for edge in range(lc.SCAN_TILE, len(flat), lc.SCAN_TILE):
        # (past the last edge of 2 * TILE_EDGE + 1 points there is only the outliers' count of the one-point last block)
        assert flat[edge - 8:edge].any() and (flat[edge:edge + 8].any() or len(flat) == edge + 1), f"counts around the tile edge at {edge}"
    kept = np.isin(classes, (1, 2))
    most, runs = lc.kept_cell_bounds(pts, org, n, 0.33, kept=kept)
    assert most <= co.MAX_POINTS_PER_CELL and runs <= co.MAX_RUNS_PER_CELL, (most, runs)
    assert np.array_equal(lc.output_order(classes, labels), index)
    for name, sel in lc.SELECTS.items():
        want = index[np.isin(labels[index], {"all": (49, 99), "ground": (49,), "nonground": (99,)}[name])]
        assert np.array_equal(lc.output_order(classes, labels, sel), want), name


@pytest.mark.parametrize("how,count", [("ring", c) for c in lc.PILE_SIZES] + [("near", lc.FLOAT_STOP + 2), ("near", 1 << 25)])
def test_piles(how, count):
    """pointsRaw = min(inside points, 2^24) and points = min(non-ground points, 2^24) on the piled cell, as the reference's
    float counts give them."""
    need_host(3 * count * 32, f"a pile of {count} points")
    pts, org, cell, nonground = lc.pile(count, how)
    n = 100
    cells = co.cell_index(pts, n, 0.33, (0.0, 0.0))
    mine = cells == cell
    assert mine.sum() >= count
    kept = co.kept_mask(pts, org, n, 0.33, (0.0, 0.0))
    assert not kept[mine].any(), "the piled points are ignored"
    assert 200 <= kept.sum() <= 1000, "a few hundred kept points of an ordinary scan"
    most, runs = lc.kept_cell_bounds(pts, org, n, 0.33)
    assert most <= co.MAX_POINTS_PER_CELL and runs <= co.MAX_RUNS_PER_CELL
    o = Oracle(*lc.PILE_GEOMETRY)
    o.init_map(0.0, 0.0, 0.0)
    labels, index, _, classes = o.filter_cloud(pts, org, 0.0, want_classes=True)
    raw, points = o.layer("pointsRaw").ravel(order="F"), o.layer("points").ravel(order="F")
    assert raw[cell] == min(int(mine.sum()), lc.FLOAT_STOP)
    assert points[cell] == min(int((labels[mine] == 99).sum()), lc.FLOAT_STOP)
    assert (labels[mine] == 99).sum() >= nonground
    if count > lc.FLOAT_STOP + 1:
        assert raw[cell] < mine.sum(), "the pile is past where a float count stops"
    assert np.array_equal(lc.output_order(classes, labels), index)


def test_capacity_cloud():
    """The largest cloud a handle takes, on both maps the GPU tests run it on; the oracle's time for it is printed."""
    need_host(12 << 30, "the capacity cloud")
    pts, org = lc.capacity_cloud(300)
    assert len(pts) == lc.CAPACITY
    for n, (dim, res) in lc.CAPACITY_GEOMETRIES.items():
        if n != 300:
            pts, org = lc.capacity_cloud(n)
        assert capi.host_cells_per_side(dim, res) == n
        o = Oracle(dim, res)
        o.init_map(0.0, 0.0, 0.0)
        t = time.perf_counter()
        labels, index, _, classes = o.filter_cloud(pts, org, 0.0, want_classes=True)
        print(f"oracle on {len(pts)} points, N = {n}: {time.perf_counter() - t:.1f} s")
        assert (classes == 0).sum() == 0, "every point inside the map"
        kept = np.isin(classes, (1, 2))
        most, runs = lc.kept_cell_bounds(pts, org, n, res, kept=kept)
        assert most <= co.MAX_POINTS_PER_CELL and runs <= co.MAX_RUNS_PER_CELL, (most, runs)
        assert (labels == 99).sum() > 0.1 * len(pts) and (labels == 49).sum() > 0.1 * len(pts)
        assert np.array_equal(lc.output_order(classes, labels), index)
        del labels, index, classes, o


@pytest.mark.parametrize("n", list(lc.WIDE_GEOMETRIES))
def test_sprinkles(n):
    dim, res = lc.WIDE_GEOMETRIES[n]
    assert capi.host_cells_per_side(dim, res) == n
    pts, org, cells = lc.sprinkle(n)
    flat = co.cell_index(pts, n, res, (0.0, 0.0))
    assert np.array_equal(np.unique(flat), np.unique(cells[:, 0] + cells[:, 1] * n)), "every point in the cell it aims at"
    i, j = flat % n, flat // n
    for edge in (i == 0, i == n - 1, j == 0, j == n - 1):
        assert len(np.unique(flat[edge])) == n, "every cell of every border row and column"
    for ci, cj in ((n - 4, n - 4), (n - 1, n - 1), (0, n - 1), (n - 1, 0)):
        assert (flat == ci + cj * n).any()
    if n > 2896:
        assert ((flat >> 23) & 1).sum() > 1000 and (flat == 1 << 23).any()
    most, runs = lc.kept_cell_bounds(pts, org, n, res)
    assert most <= co.MAX_POINTS_PER_CELL and runs <= co.MAX_RUNS_PER_CELL

"""tests/cloud_orders.py without a GPU: every generator reaches the regime it is named for (so the GPU comparisons of
tests/test_gpu_input_orders.py keep feeding the paths they are meant for when synth.py or the kernels' constants change),
the oracle behaves under re-ordering as the algorithm says it must, and its per-cell statistics on the constructed
clouds equal a float32 Welford recurrence written out here."""
import numpy as np
import pytest

import cloud_orders as co
from groundgrid_b200 import synth
from oracle import Oracle

DIM, RES, N = 99.0, 0.33, 300
GEOMETRIES = [(33.0, 0.33, 100), (33.33, 0.33, 101), (99.0, 0.33, 300)]
FAR = (1.2e5 + 0.37, -3.4e5 - 0.11)


@pytest.fixture(scope="module")
def scan64():
    return synth.scan_64(synth.make_scene(seed=1234), seed=1234)


def flat(layer):
    return layer.ravel(order="F")      # cell = i + j * n


def run_oracle(pts, org, dim=DIM, res=RES, position=(0.0, 0.0), stop_after=0):
    o = Oracle(dim, res)
    o.init_map(position[0], position[1], 0.0)
    labels, index, _ = o.filter_cloud(pts, org, 0.0, threads=1, stop_after=stop_after)
    return o, labels, index


@pytest.fixture(scope="module")
def ring_major(scan64):
    pts, org = scan64
    o, labels, index = run_oracle(pts, org)
    return {n: o.layer(n) for n in ("points", "variance", "minGroundHeight", "ground", "groundpatch")}, labels, index


def test_profile_counts_what_the_oracle_counts(scan64):
    pts, org = scan64
    for cloud in (pts, co.shuffled(pts, 3)[0]):
        o, _, _ = run_oracle(cloud, org, stop_after=1)
        prof = co.run_profile(cloud, org, N, RES, (0.0, 0.0))
        assert np.array_equal(prof.count, flat(o.layer("points")).astype(np.int64))
        assert prof.run_len.sum() == prof.count.sum() and (prof.runs <= prof.count).all()
    ring = co.run_profile(pts, org, N, RES, (0.0, 0.0))
    assert ring.runs.max() <= 57, "the ring-major cloud every other test feeds now reaches the first Shell gap too"


@pytest.mark.parametrize("name", co.REORDERINGS)
def test_reordering_reaches_its_regime(scan64, name):
    pts, org = scan64
    cloud, perm = co.reorder(name, pts, org, N, RES)
    assert np.array_equal(np.sort(perm), np.arange(len(pts))) and cloud.tobytes() == co.take(pts, perm).tobytes()
    base = co.run_profile(pts, org, N, RES, (0.0, 0.0))
    prof = co.run_profile(cloud, org, N, RES, (0.0, 0.0))
    print(f"{name}: {prof}")
    assert np.array_equal(prof.count, base.count)
    if name == "firing":
        assert prof.run_split.sum() > 10000 and prof.bands()["runs"]["24-57"] > 300
    elif name == "shuffled":
        assert (prof.runs > 57).sum() > 100
    elif name == "reversed":
        assert abs(int(prof.runs.sum()) - int(base.runs.sum())) < 100      # the same warps but for the shifted boundary
    elif name == "cell_sorted":
        assert (prof.runs <= (prof.count + 31) // 32 + 1).all() and (prof.run_len == 32).sum() > 500
    elif name == "cell_round_robin":
        assert (prof.run_len == 1).all() and np.array_equal(prof.runs, prof.count) and prof.runs.max() > 600
    elif name == "two_cell_alternation":
        assert prof.run_split.sum() > 0.8 * len(prof.run_len)


@pytest.mark.parametrize("dim,res,n", GEOMETRIES)
@pytest.mark.parametrize("position", [(0.0, 0.0), FAR])
def test_runs_ladder_has_every_run_count(dim, res, n, position):
    pts, org, targets = co.runs_ladder(n, res, position, seed=n)
    prof = co.run_profile(pts, org, n, res, position)
    print(f"runs_ladder N={n}: {prof}")
    assert set(co.RUNS_LADDER) <= set(targets)
    for k, cells in targets.items():
        assert all(prof.runs[c] == k for c in cells), (k, [int(prof.runs[c]) for c in cells])
    assert (prof.count > 0).sum() == sum(len(c) for c in targets.values())
    assert {1, 2, 3, 31, 32} <= set(prof.run_len.tolist())
    single = prof.run_len == 1
    assert (prof.run_first_lane[single] == 0).any() and (prof.run_first_lane[single] == 31).any()
    assert prof.run_split.sum() > 100
    assert prof.count.max() <= co.MAX_POINTS_PER_CELL and prof.runs.max() <= co.MAX_RUNS_PER_CELL
    assert (pts["z"] == org[2]).sum() > 50          # the mean == 0 restart


@pytest.mark.parametrize("dim,res,n", GEOMETRIES)
@pytest.mark.parametrize("scattered", [False, True])
def test_count_ladder_has_every_count(dim, res, n, scattered):
    pts, org, targets = co.count_ladder(n, res, seed=n, scattered=scattered)
    prof = co.run_profile(pts, org, n, res, (0.0, 0.0))
    print(f"count_ladder N={n} scattered={scattered}: {prof}")
    assert tuple(targets) == co.COUNT_LADDER
    assert all(prof.count[cell] == c for c, cell in targets.items())
    assert prof.count.max() == 8192 <= co.MAX_POINTS_PER_CELL and prof.runs.max() <= co.MAX_RUNS_PER_CELL
    big = targets[8192]
    assert prof.runs[big] > 1000 if scattered else prof.runs[big] == 257
    assert prof.bands()["points"]["6144+"] == 1


def test_nonfinite_and_far_clouds(scan64):
    pts, org = scan64
    bad = co.nonfinite_heights(pts, seed=1)
    z = bad["z"]
    assert np.isnan(z).sum() > 100 and (z == np.inf).sum() > 100 and (z == -np.inf).sum() > 100
    assert np.isfinite(bad["x"]).all() and np.isfinite(bad["y"]).all()
    assert ((bad["ring"] > 1024) & ~np.isfinite(z)).sum() > 10
    for where, most in (((1.2e5, -3.4e5), 120000), ((4.1e5, 5.6e6), 60000)):
        far, forg = co.coarse_far_cloud(where)
        pairs = len(np.unique(np.stack([far["x"], far["y"]], 1), axis=0))
        assert pairs < min(most, len(far)), pairs
        assert (co.cell_index(far, N, RES, where) < N * N).sum() > 100000


@pytest.mark.parametrize("name", co.REORDERINGS)
def test_oracle_under_reordering(scan64, ring_major, name):
    """The obstacle count, the kept count and the minimum height of a cell do not depend on the point order; the variance
    does (fp32 Welford), which is what makes the bit-exact GPU comparison on these clouds say something.  A label may
    only change in a cell whose terrain changed with it."""
    pts, org = scan64
    L0, lab0, idx0 = ring_major
    cloud, perm = co.reorder(name, pts, org, N, RES, seed=5)
    o, lab1, idx1 = run_oracle(cloud, org)
    for layer in ("points", "minGroundHeight"):
        assert np.array_equal(o.layer(layer), L0[layer]), layer
    o1, _, _ = run_oracle(cloud, org, stop_after=1)
    o0, _, _ = run_oracle(pts, org, stop_after=1)
    assert np.array_equal(o1.layer("points"), o0.layer("points")) and np.array_equal(o1.layer("pointsRaw"), o0.layer("pointsRaw"))
    assert (lab1 != 0).sum() == (lab0 != 0).sum() and len(idx1) == len(idx0)
    assert np.array_equal(np.sort(perm[idx1]), np.sort(idx0))
    var_changed = flat(o.layer("variance")) != flat(L0["variance"])
    if name in ("shuffled", "firing", "reversed"):     # the others keep the order inside (nearly) every cell
        assert var_changed.sum() > 100, "the cloud's variance does not depend on the order: the comparison proves nothing"
    differ = np.nonzero(lab1 != lab0[perm])[0]
    if len(differ):
        cells = co.cell_index(cloud, N, RES, (0.0, 0.0))[differ]
        terrain = (flat(o.layer("ground")) != flat(L0["ground"])) | (flat(o.layer("groundpatch")) != flat(L0["groundpatch"]))
        unexplained = [int(c) for c in cells if not terrain[c]]
        assert not unexplained and var_changed.any(), f"{name}: labels changed in cells {unexplained[:5]} whose terrain did not"


def welford(z, oz):
    """The accumulate step of insert_cloud in float32, in input order: (points, mean, m2, variance, minimum)."""
    f = np.float32
    n, mean, m2, mn = f(0), f(0), f(0), np.finfo(f).max
    for v in z.astype(f):
        pd = v - oz
        if mean == 0:
            mean = pd
        if not np.isnan(pd):
            delta = pd - mean
            mean = mean + delta / (n + f(1))
            m2 = m2 + delta * (pd - mean)
        mn = min(mn, v - f(0.0001))
        n = n + f(1)
    return n, mean, m2, m2 / (n + np.finfo(f).tiny), mn


@pytest.mark.parametrize("dim,res,n", GEOMETRIES[:2])
def test_oracle_statistics_equal_the_recurrence_in_input_order(dim, res, n):
    for pts, org, targets in (co.runs_ladder(n, res, seed=11), co.count_ladder(n, res, seed=12, scattered=True)):
        o, _, _ = run_oracle(pts, org, dim, res, stop_after=1)      # later phases reuse "points" for the obstacle count
        got = {name: flat(o.layer(name)) for name in ("points", "meanVariance", "m2")}
        got["variance"] = flat(run_oracle(pts, org, dim, res, stop_after=2)[0].layer("variance"))
        got["minGroundHeight"] = flat(o.layer("minGroundHeight"))
        cell = co.cell_index(pts, n, res, (0.0, 0.0))
        order_matters = 0
        for c in np.unique(cell[cell < n * n]):
            z = pts["z"][cell == c]
            want = welford(z, org[2])
            assert tuple(got[name][c] for name in got) == want, f"cell {c} with {len(z)} points"
            order_matters += len(z) > 2 and welford(z[::-1], org[2])[2] != want[2]
        assert order_matters >= 10

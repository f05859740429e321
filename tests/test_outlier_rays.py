"""The rays of tests/outlier_rays.py without a GPU: each case lands on the decision it is named for, the oracle and pyref
agree with the numpy march on it, and the exact walk k_rasterize finishes long rays with (gg_internal.h:outlier_walk,
exported as gg_host_outlier_walk) agrees with the step-by-step march on seeded rays of up to ~1e8 steps and on every
case."""
import ctypes as C

import numpy as np
import pytest

import outlier_rays as orr
import pyref
from groundgrid_b200 import capi
from oracle import Oracle

SIZES = [(100, (0.0, 0.0)), (101, (0.0, 0.0)), (100, orr.FAR)]


@pytest.fixture(scope="module", params=SIZES, ids=["n100", "n101", "n100-far"])
def case_set(request):
    n, pos = request.param
    return orr.cases(n, pos, heavy=n == 100 and pos == (0.0, 0.0))


def by_name(cs):
    return {c.name: c for c in cs}


def test_each_case_sits_on_its_decision(case_set):
    cs = by_name(case_set)
    hit = lambda name: cs[name].want[0]
    # both sides of every boundary
    assert hit("pretest/just below") and not hit("pretest/just above")
    assert [hit(f"pretest/G {t}") for t in ("nan", "+inf", "-inf", "-0", "denormal", "+max", "-max")] == [False, True, False, True, True, True, False]
    assert hit("direction/below") and not hit("direction/above")
    vz = lambda name: orr.ray(cs[name].origin, cs[name].point).vz
    assert vz("direction/below") < np.float32(-0.01) <= vz("direction/above")   # adjacent floats z, on either side
    assert not hit("cell/C=0.01f") and hit("cell/C above 0.01f")
    assert not hit("cell/sum 1.25 at") and hit("cell/sum 1.25 above") and not hit("cell/sum 1.25 below")
    assert hit("cell/sum 0.6 at") and not hit("cell/sum 0.6 below")          # 0.6f > 0.6 in double
    for tol in (0.1, 0.0, -0.3):
        assert hit(f"cell/G at bound tol {tol}") and not hit(f"cell/G below bound tol {tol}")
    assert [hit(f"cell/{t}") for t in ("G nan", "G +inf", "G -inf", "C nan", "C +inf", "C -inf", "block +inf", "block +inf -inf",
                                       "block nan", "block FLT_MAX overflow")] == [False, True, False, False, True, False, True, False, False, True]
    assert hit("config/threshold 0") and hit("config/threshold -1") and not hit("config/threshold 1e+09")
    assert hit("config/tolerance -0.5") and not hit("config/tolerance 0.5")
    # the tree sum and the sequential sum of the planted block sit on opposite sides of the threshold
    for thr in (1.25, 0.6):
        c = cs[f"cell/tree vs sequential {thr}"]
        i, j = [(a, b) for a, b in zip(*np.nonzero(c.G == np.float32(1e6)))][0]
        e = [c.C[a, b] for a, b in orr.block_cells(i, j)]
        s = np.float32(0.0)
        for v in e:
            s = np.float32(s + v)
        assert (np.float64(pyref.tree_sum(e)) > thr) != (np.float64(s) > thr) and c.C[i, j] > np.float32(0.01)
    # edge rows: 0 and N-1 are never tested, 1 .. 3 and N-2 are (1 .. 3 with the block clamped to row 2)
    n = case_set[0].n
    for axis in "xy":
        assert not hit(f"geometry/{axis} row 0") and not hit(f"geometry/{axis} row {n - 1}")
        assert all(hit(f"geometry/{axis} row {k}") for k in (1, 2, 3, n - 2))
    # the loop end: an occluder at the cell of the loop's last step is found, one met only at the first step it does not
    # run is not
    for name, c in cs.items():
        if c.regime == "loop_end":
            steps, ix, iy, _ = orr.trace(c)
            k = int(np.nonzero(steps == c.want[1])[0][0]) if c.want[0] else -2
            assert (ix[k], iy[k]) == (ix[-1], iy[-1]), name   # found in the cell of the loop's last step
        if c.regime == "loop_end beyond" and not c.want[0]:
            assert orr.march(c)[2] == int(orr.trace(c)[0][-1]) + 1, name
    # long rays: the hit lands on the named step
    for tag, step in (("2^20-1", orr.OLD_CAP - 1), ("2^20", orr.OLD_CAP), ("2^20+1", orr.OLD_CAP + 1), ("walk-1", orr.WALK_FROM - 1),
                      ("walk", orr.WALK_FROM), ("walk+1", orr.WALK_FROM + 1)):
        assert cs[f"long/hit at {tag}"].want == (True, step)
    assert cs["long/cap probe z -3e+06"].want[1] > orr.OLD_CAP and cs["long/origin 2e6 m outside"].want[1] > orr.OLD_CAP


def oracle_outlier(c):
    o = Oracle(c.dim, c.res)
    if c.cfg:
        o.set_config(**c.cfg)
    o.init_map(float(c.position[0]), float(c.position[1]), 0.0)
    o.set_layer("ground", c.G)
    o.set_layer("groundpatch", c.C)
    o.filter_cloud(c.cloud(), c.origin, 0.0, threads=1, stop_after=1)
    kept = o.layer("points").sum() + o.layer("pointsRaw").sum() * 0
    o.close()
    return kept == 0


def test_oracle_and_pyref_agree_with_the_march(case_set):
    for c in case_set:
        assert oracle_outlier(c) == c.want[0], c.name
        if c.regime.startswith("long"):
            continue
        G, Cf = c.G.copy(), c.C.copy()
        out = pyref.filter_cloud(c.cloud(), c.origin, 0.0, G, Cf, None, c.geo(), c.cfg, stop_after=1)
        assert (out["outliers"] == [0]) == c.want[0], c.name


def walk(c, start):
    L = capi.load()
    f = L.gg_host_outlier_walk
    f.restype = C.c_int
    f.argtypes = [C.c_double, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_longlong]
    G, Cf = np.asfortranarray(c.G, np.float32), np.asfortranarray(c.C, np.float32)
    pos = np.array(c.position, np.float64)
    o, p = np.ascontiguousarray(c.origin, np.float32), np.ascontiguousarray(c.point, np.float32)
    r = f(c.dim, np.float32(c.res), pos.ctypes.data, G.ctypes.data, Cf.ctypes.data, float(c.thr()), float(c.tol()), o.ctypes.data,
          p.ctypes.data, int(start))
    return None if r < 0 else bool(r)


def test_walk_against_the_march_on_every_case(case_set):
    for c in case_set:
        want = orr.march(c)[0] if orr.ray(c.origin, c.point).vz < np.float32(-0.01) else None
        for start in (3, orr.WALK_FROM):
            w = orr.march(c, start=start)[0] if start != 3 and want is not None else want
            assert walk(c, start) == w, f"{c.name} from {start}"


def random_ray(rng, n, position, length):
    """A ray of about `length` steps over a random prior, hitting the map at a random angle; the occluders are sparse so
    that many rays run to their end."""
    G, Cf = orr.blank(n)
    m = rng.uniform(size=(n, n)) < 0.02
    Cf[m] = rng.choice(np.array([0.005, 0.3, 1.0, np.inf, np.nan], np.float32), m.sum())
    G[m] = rng.uniform(-length, 5.0, m.sum()).astype(np.float32)
    half = 0.5 * orr.GEOMETRY[n][0]
    p = np.array([position[0] + rng.uniform(-half, half), position[1] + rng.uniform(-half, half), 0.0], np.float32)
    ang = rng.uniform(0, 2 * np.pi)
    dist = rng.choice([rng.uniform(4, 30), rng.uniform(1e3, 3e6)])
    steep = rng.uniform(0.02, 1.0)
    o = np.array([p[0] - dist * np.cos(ang), p[1] - dist * np.sin(ang), 0.0], np.float32)
    o[0] = o[0] if rng.uniform() < 0.8 else np.float32(position[0] + rng.integers(-50, 50) * np.float32(0.33))   # on an edge
    o[2] = np.float32(length * steep)
    p[2] = np.float32(-length * (1 - steep) - 1.0)
    cfg = dict(min_outlier_detection_ground_confidence=float(rng.choice([-1.0, 0.0, 0.6, 1.25])), outlier_tolerance=float(rng.choice([-0.3, 0.0, 0.1])))
    return orr.Case("random", n, position, G, Cf, o, p, cfg)


@pytest.mark.parametrize("seed", range(6))
def test_walk_against_the_march_on_seeded_rays(seed):
    """Lengths from a few steps to ~1e8; vx = +-0 rays, rays whose positions leave int32 cell indices, (float) step above
    2^24."""
    rng = np.random.default_rng(seed)
    n, pos = [(100, (0.0, 0.0)), (101, orr.FAR)][seed % 2]
    lengths = [10.0, 60.0, 3e3, 5e3, 2e4] + ([1e8] if seed == 0 else [3e7] if seed == 1 else [])
    for k, length in enumerate(lengths * 3):
        c = random_ray(rng, n, pos, length)
        if k % 5 == 1:   # vx = +-0: straight along y
            c.point[0] = c.origin[0]
        if k % 5 == 2:   # an origin whose ray starts ~3e9 cells from the map
            c.origin[0] = np.float32(pos[0] + 1e9)
        want = orr.march(c)[0] if orr.ray(c.origin, c.point).vz < np.float32(-0.01) else None
        assert walk(c, 3) == want, f"seed {seed} ray {k} length {length:g}"

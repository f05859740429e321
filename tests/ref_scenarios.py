"""Scenarios that pin an implementation to the reference itself, replayed from stored digests.

Every scenario drives one implementation (the reference, the oracle port or the CUDA path, behind the small adapters
below) through the same seeded sequence of map creation, pose updates and scans, and hands every value the
reference answers with (labels, output order and cloud, every layer, map position, moved flags, grid arithmetic) to
a Recorder.  tests/golden/make_ref_digests.py runs the scenarios on the reference itself (oracle/_ref: its unmodified
sources on CPU stand-ins, oracle/build_ref.py) and stores one SHA-256 per value in tests/golden/ref_digests.json; the
tests replay them on the oracle port and on the CUDA path and require every digest to match, i.e. bit-exact equality
with the reference (NaN payloads and the sign of zero are made canonical first, as np.array_equal(equal_nan=True)
compares them).
"""
import hashlib
import json
import os

import numpy as np

import cloud_orders as co
from groundgrid_b200 import synth
from groundgrid_b200.synth import base_from_map_qt, tf2_matrix

DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_digests.json")
LAYERS = ("points", "ground", "groundpatch", "minGroundHeight", "maxGroundHeight", "groundCandidates", "planeDist", "m2",
          "meanVariance", "pointsRaw", "variance")
CLOUD_FIELDS = ("x", "y", "z", "intensity", "ring")   # padding bytes of the records are not part of the value
# the reference's labels at thread_count = 1 for sequential_scan() (the racy shipped threading is compared with them)
SEQUENTIAL_LABELS = os.path.join(os.path.dirname(DIGESTS), "ref_labels_scan64_seed1234.npz")


def sequential_scan():
    """One 64-beam scan (seed 1234) on a fresh 300 x 300 @ 0.33 m map: (dimension, resolution, points, origin)."""
    pts, org = synth.scan_64(synth.make_scene(seed=1234), seed=1234)
    return 99.0, 0.33, pts, org


def digest(a):
    a = np.ascontiguousarray(a)
    if a.dtype.kind == "f":
        a = np.where(np.isnan(a), np.array(np.nan, a.dtype), a + a.dtype.type(0))   # one NaN, +0.0 for -0.0
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()[:32]


def summary(a):
    """What a failed comparison reports about the value an implementation produced."""
    a = np.asarray(a)
    if a.dtype.kind == "f":
        fin = a[np.isfinite(a)]
        return (f"{a.dtype}{a.shape}: {np.isnan(a).sum()} NaN, {a.size - fin.size} non-finite, "
                f"finite min {fin.min() if fin.size else None} max {fin.max() if fin.size else None} sum {float(fin.astype(np.float64).sum())!r}")
    if a.dtype.kind in "iub" and a.size and a.min() >= 0 and a.max() < 256:
        vals, counts = np.unique(a, return_counts=True)
        return f"{a.dtype}{a.shape}: counts {dict(zip(vals.tolist()[:8], counts.tolist()[:8]))}"
    return f"{a.dtype}{a.shape}: {a.ravel()[:6].tolist()}"


class Recorder:
    """record=True collects the digests of one scenario; otherwise each value is checked against the stored one."""

    def __init__(self, scenario, record=False):
        self.scenario = scenario
        self.record = record
        self.got = {}
        if not record:
            with open(DIGESTS) as f:
                self.want = json.load(f)[scenario]

    def __call__(self, key, value):
        d = digest(np.asarray(value))
        assert key not in self.got, f"{self.scenario}: {key} recorded twice"
        self.got[key] = d
        if not self.record:
            assert key in self.want, f"{self.scenario}: {key} was not produced by the reference's run"
            assert d == self.want[key], f"{self.scenario}: {key} differs from the reference; got {summary(value)}"

    def stored(self, key):
        """An integer the reference's run stored (e.g. how many random draws it rejected)."""
        self.got["#" + key] = self.want["#" + key]
        return int(self.want["#" + key])

    def store(self, key, value):
        self.got["#" + key] = int(value)

    def done(self):
        if not self.record:
            missing = sorted(set(self.want) - set(self.got))
            assert not missing, f"{self.scenario}: the reference's run also produced {missing[:5]}"
        return self.got


class Folded:
    """Takes the values of one case in place of a Recorder and hands the Recorder ONE digest of them (of their keys and
    digests, in order) under `key`: for scenarios of many cases, where a digest per value would make the stored file
    large.  A mismatch names the case; the tests that compare the CUDA path with the oracle value by value name the
    value."""

    def __init__(self, rec, key):
        self.rec, self.key, self.parts = rec, key, []

    def __call__(self, key, value):
        self.parts.append(f"{key}:{digest(np.asarray(value))}")

    def done(self):
        self.rec(self.key, np.frombuffer("\n".join(self.parts).encode(), np.uint8))


# ---- implementations ------------------------------------------------------------------------------------------------
class Reference:
    """oracle/_ref: the reference's own sources."""

    def __init__(self, dim, res):
        from oracle import ref as refmod

        self.m = refmod.Reference(dim, res)   # ValueError for geometries GroundSegmentation::init rejects
        self.n = self.m.n

    def update(self, x, y, q, t):
        return int(self.m.update(x, y, q, t))

    def filter_cloud(self, pts, org, base_z, cloud=True):
        return self.m.filter_cloud(pts, org, base_z, want_cloud=cloud)

    def __getattr__(self, name):
        return getattr(self.m, name)


class Oracle:
    """The oracle port (oracle/gg_oracle.cpp) at thread_count = 1."""

    def __init__(self, dim, res):
        from oracle import Oracle as O

        self.m = O(dim, res)
        self.n = self.m.n

    def update(self, x, y, q, t):
        return int(self.m.update(x, y, tf2_matrix(q, t)))

    def filter_cloud(self, pts, org, base_z, cloud=True):
        return self.m.filter_cloud(pts, org, base_z, threads=1, want_cloud=cloud)

    def __getattr__(self, name):
        return getattr(self.m, name)


class Cuda:
    """The CUDA path through the C-ABI (one slot, every layer kept)."""

    def __init__(self, dim, res, max_points):
        from groundgrid_b200 import capi

        self.m = capi.GroundGridB200(dim, res, n_slots=1, max_points=max_points, full_layers=True)
        self.n = self.m.n

    def expected_points(self):
        return self.m.layer("expectedPoints")

    def update(self, x, y, q, t):
        return int(self.m.update_pose(x, y, tf2_matrix(q, t)))

    def filter_cloud(self, pts, org, base_z, cloud=True):
        return self.m.filter_cloud(pts, org, base_z, want_index=True, want_cloud=cloud)

    def spiral(self, base_z):
        self.m.spiral_ground_interpolation(base_z)

    def add_layer(self, name, value=0.0):
        """Every layer exists on the device: grid_map's add(name, value) only sets it."""
        self.m.set_layer(name, np.full((self.n, self.n), value, np.float32))

    def detect_ground_patches(self):
        self.m.detect_ground_patches()

    def detect_ground_patch(self, size, i, j):
        self.m.detect_ground_patch(size, i, j)

    def __getattr__(self, name):
        return getattr(self.m, name)


# ---- helpers --------------------------------------------------------------------------------------------------------
def push_below_ground(pts, count, seed):
    rng = np.random.default_rng(seed)
    idx = rng.choice(len(pts), count, replace=False)
    pts["z"][idx] -= rng.uniform(0.25, 2.0, count).astype(np.float32)


def created(make, rec, dim, res, position=(0.0, 0.0), **cfg):
    m = make(dim, res)
    rec("cells", m.n)
    if cfg:
        m.set_config(**cfg)
    m.init_map(float(position[0]), float(position[1]), 0.0)
    for name in ("points", "ground", "groundpatch", "minGroundHeight", "maxGroundHeight"):
        rec(f"creation/{name}", m.layer(name))
    return m


def scan(m, rec, pts, org, base_z, ctx, layers=LAYERS, cloud=True):
    labels, order, out = m.filter_cloud(pts, org, base_z, cloud=cloud)
    rec(f"{ctx}/labels", labels)
    rec(f"{ctx}/order", order)
    if cloud:
        for f in CLOUD_FIELDS:
            rec(f"{ctx}/cloud.{f}", out[f])
    for name in layers:
        rec(f"{ctx}/{name}", m.layer(name))
    return labels


def update(m, rec, x, y, q, t, ctx, layers=("ground", "groundpatch")):
    moved = m.update(x, y, q, t)
    rec(f"{ctx}/moved", moved)
    rec(f"{ctx}/position", m.position())
    for name in layers:
        rec(f"{ctx}/{name}", m.layer(name))
    return moved


# ---- scenarios (former side-by-side comparisons with the reference) -----------------------------------------------
def expected_points_table(make, rec):
    for dim, res in ((99.0, 0.33), (120.0, 0.33), (120.0, 0.2), (33.0, 0.6)):
        m = make(dim, res)
        rec(f"{dim}/{res}/cells", m.n)
        rec(f"{dim}/{res}/expected", m.expected_points())


def cfg1_cfg2_64_beam_300(make, rec):
    """configs[0]/[1]: ~120 k points, 300 x 300 @ 0.33 m; three scans so that the prior is non-trivial."""
    m = created(make, rec, 99.0, 0.33)
    scene = synth.make_scene(seed=1234)
    for k in range(3):
        pts, org = synth.scan_64(scene, seed=1234 + k)
        if k == 2:
            push_below_ground(pts, 3000, 5)
        lab = scan(m, rec, pts, org, 0.0, f"scan {k}")
    assert (lab == 99).sum() > 10000 and (lab == 49).sum() > 50000


def cfg3_128_beam_600(make, rec):
    """configs[2]: ~240 k points, 600 x 600 @ 0.2 m."""
    m = created(make, rec, 120.0, 0.2)
    assert m.n == 600
    scene = synth.make_scene(seed=77)
    for k in range(2):
        pts, org = synth.scan_128(scene, seed=300 + k)
        scan(m, rec, pts, org, 0.0, f"scan {k}")


def cfg4_four_lidar_364(make, rec):
    """configs[3]: four 64-beam sensors, ~480 k points, the reference's own 364 x 364 map."""
    m = created(make, rec, 120.0, 0.33)
    assert m.n == 364
    scene = synth.make_scene(seed=99)
    for k in range(2):
        pts, org = synth.scan_4lidar(scene, seed=400 + k)
        assert len(pts) > 450000
        scan(m, rec, pts, org, 0.0, f"scan {k}")


def rolling_stream_with_outliers(make, rec):
    """12 scans: ego moves, yaws, the base frame is pitched (position-dependent seeding of exposed cells), points pushed
    below the ground (outlier ray-march against the rolled prior)."""
    m = created(make, rec, 99.0, 0.33)
    scene = synth.make_scene(seed=1234, stream_len=30.0, undulation=0.3)
    moved_any = 0
    for k in range(12):
        (ex, ey), yaw = synth.stream_pose(k, step=0.9)
        ey = -0.37 * k
        pts, org = synth.scan_64(scene, (ex, ey), yaw, seed=500 + k, az_steps=1024)
        if k:
            q, t = base_from_map_qt(ex, ey, yaw, 0.01 * k, pitch=0.02)
            moved_any += update(m, rec, ex, ey, q, t, f"roll {k}")
            push_below_ground(pts, 1500, 600 + k)
        scan(m, rec, pts, org, 0.01 * k, f"scan {k}")
    assert moved_any >= 8


def large_jump_clears_the_map(make, rec):
    """A pose jump of more than the map length drops the whole map (grid_map::move -> clearAll + one full region)."""
    m = created(make, rec, 33.0, 0.33)
    scene = synth.make_scene(seed=10, n_boxes=8, rmin=4.0, rmax=14.0)
    pts, org = synth.lidar_scan(scene, beams=24, az_steps=256, seed=1)
    scan(m, rec, pts, org, 0.0, "before jump")
    q, t = base_from_map_qt(100.0, -70.0, 0.3, 0.2, pitch=0.01)
    assert update(m, rec, 100.0, -70.0, q, t, "jump") == 1


def random_geometry_and_config(make, rec, seed):
    """Seeded random geometries (integer map lengths: GroundSegmentation::init takes the dimension as size_t) and
    configurations, three scans with a roll in between.  Geometries the reference rejects are drawn again; the replay
    skips as many draws as the reference's run rejected."""
    rng = np.random.default_rng(9000 + seed)
    rejected = 0
    while True:
        dim = float(rng.integers(24, 70))
        res = float(np.float32(rng.uniform(0.2, 0.6)))
        if rec.record:
            try:
                Reference(dim, res)
            except ValueError:
                rejected += 1
                continue
            rec.store("rejected", rejected)
        elif rejected < rec.stored("rejected"):
            rejected += 1
            continue
        break
    rec("geometry", np.array([dim, res]))
    cfg = dict(point_count_cell_variance_threshold=int(rng.integers(0, 30)), max_ring=int(rng.integers(10, 1024)),
               distance_factor=float(rng.uniform(0.0, 0.001)), minimum_distance_factor=float(rng.uniform(1e-4, 0.002)),
               miminum_point_height_threshold=float(rng.uniform(0.1, 0.6)),
               minimum_point_height_obstacle_threshold=float(rng.uniform(0.02, 0.2)),
               outlier_tolerance=float(rng.uniform(-0.2, 0.3)),
               ground_patch_detection_minimum_point_count_threshold=float(rng.uniform(0.05, 0.8)),
               patch_size_change_distance=float(rng.uniform(3.0, 30.0)),
               occupied_cells_decrease_factor=float(rng.uniform(1.5, 20.0)),
               occupied_cells_point_count_factor=float(rng.uniform(2.0, 40.0)),
               min_outlier_detection_ground_confidence=float(rng.uniform(0.2, 3.0)))
    m = created(make, rec, dim, res, **cfg)
    half = 0.5 * dim
    scene = synth.make_scene(seed=seed, n_boxes=10, rmin=3.0, rmax=0.8 * half)
    ex = ey = 0.0
    for k in range(3):
        ex += float(rng.uniform(-1.5, 1.5)) * (k > 0)
        ey += float(rng.uniform(-1.5, 1.5)) * (k > 0)
        yaw = float(rng.uniform(-0.5, 0.5))
        pts, org = synth.lidar_scan(scene, (ex, ey), yaw, beams=32, az_steps=512, seed=seed * 10 + k)
        if k:
            q, t = base_from_map_qt(ex, ey, yaw, 0.05 * k, pitch=float(rng.uniform(-0.03, 0.03)))
            update(m, rec, ex, ey, q, t, f"roll {k}", layers=())
            push_below_ground(pts, 400, seed + k)
        scan(m, rec, pts, org, 0.05 * k, f"scan {k}")


def geometry_primitives_agree(make, rec):
    """grid_map index <-> position arithmetic on random and on edge positions, before and after a move."""
    m = created(make, rec, 33.0, 0.33)
    rng = np.random.default_rng(4)

    def check(ctx):
        c = m.position()
        xs = np.concatenate([rng.uniform(-20, 20, 400) + c[0], c[0] + 0.5 * 33.0 + np.array([-1e-9, 0.0, 1e-9]),
                             c[0] - 0.5 * 33.0 + np.array([-1e-9, 0.0, 1e-9])])
        ys = np.concatenate([rng.uniform(-20, 20, 400) + c[1], c[1] + rng.uniform(-16, 16, 6)])
        idx = []
        for x, y in zip(xs, ys):
            for fx, fy in ((float(np.float32(x)), float(np.float32(y))), (float(x), float(y))):
                i, j, inside = m.grid_index(fx, fy)
                idx.append((int(inside), i if inside else 0, j if inside else 0))   # the index of an outside point is undefined
        rec(f"{ctx}/grid_index", np.array(idx, np.int64))
        rec(f"{ctx}/cell_position", np.array([m.cell_position(int(i), int(j)) for i, j in rng.integers(0, m.n, (50, 2))]))

    check("before move")
    q, t = base_from_map_qt(3.21, -1.77, 0.1, 0.0)
    assert update(m, rec, 3.21, -1.77, q, t, "move", layers=()) == 1
    check("after move")


def single_phase_calls_agree(make, rec):
    """interpolate_cell and the whole spiral called on their own (public methods, GroundSegmentation.h:56-62)."""
    m = created(make, rec, 33.0, 0.33)
    rng = np.random.default_rng(12)
    G = rng.normal(0.0, 0.5, (m.n, m.n)).astype(np.float32)
    Cf = rng.uniform(0.0, 1.0, (m.n, m.n)).astype(np.float32)
    Cf[rng.uniform(size=Cf.shape) < 0.5] = 0.0
    m.set_layer("ground", G)
    m.set_layer("groundpatch", Cf)
    for x, y in ((5, 7), (48, 49), (49, 49), (1, 1), (97, 97), (60, 12)):
        m.interpolate_cell(x, y)
    for name in ("ground", "groundpatch"):
        rec(f"interpolate_cell/{name}", m.layer(name))
    m.spiral(0.25)
    for name in ("ground", "groundpatch"):
        rec(f"spiral/{name}", m.layer(name))


# BASELINE.json's full sizes through the CUDA path: (dimension, resolution, sensor, max points)
FULL_SIZES = {"cfg2_300": (99.0, 0.33, "scan_64", 140000), "cfg3_600": (120.0, 0.2, "scan_128", 280000),
              "cfg4_364": (120.0, 0.33, "scan_4lidar", 520000)}


def full_size_stream(make, rec, cfg):
    """Three scans with a map roll and pushed-down points at one of BASELINE.json's full sizes: labels, output order,
    every layer after every scan."""
    dim, res, sensor, _ = FULL_SIZES[cfg]
    m = make(dim, res)
    rec("cells", m.n)
    rec("expected", m.expected_points())
    m.init_map(0.0, 0.0, 0.0)
    scene = synth.make_scene(seed=4321, stream_len=20.0, undulation=0.3)
    rng = np.random.default_rng(17)
    for k in range(3):
        ex, ey, yaw = 1.1 * k, -0.45 * k, 0.01 * k
        pts, org = getattr(synth, sensor)(scene, (ex, ey), yaw, seed=700 + k)
        if k:
            q, t = base_from_map_qt(ex, ey, yaw, 0.0, pitch=0.02)
            update(m, rec, ex, ey, q, t, f"roll {k}", layers=())
            idx = rng.choice(len(pts), 2000, replace=False)
            pts["z"][idx] -= rng.uniform(0.25, 2.0, 2000).astype(np.float32)
        scan(m, rec, pts, org, 0.0, f"scan {k}", cloud=False)


# ---- point orders, cell densities, non-finite heights, maps far from the origin (tests/cloud_orders.py) -----------------
def input_orders(make, rec):
    """Three scans on one 300 x 300 map, each in another point order (firing, shuffled, one point of a cell per warp), so
    the prior is non-trivial and the order changes from scan to scan; the third with points pushed below the ground."""
    m = created(make, rec, 99.0, 0.33)
    scene = synth.make_scene(seed=2024)
    for k, order in enumerate(("firing", "shuffled", "cell_round_robin")):
        pts, org = synth.scan_64(scene, seed=2100 + k)
        if k == 2:
            push_below_ground(pts, 3000, 7)
        pts, _ = co.reorder(order, pts, org, m.n, 0.33, seed=k)
        scan(m, rec, pts, org, 0.0, f"scan {k} {order}")


DENSE_GEOMETRY = {100: (33.0, 0.33), 101: (33.0, float(np.float32(33.0 / 101.0)))}


def dense_cells(make, rec, n):
    """Cells with a chosen number of runs (1 .. 120) and of points (1 .. 8 192) on an even and an odd map."""
    dim, res = DENSE_GEOMETRY[n]
    m = created(make, rec, dim, res)
    assert m.n == n
    for k, (pts, org, _) in enumerate((co.runs_ladder(n, res, seed=1), co.count_ladder(n, res, seed=2),
                                       co.count_ladder(n, res, seed=3, scattered=True), co.runs_ladder(n, res, seed=4))):
        scan(m, rec, pts, org, 0.0, f"scan {k}")


def nonfinite_heights(make, rec):
    """NaN, +inf and -inf heights at finite x, y: two scans (the second on the NaN-laden prior the first left), a roll,
    and a finite scan on what remains."""
    m = created(make, rec, 99.0, 0.33)
    scene = synth.make_scene(seed=606)
    for k in range(3):
        ex, ey = (0.0, 0.0) if k < 2 else (1.7, -0.8)
        pts, org = synth.scan_64(scene, (ex, ey), seed=610 + k)
        if k < 2:
            pts = co.nonfinite_heights(pts, seed=620 + k)
        else:
            q, t = base_from_map_qt(ex, ey, 0.0, 0.0, pitch=0.01)
            assert update(m, rec, ex, ey, q, t, "roll") == 1
        scan(m, rec, pts, org, 0.0, f"scan {k}")
        if k == 0:
            assert np.isnan(m.layer("ground")).sum() > 1000


FAR_POSITIONS = {"1.2e5": (1.2e5 + 0.37, -3.4e5 - 0.11), "5.6e6": (4.1e5 - 0.21, 5.6e6 + 0.43)}


def far_stream(where):
    """The poses and clouds of far_from_origin: (k, ex, ey, yaw, base_z, (q, t), points, origin) per scan; scan 4 follows
    a jump of more than the map's length."""
    px, py = FAR_POSITIONS[where]
    scene = co.far_scene((px, py), seed=31, undulation=0.2)
    for k in range(5):
        ex, ey, yaw = px + 0.9 * k, py - 0.7 * k, 0.02 * k
        if k == 4:
            ex, ey = px + 150.0, py - 120.0
            scene = co.far_scene((ex, ey), seed=32)
        pts, org = synth.scan_64(scene, (ex, ey), yaw, seed=3100 + k, az_steps=1024)
        if k:
            push_below_ground(pts, 800, 3200 + k)
        yield k, ex, ey, yaw, 0.01 * k, base_from_map_qt(ex, ey, yaw, 0.01 * k, pitch=0.02), pts, org


def far_from_origin(make, rec, where):
    """A map created 1e5 .. 6e6 m from the origin, where float32 coordinates are 0.008 .. 0.5 m apart: five scans rolling
    along a diagonal with yaw and a pitched base frame, the last after a jump that clears the map."""
    m = created(make, rec, 99.0, 0.33, position=FAR_POSITIONS[where])
    for k, ex, ey, yaw, base_z, (q, t), pts, org in far_stream(where):
        if k:
            assert update(m, rec, ex, ey, q, t, f"roll {k}") == 1
        lab = scan(m, rec, pts, org, base_z, f"scan {k}")
        assert (lab == 49).sum() > 20000 and (lab == 99).sum() > 2000


def far_geometry(make, rec, where):
    """grid_map's index and inside arithmetic at the cell edges of a far map and their float32 / float64 neighbours,
    before and after a move."""
    pos = FAR_POSITIONS[where]
    m = created(make, rec, 33.0, 0.33, position=pos)
    rng = np.random.default_rng(8)

    def check(ctx):
        c = m.position()
        edge = np.array([m.cell_position(int(i), int(i)) for i in range(m.n)]) + 0.5 * float(np.float32(0.33))
        idx = []
        for ex, ey in edge[rng.permutation(m.n)[:40]]:
            fx, fy = np.float32(ex), np.float32(ey)
            for x, y in ((ex, ey), (np.nextafter(ex, np.inf), ey), (np.nextafter(ex, -np.inf), np.nextafter(ey, -np.inf)),
                         (fx, fy), (np.nextafter(fx, np.float32(np.inf)), fy), (fx, np.nextafter(fy, np.float32(-np.inf))),
                         (np.nextafter(fx, np.float32(-np.inf)), np.nextafter(fy, np.float32(np.inf)))):
                i, j, inside = m.grid_index(float(x), float(y))
                idx.append((int(inside), i if inside else 0, j if inside else 0))
        rec(f"{ctx}/grid_index", np.array(idx, np.int64))
        rec(f"{ctx}/centre", c)

    check("created")
    q, t = base_from_map_qt(pos[0] + 3.21, pos[1] - 1.77, 0.1, 0.0)
    assert update(m, rec, pos[0] + 3.21, pos[1] - 1.77, q, t, "move", layers=()) == 1
    check("moved")


def nonfinite_confidence(make, rec):
    """Imported priors (set_layer, as a migrated slot brings them) with +-inf, NaN and other edge confidences
    (tests/spiral_priors.py) on far, near, ring-corner, centre and border cells: each non-finite value in its own map,
    the finite ones densely in one, for the default decrease factor and 1000; a scan and the per-phase spiral on each."""
    import spiral_priors as sp

    cases = sp.edge_cases(100, 0.33)
    pts, org = synth.lidar_scan(synth.make_scene(seed=5, n_boxes=6, rmin=1.0, rmax=13.0), beams=16, az_steps=256, seed=5)
    for factor in (5.0, 1000.0):
        for seed, (name, planted) in enumerate(cases.items()):
            G, C = sp.planted_prior(100, 0.33, planted, seed=seed)
            ctx = f"{factor:g}/{name}"
            for how in ("scan", "spiral"):
                m = make(33.0, 0.33)
                m.set_config(occupied_cells_decrease_factor=factor)
                m.init_map(0.0, 0.0, 0.0)
                m.set_layer("ground", G)
                m.set_layer("groundpatch", C)
                if how == "scan":
                    rec(f"{ctx}/scan/labels", m.filter_cloud(pts, org, 0.1, cloud=False)[0])
                else:
                    m.spiral(0.1)
                for layer in ("ground", "groundpatch"):
                    rec(f"{ctx}/{how}/{layer}", m.layer(layer))


# ---- patch detection on imported planes (tests/detect_planes.py) ----------------------------------------------------------
DETECT_SIZES = (12, 100, 101, 102, 300, 364)


def detection_map(make, c):
    """A fresh map of case c with its planes imported; the layers detection needs that a fresh map of the reference
    does not have yet ("groundCandidates", "m2", "variance", :61-75) are added first, as filter_cloud adds them."""
    m = make(c.dim, c.res)
    m.set_config(**c.config)
    m.init_map(0.0, 0.0, 0.0)
    for name in ("groundCandidates", "m2", "variance"):
        m.add_layer(name, 0.0)
    for name in c.planes:
        m.set_layer(name, c.planes[name])
    return m


def detection_scan(n, dim=None):
    """A small scan of an N x N map (of tests/detect_planes.geometry(n) unless the length is given): (points, origin)."""
    import detect_planes as dp

    dim = dp.geometry(n)[0] if dim is None else dim
    scene = synth.make_scene(seed=n, n_boxes=6, rmin=1.0, rmax=max(1.5, 0.4 * dim))
    return synth.lidar_scan(scene, beams=16, az_steps=256, seed=n)


def detect_planes(make, rec, n):
    """Every case of tests/detect_planes.py: detect_ground_patches over the four sections (with the variance recompute
    each starts with), then, on a fresh import, detect_ground_patch<S> at every planted cell and at the limits of the
    window; and detect_ground_patches right after a complete scan, on the layers filter_cloud left."""
    import detect_planes as dp

    for c in dp.cases(n):
        ctx = f"{c.kind}/{c.cfg_name}"
        m = detection_map(make, c)
        m.detect_ground_patches()
        for name in ("ground", "groundpatch", "variance"):
            rec(f"{ctx}/patches/{name}", m.layer(name))
        m = detection_map(make, c)
        for S, i, j in [(S, i, j) for i, j, S, _ in c.planted] + dp.window_limit_cells(n):
            m.detect_ground_patch(S, i, j)
        for name in ("ground", "groundpatch"):
            rec(f"{ctx}/patch/{name}", m.layer(name))
    dim, res = dp.geometry(n)
    m = make(dim, res)
    m.init_map(0.0, 0.0, 0.0)
    pts, org = detection_scan(n)
    rec("scan/labels", m.filter_cloud(pts, org, 0.0, cloud=False)[0])
    m.detect_ground_patches()
    for name in ("ground", "groundpatch", "variance"):
        rec(f"scan/patches/{name}", m.layer(name))


# ---- the outlier test on imported priors (tests/outlier_rays.py) ---------------------------------------------------------
OUTLIER_SIZES = ("100", "101", "far")


def outlier_priors(make, rec, which):
    """Every case of tests/outlier_rays.py (the rays on each decision of the outlier test, long rays past step 2^20, an
    origin 2e6 m outside the map): the prior imported with set_layer, then a one-point scan."""
    import outlier_rays as orr

    n, pos = {"100": (100, (0.0, 0.0)), "101": (101, (0.0, 0.0)), "far": (100, orr.FAR)}[which]
    for c in orr.cases(n, pos, heavy=False):
        m = make(c.dim, c.res)
        if c.cfg:
            m.set_config(**c.cfg)
        m.init_map(float(pos[0]), float(pos[1]), 0.0)
        m.set_layer("ground", c.G)
        m.set_layer("groundpatch", c.C)
        scan(m, rec, c.cloud(), c.origin, 0.0, c.name, layers=("points", "ground", "groundpatch", "minGroundHeight", "variance"))


# ---- cells past 2^24 points and scans across the tile edges of the output order (tests/large_clouds.py) ---------------
def crowded_cells(make, rec):
    """Piles of 2^24 + 2 and 2^24 + 3 ignored points in one cell (the reference's float counts of "pointsRaw" and "points"
    stop at 2^24), each on a fresh small map, and a scan of TILE_EDGE + 1 points after an ordinary one."""
    import large_clouds as lc

    for count, how in ((lc.FLOAT_STOP + 2, "ring"), (lc.FLOAT_STOP + 3, "near")):
        m = make(*lc.PILE_GEOMETRY)
        m.init_map(0.0, 0.0, 0.0)
        pts, org, _, _ = lc.pile(count, how)
        scan(m, rec, pts, org, 0.0, f"pile {count} {how}", cloud=False)
    m = make(*lc.BOUNDARY_GEOMETRY)
    m.init_map(0.0, 0.0, 0.0)
    scan(m, rec, *lc.prior_scan(), 0.0, "prior")
    scan(m, rec, *lc.boundary_cloud(lc.TILE_EDGE + 1), 0.0, f"{lc.TILE_EDGE + 1} points")


# ---- every configuration field at the ends of its range and beyond (tests/config_limits.py) -----------------------------
def near_returns(count, seed, radius=3.3):
    """`count` returns on the ground within `radius` m (< sqrt(12) m) of the sensor at the origin, on rings 0 .. 31: points
    filter_cloud ignores for the statistics and still labels."""
    rng = np.random.default_rng(seed)
    r = np.sqrt(rng.uniform(0.01, radius * radius, count))
    a = rng.uniform(-np.pi, np.pi, count)
    pts = np.zeros(count, synth.POINT_DTYPE)
    pts["x"], pts["y"] = (r * np.cos(a)).astype(np.float32), (r * np.sin(a)).astype(np.float32)
    pts["z"] = rng.uniform(-0.1, 0.6, count).astype(np.float32)
    pts["ring"] = rng.integers(0, 32, count)
    return pts


def config_limits_stream(n, scans=3):
    """The scans of config_limits on an N x N map: (ego x, y, yaw, base_z, points, origin) per scan; every scan after the
    first follows a roll with yaw and a pitched base frame and has points pushed below the ground."""
    dim, _ = DENSE_GEOMETRY[n]
    scene = synth.make_scene(seed=70 + n, n_boxes=8, rmin=3.0, rmax=0.4 * dim)
    out = []
    for k in range(scans):
        ex, ey, yaw = 0.9 * k, -0.6 * k, 0.15 * k
        pts, org = synth.lidar_scan(scene, (ex, ey), yaw, beams=32, az_steps=512, seed=7000 + 10 * n + k)
        near = near_returns(300, 7100 + 10 * n + k)
        near["x"] += np.float32(org[0])
        near["y"] += np.float32(org[1])
        pts = np.concatenate([pts, near]).astype(synth.POINT_DTYPE)   # concatenate drops the padding of the records
        if k:
            push_below_ground(pts, 500, 7200 + 10 * n + k)
        out.append((ex, ey, yaw, 0.02 * k, pts, org))
    return out


def config_limits(make, rec, n):
    """Every case of tests/config_limits.py on a fresh N x N map (N = 100: the TMA detection and the skewed spiral; N = 101:
    the plain-load detection on an odd map): three scans with a roll in between; the roll's moved flag and position, and
    labels, output order and cloud and all eleven layers after every scan, folded into one digest per case."""
    import config_limits as cl

    dim, res = DENSE_GEOMETRY[n]
    stream = config_limits_stream(n)
    for name, cfg in cl.CASES.items():
        m = make(dim, res)
        assert m.n == n
        m.set_config(**cfg)
        m.init_map(0.0, 0.0, 0.0)
        case = Folded(rec, name)
        for k, (ex, ey, yaw, base_z, pts, org) in enumerate(stream):
            if k:
                q, t = base_from_map_qt(ex, ey, yaw, base_z, pitch=0.02)
                update(m, case, ex, ey, q, t, f"roll {k}", layers=())
            scan(m, case, pts, org, base_z, f"scan {k}")
            if name == "minimum_distance_factor=0.0":   # cells of one point have variance 0: the label tolerance is 0 / 0
                assert ((m.layer("pointsRaw") == 1) & (m.layer("variance") == 0)).sum() > 100
        case.done()


SCENARIOS = {
    "expected_points_table": (expected_points_table, [()]),
    "cfg1_cfg2_64_beam_300": (cfg1_cfg2_64_beam_300, [()]),
    "cfg3_128_beam_600": (cfg3_128_beam_600, [()]),
    "cfg4_four_lidar_364": (cfg4_four_lidar_364, [()]),
    "rolling_stream_with_outliers": (rolling_stream_with_outliers, [()]),
    "large_jump_clears_the_map": (large_jump_clears_the_map, [()]),
    "random_geometry_and_config": (random_geometry_and_config, [(s,) for s in range(8)]),
    "geometry_primitives_agree": (geometry_primitives_agree, [()]),
    "single_phase_calls_agree": (single_phase_calls_agree, [()]),
    "full_size_stream": (full_size_stream, [(c,) for c in FULL_SIZES]),
    "input_orders": (input_orders, [()]),
    "dense_cells": (dense_cells, [(n,) for n in DENSE_GEOMETRY]),
    "nonfinite_heights": (nonfinite_heights, [()]),
    "far_from_origin": (far_from_origin, [(w,) for w in FAR_POSITIONS]),
    "far_geometry": (far_geometry, [(w,) for w in FAR_POSITIONS]),
    "nonfinite_confidence": (nonfinite_confidence, [()]),
    "detect_planes": (detect_planes, [(n,) for n in DETECT_SIZES]),
    "outlier_priors": (outlier_priors, [(w,) for w in OUTLIER_SIZES]),
    "crowded_cells": (crowded_cells, [()]),
    "config_limits": (config_limits, [(n,) for n in DENSE_GEOMETRY]),
}


def key(name, args):
    return name + "".join(f"[{a}]" for a in args)


def run(name, make, *args, record=False):
    """Runs scenario `name` on the implementation `make(dim, res)` builds; returns the digests it saw."""
    rec = Recorder(key(name, args), record)
    SCENARIOS[name][0](make, rec, *args)
    return rec.done()

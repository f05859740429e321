"""The CUDA path against the CPU oracle, bit for bit, on the inputs tests/cloud_orders.py makes: point orders other than
ring-major, cells with a chosen number of runs and points, non-finite heights at finite positions, maps far from the
origin.  Every other GPU test feeds ring-major clouds near (0, 0), for which the order recovery of k_cell_stats (register
network up to 8 runs, Shell sort above, first gap 57) and the run bookkeeping of k_rasterize / k_scatter are hardly
exercised; a wrong order only changes the last bits of variance / m2 / meanVariance, so nothing but these comparisons
would notice it.  tests/test_cloud_orders.py asserts (without a GPU) that the clouds reach the regimes named here."""
import numpy as np
import pytest

import cloud_orders as co
import ref_scenarios as rs
import sample_ref
from groundgrid_b200 import capi, synth
from oracle import Oracle, nextrows
from test_gpu_parity import DEAD, LIVE, assert_layers_equal, diff_report, make_pair

pytestmark = pytest.mark.gpu

ALL = ("points",) + LIVE + DEAD
GEOMETRIES = {300: (99.0, 0.33, "scan_64", 140000), 101: (33.33, 0.33, "scan_64", 140000), 364: (120.0, 0.33, "scan_4lidar", 520000)}
LADDER_GEOMETRIES = {100: (33.0, 0.33), 101: (33.33, 0.33), 300: (99.0, 0.33)}
PC_KEPT, PC_KEPT_BORDER, PC_IGNORED, PC_IGNORED_BORDER = 1, 2, 3, 4


def check_scan(g, o, pts, org, base_z, ctx, layers=ALL):
    """One whole scan on both: labels, output order, output cloud, layers."""
    labels, index, cloud = g.filter_cloud(pts, org, base_z, want_index=True, want_cloud=True)
    lab_o, idx_o, cloud_o = o.filter_cloud(pts, org, base_z, threads=1, want_cloud=True)
    assert np.array_equal(labels, lab_o), f"{ctx}: {(labels != lab_o).sum()} labels differ"
    assert np.array_equal(index, idx_o), f"{ctx}: output order"
    assert cloud.tobytes() == cloud_o.tobytes(), f"{ctx}: output cloud"
    assert_layers_equal(g, o, layers, ctx)
    return labels


def classes_on_a_fresh_map(pts, org, n, res, position, max_ring=1024):
    """gg_get_point_classes of a scan on a fresh map (no outliers): class << 24 | cell."""
    cell = co.cell_index(pts, n, res, position)
    inside = cell < n * n
    kept = co.kept_mask(pts, org, n, res, position, max_ring)
    i, j = cell % n, cell // n
    border = (n <= i + 3) | (n <= j + 3)
    cls = np.where(kept, np.where(border, PC_KEPT_BORDER, PC_KEPT), np.where(border, PC_IGNORED_BORDER, PC_IGNORED))
    return np.where(inside, (cls.astype(np.uint32) << 24) | cell.astype(np.uint32), 0).astype(np.uint32)


def two_clouds(n, seed):
    dim, res, sensor, maxp = GEOMETRIES[n]
    scene = synth.make_scene(seed=seed)
    return dim, res, maxp, [getattr(synth, sensor)(scene, seed=seed + k) for k in range(2)]


@pytest.mark.parametrize("n", list(GEOMETRIES))
@pytest.mark.parametrize("k", range(len(co.REORDERINGS)))
def test_two_scans_in_different_orders(n, k):
    """Two consecutive scans per handle, each in another order: the second relies on every per-cell counter having been
    zeroed cell by cell by the first."""
    dim, res, maxp, clouds = two_clouds(n, 5000 + n)
    full = bool(k & 1) or n == 300
    g, o = make_pair(dim, res, full=full, max_points=maxp)
    g.init_map(0.0, 0.0, 0.0)
    o.init_map(0.0, 0.0, 0.0)
    for s, (pts, org) in enumerate(clouds):
        name = co.REORDERINGS[(k + 3 * s) % len(co.REORDERINGS)]
        if s:
            rs.push_below_ground(pts, 2000, n + k)
        cloud, _ = co.reorder(name, pts, org, g.n, res, seed=k)
        check_scan(g, o, cloud, org, 0.0, f"N {n} scan {s} {name}", ALL if full else ("points",) + LIVE)
    g.close()


@pytest.mark.parametrize("name", ["shuffled", "firing", "cell_round_robin"])
@pytest.mark.parametrize("stage", [1, 2, 3])
def test_reordered_scan_phase_by_phase(name, stage):
    pts, org = synth.scan_64(synth.make_scene(seed=1234), seed=1234)
    cloud, _ = co.reorder(name, pts, org, 300, 0.33, seed=stage)
    g, o = make_pair(99.0, 0.33)
    g.init_map(0.0, 0.0, 0.0)
    o.init_map(0.0, 0.0, 0.0)
    g.run_single(cloud, org, 0.0, stop_after=stage)
    o.filter_cloud(cloud, org, 0.0, threads=1, stop_after=stage)
    assert_layers_equal(g, o, tuple(x for x in ALL if stage > 1 or x != "variance"), f"{name} stage {stage}")
    if stage == 1:
        assert np.array_equal(g.point_classes(len(cloud)), classes_on_a_fresh_map(cloud, org, 300, 0.33, (0.0, 0.0)))
    g.close()


def ladder(kind, n, res, position=(0.0, 0.0)):
    if kind == "runs":
        return co.runs_ladder(n, res, position, seed=n)
    return co.count_ladder(n, res, position, seed=n, scattered=kind == "count_scattered")


@pytest.mark.parametrize("n", list(LADDER_GEOMETRIES))
@pytest.mark.parametrize("kind", ["runs", "count_block", "count_scattered"])
def test_ladders_five_times_on_one_slot(n, kind):
    """Cells with exactly 1 .. 120 runs (both sides of the 8-run network and of every Shell gap) and with 1 .. 8 192 points
    (both sides of the worklist's 32 / 33 step, one cell beyond its last class).  The same cloud five times on one slot:
    the runs may arrive in another order every time, the result may not."""
    dim, res = LADDER_GEOMETRIES[n]
    pts, org, _ = ladder(kind, n, res)
    prof = co.run_profile(pts, org, n, res, (0.0, 0.0))
    assert prof.count.max() <= co.MAX_POINTS_PER_CELL and prof.runs.max() <= co.MAX_RUNS_PER_CELL
    print(f"{kind} N={n}: {prof}")
    g, o = make_pair(dim, res, max_points=65536)
    assert g.n == o.n == n
    g.init_map(0.0, 0.0, 0.0)
    o.init_map(0.0, 0.0, 0.0)
    g.profile_enable(True)
    first = None
    for rep in range(5):
        check_scan(g, o, pts, org, 0.0, f"{kind} N {n} repetition {rep}")
        stats = [g.layer(x) for x in ("m2", "meanVariance", "minGroundHeight", "variance")]
        if rep == 0:
            first = stats
            times = g.profile_read(reset=True)
            print(f"{kind} N={n}: first scan " + ", ".join(f"{k} {v[0]:.3f} ms" for k, v in times.items() if "cell_stats" in k or "rasterize" in k or "scatter" in k))
        assert all(diff_report("stats", a, b) is None for a, b in zip(stats, first)), f"repetition {rep} differs from the first"
    g.close()


def payload18(pts):
    raw = np.zeros((len(pts), 18), np.uint8)
    for name, off, width in zip(co.FIELDS, (0, 4, 8, 12, 16), (4, 4, 4, 4, 2)):
        raw[:, off:off + width] = np.ascontiguousarray(pts[name]).view(np.uint8).reshape(len(pts), width)
    return raw


ROUTES = ("filter_cloud", "batch_packed", "batch_raw", "upload_run", "to_device", "cloud_msgs")


@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("kind", ["shuffled", "runs_ladder"])
def test_every_input_route(monkeypatch, route, kind):
    """The same clouds through every way a cloud reaches k_rasterize (32-byte records from host or device memory, the
    packed SoA copy, the PointCloud2 unpack), twice on one slot."""
    import torch

    if route.startswith("batch"):
        monkeypatch.setenv("GG_HOST_PACK", "1" if route == "batch_packed" else "0")
    if kind == "shuffled":
        clouds = [(co.shuffled(p, s)[0], org) for s, (p, org) in enumerate(two_clouds(300, 6000)[3])]
    else:
        clouds = [co.runs_ladder(300, 0.33, seed=s)[:2] for s in (21, 22)]
    g, o = make_pair(99.0, 0.33)
    g.init_map(0.0, 0.0, 0.0)
    o.init_map(0.0, 0.0, 0.0)
    for s, (pts, org) in enumerate(clouds):
        want, idx_o, _ = o.filter_cloud(pts, org, 0.0, threads=1)
        if route == "filter_cloud":
            labels = g.filter_cloud(pts, org, 0.0)
        elif route.startswith("batch"):
            hp = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).pin_memory()
            hl = torch.zeros(len(pts), dtype=torch.uint8).pin_memory()
            g.filter_cloud_batch_ptrs(g.make_descs([0], [len(pts)], [org], [0.0]), [hp.data_ptr()], [hl.data_ptr()])
            labels = hl.numpy().copy()
            assert g.last_batch_transfer()[0] == (1 if route == "batch_packed" else 0)
        elif route == "upload_run":
            labels = g.run_single(pts, org, 0.0)
        else:
            if route == "to_device":
                dev = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).cuda()
                out = g.run_scans_to_device([dev], [0], [org], 0.0, select="all", index=True)
            else:
                dev = torch.from_numpy(payload18(pts)).cuda()
                out = g.run_cloud_msgs_to_device([dev], 18, (0, 4, 8, 12, 16), None, [0], [org], 0.0, select="all", index=True)
            torch.cuda.synchronize()
            labels = out.labels[0].cpu().numpy()
            count = int(out.counts[0].item())
            assert np.array_equal(out.index[0][:count].cpu().numpy().astype(np.uint32), idx_o), f"{route} scan {s}: output order"
        assert np.array_equal(labels, want), f"{route} {kind} scan {s}: {(labels != want).sum()} labels differ"
        assert_layers_equal(g, o, ALL, f"{route} {kind} scan {s}")
    g.close()


def test_batch_of_ten_slots_each_in_another_order():
    """Ten slots over several stream groups, every slot another order of another cloud, two calls with the orders rotated;
    slots 3 and 7 run their own configuration whose max_ring ignores the upper rings, which punches holes into the warps."""
    import torch

    B, dim, res = 10, 99.0, 0.33
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=131072, full_layers=True)
    oracles = []
    for b in range(B):
        o = Oracle(dim, res)
        if b in (3, 7):
            g.set_config(slot=b, max_ring=20 + b)
            o.set_config(max_ring=20 + b)
        g.init_map(0.1 * b, -0.05 * b, 0.0, slot=b)
        o.init_map(0.1 * b, -0.05 * b, 0.0)
        oracles.append(o)
    kinds = list(co.REORDERINGS) + ["runs_ladder", "count_ladder"]
    for call in range(2):
        clouds = []
        for b in range(B):
            kind = kinds[(b + 3 * call) % len(kinds)]
            pos = (0.1 * b, -0.05 * b)
            if kind == "runs_ladder":
                pts, org, _ = co.runs_ladder(g.n, res, pos, seed=b)
            elif kind == "count_ladder":
                pts, org, _ = co.count_ladder(g.n, res, pos, seed=b, scattered=True)
            else:
                pts, org = synth.scan_64(synth.make_scene(seed=7000 + b), ego_xy=pos, seed=7000 + 10 * call + b)
                pts, _ = co.reorder(kind, pts, org, g.n, res, pos, seed=b)
            clouds.append((pts, org))
        hp = [torch.from_numpy(np.ascontiguousarray(p).view(np.uint8).copy()).pin_memory() for p, _ in clouds]
        hl = [torch.zeros(len(p), dtype=torch.uint8).pin_memory() for p, _ in clouds]
        descs = g.make_descs(list(range(B)), [len(p) for p, _ in clouds], [org for _, org in clouds], [0.0] * B)
        g.filter_cloud_batch_ptrs(descs, [t.data_ptr() for t in hp], [t.data_ptr() for t in hl])
        for b in range(B):
            want, _, _ = oracles[b].filter_cloud(clouds[b][0], clouds[b][1], 0.0, threads=1)
            assert np.array_equal(hl[b].numpy(), want), f"call {call} slot {b}: {(hl[b].numpy() != want).sum()} labels differ"
            errs = [r for r in (diff_report(x, g.layer(x, slot=b), oracles[b].layer(x)) for x in ALL) if r]
            assert not errs, f"call {call} slot {b}: " + " | ".join(errs)
    g.close()


def test_full_scan_after_a_partial_one():
    """stop_after = 1 leaves the slot's per-cell counters and the raw point counts clean for a full scan of a differently
    ordered cloud."""
    dim, res, maxp, clouds = two_clouds(300, 8000)
    g, o = make_pair(dim, res)
    g.init_map(0.0, 0.0, 0.0)
    o.init_map(0.0, 0.0, 0.0)
    a, _ = co.shuffled(clouds[0][0], 1)
    g.run_single(a, clouds[0][1], 0.0, stop_after=1)
    o.filter_cloud(a, clouds[0][1], 0.0, threads=1, stop_after=1)
    assert_layers_equal(g, o, tuple(x for x in ALL if x != "variance"), "partial scan")
    b, _ = co.firing(*clouds[1])
    check_scan(g, o, b, clouds[1][1], 0.0, "full scan after the partial one")
    g.close()


def test_nonfinite_heights():
    """NaN, +inf and -inf heights at finite x, y run through the cell statistics, the patch sums, the spiral and the
    label rule: every layer with NaN as NaN and inf with its sign, labels, output order; the 8-bit image and the
    sampled values of the NaN-laden terrain; then a roll and a finite scan."""
    import torch

    g, o = make_pair(99.0, 0.33)
    g.init_map(0.0, 0.0, 0.0)
    o.init_map(0.0, 0.0, 0.0)
    scene = synth.make_scene(seed=606)
    for k in range(3):
        ex, ey = (0.0, 0.0) if k < 2 else (1.7, -0.8)
        pts, org = synth.scan_64(scene, (ex, ey), seed=610 + k)
        if k < 2:
            pts = co.nonfinite_heights(pts, seed=620 + k)
        else:
            T = synth.base_from_map(ex, ey, 0.0, base_z=0.0, pitch=0.01)
            assert int(g.update_pose(ex, ey, T)) == o.update(ex, ey, T) == 1
            assert_layers_equal(g, o, ("ground", "groundpatch"), "after the roll")
        labels = check_scan(g, o, pts, org, 0.0, f"non-finite scan {k}")
        ground = o.layer("ground")
        if k < 2:
            assert np.isnan(ground).sum() > 1000 and (labels == 49).sum() > 1000
            img, lo, hi = g.layer_image_u8("ground")
            want, wlo, whi = nextrows.layer_image_u8(ground)
            assert np.array_equal(img, want) and (lo, hi) == (wlo, whi), f"scan {k}: 8-bit image of the terrain"
            xy = torch.from_numpy(np.stack([pts["x"], pts["y"]], 1).copy()).cuda()
            got = g.sample_layers_to_device([0], [xy], names=("ground",), mode="nearest")[0]
            px, py = o.position()
            vals, _ = sample_ref.sample_layers([ground], g.n, 0.33, px, py, pts["x"], pts["y"], "nearest")
            torch.cuda.synchronize()
            assert np.array_equal(got.cpu().numpy(), vals, equal_nan=True), f"scan {k}: sampled terrain"   # NaN as NaN, inf with its sign
    g.close()


@pytest.mark.parametrize("where", list(rs.FAR_POSITIONS))
@pytest.mark.parametrize("route", ["single", "batch"])
def test_far_from_origin(where, route):
    """A rolling stream on a map 1e5 .. 6e6 m from the origin (float32 coordinates 0.008 .. 0.5 m apart: points pile up
    on cell edges), through gg_update_pose + gg_filter_cloud and through the batched calls, against the oracle at every
    step; then the terrain and the heights at the scan's own points."""
    import torch

    pos = rs.FAR_POSITIONS[where]
    g, o = make_pair(99.0, 0.33)
    g.init_map(pos[0], pos[1], 0.0)
    o.init_map(pos[0], pos[1], 0.0)
    for k, ex, ey, yaw, base_z, (q, t), pts, org in rs.far_stream(where):
        T = synth.tf2_matrix(q, t)
        if k:
            if route == "single":
                moved = int(g.update_pose(ex, ey, T))
            else:
                moved = int(g.update_pose_batch([0], [[ex, ey]], [T.reshape(12)])[0])
            assert moved == o.update(ex, ey, T) == 1
            assert np.array_equal(g.position(), o.position())
            assert_layers_equal(g, o, ("ground", "groundpatch"), f"{where} roll {k}")
        if route == "single":
            check_scan(g, o, pts, org, base_z, f"{where} scan {k}")
        else:
            hp = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).pin_memory()
            hl = torch.zeros(len(pts), dtype=torch.uint8).pin_memory()
            g.filter_cloud_batch_ptrs(g.make_descs([0], [len(pts)], [org], [base_z]), [hp.data_ptr()], [hl.data_ptr()])
            want, _, _ = o.filter_cloud(pts, org, base_z, threads=1)
            assert np.array_equal(hl.numpy(), want), f"{where} scan {k}: {(hl.numpy() != want).sum()} labels differ"
            assert_layers_equal(g, o, ALL, f"{where} batched scan {k}")
        if k in (1, 4):
            ground = o.layer("ground")
            px, py = o.position()
            vals, cells = sample_ref.sample_layers([ground], g.n, 0.33, px, py, pts["x"], pts["y"], "nearest")
            xy = torch.from_numpy(np.stack([pts["x"], pts["y"]], 1).copy()).cuda()
            got, got_cells = g.sample_layers_to_device([0], [xy], names=("ground",), mode="nearest", cells=True)
            codes, height = g.point_info_to_device([0])
            torch.cuda.synchronize()
            assert np.array_equal(got_cells[0].cpu().numpy(), cells), f"{where} scan {k}: cells of the scan's points"
            assert np.array_equal(got[0].cpu().numpy().view(np.uint32), vals.view(np.uint32)), f"{where} scan {k}: sampled terrain"
            inside = cells >= 0
            assert np.array_equal((codes[0].cpu().numpy() & 0xFFFFFF)[inside], cells[inside])
            assert np.array_equal(height[0].cpu().numpy()[inside], (pts["z"] - vals[0])[inside]), f"{where} scan {k}: heights"
    g.close()


@pytest.mark.parametrize("name,args", [("input_orders", ()), ("dense_cells", (100,)), ("dense_cells", (101,)), ("nonfinite_heights", ()),
                                       ("far_from_origin", ("1.2e5",)), ("far_from_origin", ("5.6e6",))])
def test_cuda_path_against_the_reference_itself(name, args):
    """The same inputs against the reference's own answers (tests/golden/ref_digests.json)."""
    rs.run(name, lambda dim, res: rs.Cuda(dim, res, 140000), *args)

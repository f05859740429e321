"""The CUDA path against the CPU oracle, bit for bit, at the sizes a handle accepts (tests/large_clouds.py): scans across
the tile edges of the output scan (k_out_scan carries its running total from one 4096-count tile to the next only above
1 397 760 points), cells with more than 2^24 points (where the reference's float counts of "pointsRaw" and "points"
stop), the largest cloud a handle takes (2^26 - 256 points), and maps of 4094 .. 4096 cells per side (bit 23 of the
point code's 24-bit cell set, the "not rasterised" key equal to N^2).  tests/test_large_clouds.py checks without a GPU
that the clouds reach these regimes.

The GPUs these run on are shared: every large case first reads the free device and host memory and skips with the
shortfall when there is not enough, and every handle is destroyed and torch's cache emptied before the next test.
"""
import gc
import os
import time

import numpy as np
import pytest

import cloud_orders as co
import large_clouds as lc
from groundgrid_b200 import capi, synth
from oracle import Oracle, nextrows
from test_gpu_input_orders import ALL, check_scan, classes_on_a_fresh_map, payload18
from test_gpu_parity import assert_layers_equal, diff_report, make_pair

pytestmark = pytest.mark.gpu

GIB = 1 << 30
HANDLE_BYTES_PER_POINT = 69 + 32       # a slot's per-point buffers, and the output cloud's 32-byte records
SLOT_BYTES_PER_CELL = 110              # an N x N slot with every layer (N = 4096: about 1.8 GB), plus its detect table


@pytest.fixture(autouse=True)
def _release():
    """Handles are closed by the tests; what is left of torch's and Python's memory goes before the next test."""
    yield
    import torch

    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def need(device_bytes, host_bytes, what):
    import torch

    free, _ = torch.cuda.mem_get_info()
    host = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if free < device_bytes:
        pytest.skip(f"{what}: needs {device_bytes / GIB:.1f} GiB of device memory, {free / GIB:.1f} GiB free "
                    f"({(device_bytes - free) / GIB:.1f} GiB short)")
    if host < host_bytes:
        pytest.skip(f"{what}: needs {host_bytes / GIB:.1f} GiB of host memory, {host / GIB:.1f} GiB available "
                    f"({(host_bytes - host) / GIB:.1f} GiB short)")


def device_need(points, n, slots=1, buffers=0):
    """Device bytes of a handle of `slots` slots of `points` capacity on an N x N map, plus the test's own buffers."""
    return slots * (points * HANDLE_BYTES_PER_POINT + n * n * SLOT_BYTES_PER_CELL + (256 << 20)) + buffers + (1 << 30)


def report(ctx, t0):
    """Wall time of a test, torch's peak allocations and the device memory in use once its handles are closed."""
    import torch

    free, total = torch.cuda.mem_get_info()
    print(f"{ctx}: {time.perf_counter() - t0:.1f} s, torch peak {torch.cuda.max_memory_allocated() / GIB:.2f} GiB, "
          f"device in use at the end {(total - free) / GIB:.2f} GiB")


def cuda_records(pts):
    import torch

    return torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).reshape(-1)).cuda()


def selected_cloud(pts, labels, idx):
    """The output records of the points idx: the input record with the label as intensity."""
    out = co.take(pts, idx)
    out["intensity"] = labels[idx].astype(np.float32)
    return out


def assert_device_outputs(out, k, pts, labels, classes, select, ctx):
    """Labels, count, index and cloud of scan k of a DeviceOutputs against the oracle's labels and classes."""
    want = lc.output_order(classes, labels, lc.SELECTS[select])
    count = int(out.counts[k].item())
    assert np.array_equal(out.labels[k].cpu().numpy(), labels), f"{ctx}: labels"
    assert count == len(want), f"{ctx}: count {count}, want {len(want)}"
    assert np.array_equal(out.index[k][:count].cpu().numpy().astype(np.uint32), want), f"{ctx}: output order"
    got = out.cloud[k][:count].cpu().numpy().view(lc.POINT_DTYPE).reshape(-1)
    w = selected_cloud(pts, labels, want)
    for f in co.FIELDS:
        assert np.array_equal(got[f], w[f]), f"{ctx}: output cloud field {f}"


def fresh_with_prior(g, o):
    g.init_map(0.0, 0.0, 0.0)
    o.init_map(0.0, 0.0, 0.0)
    p0, org0 = lc.prior_scan()
    check_scan(g, o, p0, org0, 0.0, "prior scan")


# ---- scans across the tile edges of the output scan --------------------------------------------------------------------
@pytest.mark.parametrize("n_points", lc.BOUNDARY_SIZES)
def test_boundary_cloud_every_route(n_points):
    """A scan of 1 397 760 .. 3 000 000 points after an ordinary one (its outliers tested against the prior that one
    left): gg_filter_cloud with labels, index, cloud and every layer; gg_run_scans_to_device with every select, with the
    counts; gg_run_cloud_msgs_to_device on 18-byte payloads.  Each route starts from a fresh map and the same prior."""
    t0 = time.perf_counter()
    need(device_need(n_points, 300, buffers=n_points * 64), n_points * 200, f"{n_points} points")
    pts, org = lc.boundary_cloud(n_points)
    g, o = make_pair(*lc.BOUNDARY_GEOMETRY, max_points=n_points)
    try:
        fresh_with_prior(g, o)
        labels, index, cloud, classes = o.filter_cloud(pts, org, 0.0, want_cloud=True, want_classes=True)
        layers = {x: o.layer(x) for x in ALL}
        got, gidx, gcloud = g.filter_cloud(pts, org, 0.0, want_index=True, want_cloud=True)
        assert np.array_equal(got, labels), f"{n_points} points: {(got != labels).sum()} labels differ"
        assert np.array_equal(gidx, index), f"{n_points} points: output order"
        assert gcloud.tobytes() == cloud.tobytes(), f"{n_points} points: output cloud"
        assert_layers_equal(g, o, ALL, f"{n_points} points")
        assert np.array_equal(lc.output_order(classes, labels), index)
        codes = g.point_classes(len(pts))
        assert np.array_equal(codes >> 24, classes), "point classes"
        del got, gidx, gcloud, cloud
        for select in ("all", "ground", "nonground"):
            for route in ("to_device", "cloud_msgs"):
                if route == "cloud_msgs" and select != "all":
                    continue
                fresh_with_prior(g, Oracle(*lc.BOUNDARY_GEOMETRY))
                if route == "to_device":
                    out = g.run_scans_to_device([cuda_records(pts)], [0], [org], 0.0, select=select, index=True)
                else:
                    import torch

                    dev = torch.from_numpy(payload18(pts)).cuda()
                    out = g.run_cloud_msgs_to_device([dev], 18, (0, 4, 8, 12, 16), None, [0], [org], 0.0, select=select, index=True)
                ctx = f"{n_points} points {route} select {select}"
                assert_device_outputs(out, 0, pts, labels, classes, select, ctx)
                errs = [r for r in (diff_report(x, g.layer(x), layers[x]) for x in ALL) if r]
                assert not errs, f"{ctx}: " + " | ".join(errs)
                del out
    finally:
        g.close()
    report(f"boundary cloud {n_points}", t0)


def test_batch_small_scans_inside_a_large_launch(monkeypatch):
    """Four slots on one stream group with 0, 1000, 1 397 761 and 3 000 000 points: the output scan of the launch runs
    over the 3 * 2930 block counts of the largest, so the small scans' totals come after many tiles of zero counts."""
    t0 = time.perf_counter()
    sizes = (0, 1000, lc.TILE_EDGE + 1, 3_000_000)
    need(device_need(max(sizes), 300, slots=4, buffers=sum(sizes) * 64), sum(sizes) * 200, "a batch of four slots")
    import torch

    monkeypatch.setenv("GG_STREAMS", "1")
    g = capi.GroundGridB200(*lc.BOUNDARY_GEOMETRY, n_slots=4, max_points=max(sizes), full_layers=True)
    try:
        assert g.n_streams == 1
        scans, oracles = [], []
        p0, org0 = lc.prior_scan()
        for b, n in enumerate(sizes):
            o = Oracle(*lc.BOUNDARY_GEOMETRY)
            o.init_map(0.0, 0.0, 0.0)
            g.init_map(0.0, 0.0, 0.0, slot=b)
            o.filter_cloud(p0, org0, 0.0)
            oracles.append(o)
            scans.append((co.take(p0, np.arange(n)), org0) if n <= 1000 else lc.boundary_cloud(n, seed=b))
        g.run_scans_to_device([cuda_records(p0)] * 4, [0, 1, 2, 3], [org0] * 4, 0.0, select=None)
        for select in ("all", "nonground"):   # the second call runs the same scans on the maps the first one left
            want = [o.filter_cloud(p, org, 0.0, want_classes=True) for o, (p, org) in zip(oracles, scans)]
            devs = [cuda_records(p) if len(p) else torch.empty(0, dtype=torch.uint8, device="cuda") for p, _ in scans]
            out = g.run_scans_to_device(devs, [0, 1, 2, 3], [org for _, org in scans], 0.0, select=select, index=True)
            for b in range(4):
                labels, _, _, classes = want[b]
                ctx = f"slot {b} ({sizes[b]} points) select {select}"
                assert_device_outputs(out, b, scans[b][0], labels, classes, select, ctx)
                errs = [r for r in (diff_report(x, g.layer(x, slot=b), oracles[b].layer(x)) for x in ALL) if r]
                assert not errs, f"{ctx}: " + " | ".join(errs)
    finally:
        g.close()
    report("batch of four slots", t0)


# ---- cells past 2^24 points ----------------------------------------------------------------------------------------------
PILES = [("ring", c) for c in lc.PILE_SIZES] + [("near", lc.FLOAT_STOP + 2), ("near", 1 << 25)]


@pytest.mark.parametrize("how,count", PILES)
def test_pile(how, count):
    """One cell of 2^24 - 1 .. 2^25 ignored points: "pointsRaw" and "points" stop at 2^24 like the reference's float
    counts; labels, output order and cloud, every layer; the terrain image, the 8-bit image of "pointsRaw" and the
    evaluation tallies against oracle/nextrows.py on the oracle's results."""
    t0 = time.perf_counter()
    total = count + 1000
    need(device_need(total, 100, buffers=total * 8), total * 200, f"a pile of {count} points")
    pts, org, cell, _ = lc.pile(count, how)
    g, o = make_pair(*lc.PILE_GEOMETRY, max_points=len(pts))
    try:
        g.init_map(0.0, 0.0, 0.0)
        o.init_map(0.0, 0.0, 0.0)
        labels = check_scan(g, o, pts, org, 0.0, f"pile {how} {count}")
        raw = g.layer("pointsRaw").ravel(order="F")[cell]
        mine = co.cell_index(pts, 100, 0.33, (0.0, 0.0)) == cell
        assert raw == min(int(mine.sum()), lc.FLOAT_STOP)
        assert g.layer("points").ravel(order="F")[cell] == min(int((labels[mine] == 99).sum()), lc.FLOAT_STOP)
        want = nextrows.terrain_image(o.layer("ground"), o.layer("pointsRaw"))
        assert np.array_equal(g.terrain_image().view(np.uint32), want.view(np.uint32)), "terrain image"
        img, lo, hi = g.layer_image_u8("pointsRaw")
        wimg, wlo, whi = nextrows.layer_image_u8(o.layer("pointsRaw"))
        assert np.array_equal(img, wimg) and (lo, hi) == (wlo, whi), "8-bit image of pointsRaw"
        g.eval_accumulate()
        assert np.array_equal(g.eval_read(reset=True), nextrows.eval_counts(labels, pts["ring"])), "evaluation tallies"
    finally:
        g.close()
    report(f"pile {how} {count}", t0)


# ---- the largest cloud a handle takes ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", list(lc.CAPACITY_GEOMETRIES))
def test_capacity_cloud(n):
    """2^26 - 256 points on one slot of N = 300 and N = 4096, once through each route: gg_filter_cloud (labels, output
    order and cloud, point classes, point info, tallies), gg_run_scans_to_device, and a merged scan of three PointCloud2
    payloads whose parts fill the capacity exactly.  Each route starts from a fresh map."""
    import torch

    t0 = time.perf_counter()
    N = lc.CAPACITY
    need(device_need(N, n, buffers=N * 45), 13 * GIB, "the capacity cloud")
    dim, res = lc.CAPACITY_GEOMETRIES[n]
    pts, org = lc.capacity_cloud(n)
    o = Oracle(dim, res)
    o.init_map(0.0, 0.0, 0.0)
    t = time.perf_counter()
    labels, index, _, classes = o.filter_cloud(pts, org, 0.0, want_classes=True)
    print(f"oracle on {N} points, N = {n}: {time.perf_counter() - t:.1f} s")
    layers = {x: o.layer(x) for x in ALL}
    del o
    g = capi.GroundGridB200(dim, res, n_slots=1, max_points=N, full_layers=True)
    try:
        assert g.n == n
        g.init_map(0.0, 0.0, 0.0)
        got, gidx, gcloud = g.filter_cloud(pts, org, 0.0, want_index=True, want_cloud=True)
        assert np.array_equal(got, labels), f"{(got != labels).sum()} labels differ"
        assert np.array_equal(gidx, index), "output order"
        w = selected_cloud(pts, labels, index)
        for f in co.FIELDS:
            assert np.array_equal(gcloud[f], w[f]), f"output cloud field {f}"
        del gcloud, w, got, gidx
        errs = [r for r in (diff_report(x, g.layer(x), layers[x]) for x in ALL) if r]
        assert not errs, " | ".join(errs)
        codes = g.point_classes(N)
        assert np.array_equal(codes >> 24, classes), "point classes"
        dcodes, _ = g.point_info_to_device([0], height=False)
        assert np.array_equal(dcodes[0].cpu().numpy().view(np.uint32), codes), "point info codes"
        del dcodes, codes
        g.eval_accumulate()
        assert np.array_equal(g.eval_read(reset=True), nextrows.eval_counts(labels, pts["ring"])), "evaluation tallies"

        g.init_map(0.0, 0.0, 0.0)
        dev = cuda_records(pts)
        out = g.run_scans_to_device([dev], [0], [org], 0.0, select="all", index=True)
        assert_device_outputs(out, 0, pts, labels, classes, "all", "to_device")
        del out, dev

        g.init_map(0.0, 0.0, 0.0)
        cut = [0, N // 3 + 17, 2 * N // 3 - 5, N]
        raw = payload18(pts)                       # 1.2 GB: three parts of 18-byte records, together exactly N points
        parts = [torch.from_numpy(raw[a:b]).cuda() for a, b in zip(cut[:-1], cut[1:])]
        del raw
        out = g.run_merged_cloud_msgs_to_device([parts], 18, (0, 4, 8, 12, 16), None, [0], [org], 0.0, select="all", index=True)
        assert_device_outputs(out, 0, pts, labels, classes, "all", "merged payloads")
        errs = [r for r in (diff_report(x, g.layer(x), layers[x]) for x in ALL) if r]
        assert not errs, "merged payloads: " + " | ".join(errs)
        del out, parts
    finally:
        g.close()
    report(f"capacity cloud N = {n}", t0)


# ---- maps of 4094 .. 4096 cells per side ---------------------------------------------------------------------------------
ROLLS = {"+1 -1": (1, -1), "-2048 +2048": (-2048, 2048), "N - 1": ("N-1", 0), "more than N": ("N+5", -3)}


def cells_of(v, n):
    return n - 1 if v == "N-1" else n + 5 if v == "N+5" else v


@pytest.mark.parametrize("n", list(lc.WIDE_GEOMETRIES))
def test_wide_map(n):
    """Sprinkles over every border row and column, the corners, cells with bit 23 set and the last inner cell: classes
    after rasterisation against the numpy restatement; then scans with rolls of +-1, +-2048, N - 1 and more than N cells
    between them, each on labels and every layer; the layer images and the terrain image against oracle/nextrows.py."""
    import torch

    t0 = time.perf_counter()
    dim, res = lc.WIDE_GEOMETRIES[n]
    assert capi.host_cells_per_side(dim, res) == n
    need(device_need(1 << 20, n, slots=1, buffers=n * n * 20), 6 * GIB, f"an N = {n} map")
    r = float(np.float32(res))
    g, o = make_pair(dim, res, max_points=1 << 20)
    try:
        assert g.n == o.n == n
        g.init_map(0.0, 0.0, 0.0)
        o.init_map(0.0, 0.0, 0.0)
        pts, org, _ = lc.sprinkle(n)
        g.run_single(pts, org, 0.0, stop_after=1)
        assert np.array_equal(g.point_classes(len(pts)), classes_on_a_fresh_map(pts, org, n, res, (0.0, 0.0))), "classes"
        check_scan(g, o, pts, org, 0.0, f"N {n} scan 0")
        ex = ey = 0.0
        for k, (name, (di, dj)) in enumerate(ROLLS.items()):
            ex += cells_of(di, n) * r
            ey += cells_of(dj, n) * r
            T = synth.base_from_map(ex, ey, 0.0, base_z=0.0)
            assert int(g.update_pose(ex, ey, T)) == o.update(ex, ey, T) == 1, name
            assert np.array_equal(g.position(), o.position()), name
            assert_layers_equal(g, o, ("ground", "groundpatch"), f"N {n} roll {name}")
            pts, org, _ = lc.sprinkle(n, tuple(o.position()), seed=k + 1)
            check_scan(g, o, pts, org, 0.0, f"N {n} scan after roll {name}")
        names = ("ground", "groundpatch", "pointsRaw", "variance")
        imgs, ranges = g.layer_images_to_device([0], names)
        terrain = g.terrain_images_to_device([0])
        torch.cuda.synchronize()
        for l, name in enumerate(names):
            want, lo, hi = nextrows.layer_image_u8(o.layer(name))
            assert np.array_equal(imgs[0, l].cpu().numpy(), want), f"N {n}: 8-bit image of {name}"
            assert tuple(ranges[0, l].cpu().numpy().tolist()) == (lo, hi), f"N {n}: range of {name}"
        want = nextrows.terrain_image(o.layer("ground"), o.layer("pointsRaw"))
        assert np.array_equal(terrain[0].cpu().numpy().view(np.uint32), want.view(np.uint32)), f"N {n}: terrain image"
    finally:
        g.close()
    report(f"N = {n}", t0)


def test_wide_maps_batch_of_two_slots():
    """Two N = 4096 slots of one handle, each on its own configuration, through the batched host-buffer path."""
    import torch

    t0 = time.perf_counter()
    dim, res = lc.WIDE_GEOMETRIES[4096]
    need(device_need(1 << 20, 4096, slots=2), 8 * GIB, "two N = 4096 slots")
    g = capi.GroundGridB200(dim, res, n_slots=2, max_points=1 << 20, full_layers=True)
    try:
        cfgs = ({"max_ring": 40}, {"minimum_point_height_obstacle_threshold": 0.3, "patch_size_change_distance": 500.0})
        oracles = []
        for b, cfg in enumerate(cfgs):
            o = Oracle(dim, res)
            g.set_config(slot=b, **cfg)
            o.set_config(**cfg)
            g.init_map(0.5 * b, -0.5 * b, 0.0, slot=b)
            o.init_map(0.5 * b, -0.5 * b, 0.0)
            oracles.append(o)
        for call in range(2):
            clouds = [lc.sprinkle(4096, tuple(oracles[b].position()), seed=10 + 2 * call + b)[:2] for b in range(2)]
            hp = [torch.from_numpy(np.ascontiguousarray(p).view(np.uint8).copy()).pin_memory() for p, _ in clouds]
            hl = [torch.zeros(len(p), dtype=torch.uint8).pin_memory() for p, _ in clouds]
            g.filter_cloud_batch_ptrs(g.make_descs([0, 1], [len(p) for p, _ in clouds], [org for _, org in clouds], [0.0, 0.0]),
                                      [t.data_ptr() for t in hp], [t.data_ptr() for t in hl])
            for b in range(2):
                want, _, _ = oracles[b].filter_cloud(*clouds[b], 0.0)
                assert np.array_equal(hl[b].numpy(), want), f"call {call} slot {b}: {(hl[b].numpy() != want).sum()} labels differ"
                errs = [r for r in (diff_report(x, g.layer(x, slot=b), oracles[b].layer(x)) for x in ALL) if r]
                assert not errs, f"call {call} slot {b}: " + " | ".join(errs)
    finally:
        g.close()
    report("two N = 4096 slots", t0)

"""Device-resident outputs (gg_run_scans_to_device): labels and the segmented cloud written into caller-owned CUDA
memory, ordered on the caller's stream.  Every check is bit-exact against a twin handle driven through
gg_run_scans_device + gg_download_labels + gg_get_output (and, for one slot per step, against the oracle)."""
import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from oracle import Oracle

pytestmark = pytest.mark.gpu

LIVE = ("points", "variance", "minGroundHeight", "ground", "groundpatch")
DEAD = ("m2", "meanVariance", "groundCandidates", "planeDist", "maxGroundHeight", "pointsRaw")
SELECTS = ("all", "nonground", "ground")
# two slots of every handle run a configuration other than the default one
OTHER_CFGS = [
    dict(max_ring=48, occupied_cells_decrease_factor=1.5, patch_size_change_distance=8.0, miminum_point_height_threshold=0.2,
         minimum_point_height_obstacle_threshold=0.05, outlier_tolerance=0.25, min_outlier_detection_ground_confidence=0.6),
    dict(max_ring=40, occupied_cells_decrease_factor=2000.0, patch_size_change_distance=30.0, distance_factor=0.0003,
         outlier_tolerance=0.05, point_count_cell_variance_threshold=20),
]


def torch_mod():
    import torch

    return torch


def make_pair(dim, res, B, full_layers=False, max_points=65536):
    """(handle under test, twin) with identical per-slot configurations; slots 1 and B - 1 run OTHER_CFGS."""
    hs = [capi.GroundGridB200(dim, res, n_slots=B, max_points=max_points, full_layers=full_layers) for _ in range(2)]
    for h in hs:
        for slot, kw in zip((1, B - 1), OTHER_CFGS):
            h.set_config(slot=slot, **kw)
    return hs


def make_steps(B, steps, seed):
    """[step][slot] -> (points, origin, ego xy, T): rolls between steps, pushed-down below-ground returns."""
    rng = np.random.default_rng(seed)
    scenes = [synth.make_scene(seed=seed + b, stream_len=10.0, undulation=0.2) for b in range(B)]
    out = []
    for k in range(steps):
        row = []
        for b in range(B):
            ex, ey, yaw = 0.8 * k + 0.05 * b, -0.35 * k * (b % 3), 0.04 * k * (1 + b % 2)
            pts, org = synth.lidar_scan(scenes[b], ego_xy=(ex, ey), yaw=yaw, beams=64, az_steps=768, seed=seed + 100 * k + b)
            if k:
                idx = rng.choice(len(pts), len(pts) // 200, replace=False)
                pts["z"][idx] -= rng.uniform(0.3, 1.2, len(idx)).astype(np.float32)
            row.append((pts, org, (ex, ey), synth.base_from_map(ex, ey, yaw, base_z=0.0, pitch=0.01)))
        out.append(row)
    return out


def to_device(pts):
    torch = torch_mod()
    return torch.from_numpy(np.ascontiguousarray(pts).view(np.float32).reshape(-1, 8).copy()).cuda()


def advance(handles, k, row, slots):
    """init_map (step 0) or one batched roll (later steps) on every handle."""
    for h in handles:
        if k == 0:
            for b, r in enumerate(row):
                h.init_map(r[2][0], r[2][1], 0.0, slot=int(slots[b]))
        else:
            h.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))


def twin_run(twin, slots, row, dev, base_z):
    """Labels, output index and output cloud of every scan through the existing calls."""
    descs = twin.make_descs(list(slots), [len(r[0]) for r in row], [r[1] for r in row], [base_z] * len(row))
    twin.run_scans_device(descs, [t.data_ptr() for t in dev])
    labels = [twin.download_labels(len(r[0]), slot=int(s)) for s, r in zip(slots, row)]
    twin.synchronize()
    outs = [twin.get_output(slot=int(s), want_cloud=True) for s in slots]
    return labels, [o[0] for o in outs], [o[1] for o in outs]


def selected(labels, index, cloud, select):
    """The twin's output cloud restricted to `select`, order kept: (index, raw records [n, 32] bytes).  The records are
    masked as raw bytes: indexing the structured array would not carry its padding bytes over."""
    lab = labels[index]
    keep = {"all": np.ones(len(index), bool), "nonground": lab == capi.LABEL_NONGROUND, "ground": lab == capi.LABEL_GROUND}[select]
    return index[keep], np.ascontiguousarray(cloud).view(np.uint8).reshape(-1, 32)[keep]


def records(cloud_view):
    """float32 [n, 8] device records -> raw bytes [n, 32]."""
    return cloud_view.cpu().numpy().view(np.uint8).reshape(-1, 32)


def check_outputs(out, select, want_labels, want_index, want_cloud, ctx, with_index=True):
    torch = torch_mod()
    torch.cuda.synchronize()
    counts = out.counts.cpu().numpy()
    cloud, index = out.trimmed()
    for k in range(len(want_labels)):
        assert np.array_equal(out.labels[k].cpu().numpy(), want_labels[k]), f"{ctx} scan {k}: labels"
        wi, wc = selected(want_labels[k], want_index[k], want_cloud[k], select)
        assert counts[k] == len(wi), f"{ctx} scan {k}: count {counts[k]} != {len(wi)}"
        assert np.array_equal(records(cloud[k]), wc), f"{ctx} scan {k}: cloud"
        if with_index:
            assert np.array_equal(index[k].cpu().numpy().view(np.uint32), wi), f"{ctx} scan {k}: index"


def assert_layers_equal(g, twin, slots, names, ctx):
    for s in slots:
        for name in names:
            a, b = g.layer(name, slot=int(s)), twin.layer(name, slot=int(s))
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{ctx} slot {s}: layer {name} differs"


def assert_state_equal(g, twin, slots, row, names, ctx):
    """Layers, gg_download_labels and gg_get_output of the handle under test equal the twin's."""
    assert_layers_equal(g, twin, slots, names, ctx)
    for s, r in zip(slots, row):
        s = int(s)
        gl, tl = g.download_labels(len(r[0]), slot=s), twin.download_labels(len(r[0]), slot=s)
        g.synchronize()
        twin.synchronize()
        assert np.array_equal(gl, tl), f"{ctx} slot {s}: labels"
        gi, gc = g.get_output(slot=s, want_cloud=True)
        ti, tc = twin.get_output(slot=s, want_cloud=True)
        assert np.array_equal(gi, ti) and gc.tobytes() == tc.tobytes(), f"{ctx} slot {s}: get_output"


@pytest.mark.parametrize("dim,res,B,full_layers", [
    (99.0, 0.33, 4, True),       # N = 300: TMA patch detection, one slot per stream group
    (99.0, 0.33, 10, False),     # ten slots over eight stream groups
    (33.33, 0.33, 10, True),     # N = 101: plain-load patch detection
    (33.33, 0.33, 4, False),
])
def test_parity_with_the_twin_over_a_rolling_stream(dim, res, B, full_layers):
    g, twin = make_pair(dim, res, B, full_layers)
    o = Oracle(dim, res)                                 # slot 0 runs the default configuration
    slots = np.arange(B, dtype=np.int32)[::-1].copy()   # batch order differs from slot order
    names = LIVE + (DEAD if full_layers else ())
    steps = make_steps(B, 4, seed=5100 + B)
    for k, row in enumerate(steps):
        advance((g, twin), k, row, slots)
        if k == 0:
            o.init_map(row[-1][2][0], row[-1][2][1], 0.0)
        else:
            o.update(row[-1][2][0], row[-1][2][1], row[-1][3])
        dev = [to_device(r[0]) for r in row]
        select = SELECTS[k % 3]
        base_z = 0.02 * k
        out = g.run_scans_to_device(dev, slots, [r[1] for r in row], base_z, labels=True, select=select, index=True)
        want_labels, want_index, want_cloud = twin_run(twin, slots, row, dev, base_z)
        ctx = f"step {k} select {select}"
        check_outputs(out, select, want_labels, want_index, want_cloud, ctx)
        # slot 0 (last in the batch) against the oracle as well
        ol, oi, _ = o.filter_cloud(row[-1][0], row[-1][1], base_z, threads=1)
        assert np.array_equal(out.labels[-1].cpu().numpy(), ol) and np.array_equal(want_index[-1], oi), f"{ctx}: oracle"
        assert_state_equal(g, twin, slots, row, names, ctx)
    g.close()
    twin.close()


def test_every_select_gives_the_filtered_output_cloud():
    """The three selections on the same scans (each from the same map state), plus no selection at all."""
    dim, res, B = 99.0, 0.33, 6
    steps = make_steps(B, 2, seed=5300)
    slots = np.arange(B, dtype=np.int32)
    for select in SELECTS + (None,):
        g, twin = make_pair(dim, res, B)
        for k, row in enumerate(steps):
            advance((g, twin), k, row, slots)
            dev = [to_device(r[0]) for r in row]
            out = g.run_scans_to_device(dev, slots, [r[1] for r in row], 0.0, labels=True, select=select, index=select is not None)
            want = twin_run(twin, slots, row, dev, 0.0)
            if select is None:
                torch_mod().cuda.synchronize()
                assert out.cloud is None and out.index is None and out.counts is None
                for k2 in range(B):
                    assert np.array_equal(out.labels[k2].cpu().numpy(), want[0][k2])
            else:
                check_outputs(out, select, *want, f"step {k} select {select}")
            assert_state_equal(g, twin, slots, row, LIVE, f"step {k} select {select}")
        g.close()
        twin.close()


def test_labels_only_needs_only_the_write_pass():
    dim, res, B = 33.33, 0.33, 5
    g, twin = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    torch = torch_mod()
    for k, row in enumerate(make_steps(B, 2, seed=5400)):
        advance((g, twin), k, row, slots)
        dev = [to_device(r[0]) for r in row]
        descs = g.make_descs(list(slots), [len(r[0]) for r in row], [r[1] for r in row], [0.0] * B)
        n = [len(r[0]) for r in row]
        lab = torch.full((sum(n) + 64,), 0xAB, dtype=torch.uint8, device="cuda")
        offs = np.concatenate([[0], np.cumsum(n)[:-1]])
        ptrs = np.zeros((B, 3), np.uint64)
        ptrs[:, 0] = lab.data_ptr() + offs
        torch.cuda.synchronize()
        l0 = g.kernel_launches
        g.run_scans_to_device_ptrs(descs, [t.data_ptr() for t in dev], ptrs, 0, None, None)   # no dev_counts needed
        added = g.kernel_launches - l0
        t0 = twin.kernel_launches
        want = twin_run(twin, slots, row, dev, 0.0)[0]
        assert added == (twin.kernel_launches - t0) - 3 * B + g.n_streams, "labels only: one write pass per stream group"
        torch.cuda.synchronize()
        got = lab.cpu().numpy()
        for b in range(B):
            assert np.array_equal(got[offs[b]:offs[b] + n[b]], want[b]), f"step {k} scan {b}: labels"
        assert (got[sum(n):] == 0xAB).all()
        assert_state_equal(g, twin, slots, row, LIVE, f"step {k}")
    g.close()
    twin.close()


def test_edge_cases_empty_full_and_empty_selection():
    """An empty cloud, a cloud at capacity and a cloud with nothing selected; sentinel-filled buffers stay untouched
    past every count."""
    torch = torch_mod()
    dim, res = 99.0, 0.33
    scene = synth.make_scene(seed=77)
    full_pts, full_org = synth.lidar_scan(scene, beams=64, az_steps=1024, seed=77)
    cap = len(full_pts)
    far = np.zeros(3000, synth.POINT_DTYPE)          # far outside the map: every point absent, selection empty
    far["x"] = 5000.0
    far["z"] = np.linspace(-1, 1, len(far), dtype=np.float32)
    small_pts, small_org = synth.lidar_scan(scene, beams=32, az_steps=256, seed=78)
    clouds = [np.zeros(0, synth.POINT_DTYPE), full_pts, far, small_pts]
    origins = [full_org, full_org, full_org, small_org]
    B = len(clouds)
    g, twin = make_pair(dim, res, B, max_points=cap)
    slots = np.arange(B, dtype=np.int32)
    row = [(c, o, (0.0, 0.0), None) for c, o in zip(clouds, origins)]
    advance((g, twin), 0, row, slots)
    dev = [to_device(c) if len(c) else torch.empty((0, 8), dtype=torch.float32, device="cuda") for c in clouds]
    n = [len(c) for c in clouds]
    pad = 40
    for select, bits in (("nonground", capi.SELECT_NONGROUND), ("all", 3)):
        for h in (g, twin):
            for s in slots:
                h.init_map(0.0, 0.0, 0.0, slot=int(s))
        lab = [torch.full((m + pad,), 0xAB, dtype=torch.uint8, device="cuda") for m in n]
        idx = [torch.full((m + pad,), -7, dtype=torch.int32, device="cuda") for m in n]
        cld = [torch.full((m + pad, 8), -3.0, dtype=torch.float32, device="cuda") for m in n]
        counts = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        ptrs = np.array([[a.data_ptr(), b.data_ptr(), c.data_ptr()] for a, b, c in zip(lab, idx, cld)], np.uint64)
        descs = g.make_descs(list(slots), n, origins, [0.0] * B)
        torch.cuda.synchronize()
        g.run_scans_to_device_ptrs(descs, [t.data_ptr() for t in dev], ptrs, bits, counts.data_ptr(), None)
        want_labels, want_index, want_cloud = twin_run(twin, slots, row, dev, 0.0)
        torch.cuda.synchronize()
        got_counts = counts.cpu().numpy()
        for b in range(B):
            wi, wc = selected(want_labels[b], want_index[b], want_cloud[b], select)
            c = int(got_counts[b])
            assert c == len(wi), f"{select} scan {b}: count"
            L, I, Cl = lab[b].cpu().numpy(), idx[b].cpu().numpy(), cld[b].cpu().numpy()
            assert np.array_equal(L[:n[b]], want_labels[b]) and (L[n[b]:] == 0xAB).all(), f"{select} scan {b}: labels"
            assert np.array_equal(I[:c].view(np.uint32), wi) and (I[c:] == -7).all(), f"{select} scan {b}: index"
            assert Cl[:c].tobytes() == wc.tobytes() and (Cl[c:] == -3.0).all(), f"{select} scan {b}: cloud"
        assert got_counts[0] == 0 and got_counts[2] == 0 and n[1] == cap
        assert_state_equal(g, twin, slots, row, LIVE, select)
    g.close()
    twin.close()


@pytest.mark.parametrize("which", ["current", "side"])
def test_stream_order_without_host_waits(which):
    """(a) work already on the stream is waited for on the device, (b) work enqueued after the call sees the outputs,
    (c) inputs freed right after the call and their memory refilled on the stream do not race with the handle's reads.
    `current` runs on torch's current (legacy default) stream, `side` on a torch.cuda.Stream passed explicitly."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 4
    g, twin = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    steps = make_steps(B, 2, seed=5600)
    stream = torch.cuda.current_stream() if which == "current" else torch.cuda.Stream()
    if which == "current":
        assert stream.cuda_stream == 0     # NULL is the legacy default stream, not "unordered"
    # warm-up step: module loads, allocator pools
    row = steps[0]
    advance((g, twin), 0, row, slots)
    dev0 = [to_device(r[0]) for r in row]
    g.run_scans_to_device(dev0, slots, [r[1] for r in row], 0.0, select="all", stream=stream)
    twin_run(twin, slots, row, dev0, 0.0)
    torch.cuda.synchronize()
    row = steps[1]
    advance((g, twin), 1, row, slots)
    host = [torch.from_numpy(np.ascontiguousarray(r[0]).view(np.float32).reshape(-1, 8).copy()) for r in row]
    twin_dev = [h.cuda() for h in host]
    src = [t.clone() for t in twin_dev]
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        inputs = [torch.zeros_like(s) for s in src]
        torch.cuda._sleep(400_000_000)               # ~200 ms of device time ahead of the writes below
        for t, s in zip(inputs, src):
            t.copy_(s)
        before = torch.cuda.Event()
        before.record(stream)
        out = g.run_scans_to_device(inputs, slots, [r[1] for r in row], 0.0, labels=True, select="all", index=True, stream=stream)
        assert not before.query(), "the call waited on the host for the stream"
        clones = ([t.clone() for t in out.labels], [t.clone() for t in out.cloud], [t.clone() for t in out.index], out.counts.clone())
        sizes = [t.numel() for t in inputs]
        del inputs
        refill = [torch.full((m,), float("nan"), dtype=torch.float32, device="cuda") for m in sizes]
    pending = not before.query()
    want_labels, want_index, want_cloud = twin_run(twin, slots, row, twin_dev, 0.0)
    torch.cuda.synchronize()
    assert pending, "the sleep did not cover the call"
    check_outputs(out, "all", want_labels, want_index, want_cloud, f"{which}: outputs")
    labels_c, cloud_c, index_c, counts_c = clones
    cnt = counts_c.cpu().numpy()
    for k in range(B):
        assert np.array_equal(labels_c[k].cpu().numpy(), want_labels[k]), f"{which} scan {k}: cloned labels"
        assert cnt[k] == len(want_index[k]), f"{which} scan {k}: cloned count"
        assert np.array_equal(index_c[k][:cnt[k]].cpu().numpy().view(np.uint32), want_index[k]), f"{which} scan {k}: cloned index"
        assert records(cloud_c[k][:cnt[k]]).tobytes() == np.ascontiguousarray(want_cloud[k]).tobytes(), f"{which} scan {k}: cloned cloud"
    assert_layers_equal(g, twin, slots, LIVE, which)
    del refill
    g.close()
    twin.close()


def test_rejected_calls_enqueue_nothing_and_leave_the_handle_usable():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 4
    cap = 65536
    g, twin = make_pair(dim, res, B + 1, max_points=cap)       # slot B is never initialised
    slots = np.arange(B, dtype=np.int32)
    row = make_steps(B, 1, seed=5700)[0]
    advance((g, twin), 0, row, slots)
    dev = [to_device(r[0]) for r in row]
    n = [len(r[0]) for r in row]
    origins = [r[1] for r in row]
    big = torch.zeros((cap + 1, 8), dtype=torch.float32, device="cuda")
    lab = [torch.zeros(m, dtype=torch.uint8, device="cuda") for m in n]
    idx = [torch.zeros(m + 4, dtype=torch.int32, device="cuda") for m in n]
    cld = [torch.zeros((m + 1, 8), dtype=torch.float32, device="cuda") for m in n]
    counts = torch.zeros(B + 1, dtype=torch.int32, device="cuda")
    good_ptrs = np.array([[a.data_ptr(), b.data_ptr(), c.data_ptr()] for a, b, c in zip(lab, idx, cld)], np.uint64)
    good_in = [t.data_ptr() for t in dev]

    def call(slots_=slots, n_=n, ins=good_in, ptrs=good_ptrs, select=3, cnt=counts.data_ptr()):
        descs = g.make_descs(list(slots_), list(n_), origins, [0.0] * len(slots_))
        g.run_scans_to_device_ptrs(descs, ins, ptrs, select, cnt, None)

    def with_ptr(col, scan, value):
        p = good_ptrs.copy()
        p[scan, col] = value
        return p

    cases = {
        "repeated slot": dict(slots_=[0, 1, 1, 3]),
        "capacity exceeded": dict(n_=[n[0], cap + 1, n[2], n[3]], ins=[good_in[0], big.data_ptr(), good_in[2], good_in[3]]),
        "null cloud": dict(ins=[good_in[0], 0, good_in[2], good_in[3]]),
        "index with select 0": dict(ptrs=np.array([[0, p[1], 0] for p in good_ptrs], np.uint64), select=0),
        "cloud with select 0": dict(ptrs=np.array([[0, 0, p[2]] for p in good_ptrs], np.uint64), select=0),
        "unknown select bits": dict(select=7),
        "no dev_counts": dict(cnt=None),
        "misaligned index": dict(ptrs=with_ptr(1, 2, int(good_ptrs[2, 1]) + 2)),
        "misaligned cloud": dict(ptrs=with_ptr(2, 1, int(good_ptrs[1, 2]) + 8)),
        "labels overlap input": dict(ptrs=with_ptr(0, 3, good_in[3] + 32 * (n[3] - 1))),
        "index overlaps input": dict(ptrs=with_ptr(1, 0, good_in[0] - 4 * n[0] + 4)),
        "cloud is the input": dict(ptrs=with_ptr(2, 2, good_in[2])),
        "dev_counts in input": dict(cnt=good_in[0] + 64 * 32),
    }
    torch.cuda.synchronize()
    for name, kw in cases.items():
        l0 = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            call(**kw)
        assert e.value.code == -1, f"{name}: code {e.value.code}"
        assert g.kernel_launches == l0, f"{name}: something was launched"
    l0 = g.kernel_launches
    with pytest.raises(capi.GroundGridError) as e:
        call(slots_=[0, 1, 2, B], n_=n, ins=good_in)
    assert e.value.code == -3 and g.kernel_launches == l0, "map not initialised"
    torch.cuda.synchronize()
    # nothing was enqueued: the handle still holds the initial maps, and a correct call matches the twin
    call()
    want_labels, want_index, want_cloud = twin_run(twin, slots, row, dev, 0.0)
    torch.cuda.synchronize()
    got_counts = counts.cpu().numpy()
    for k in range(B):
        assert np.array_equal(lab[k].cpu().numpy(), want_labels[k])
        c = int(got_counts[k])
        assert c == len(want_index[k])
        assert np.array_equal(idx[k][:c].cpu().numpy().view(np.uint32), want_index[k])
        assert records(cld[k][:c]).tobytes() == np.ascontiguousarray(want_cloud[k]).tobytes()
    assert_state_equal(g, twin, slots, row, LIVE, "after the rejected calls")
    g.close()
    twin.close()

"""Batched evaluation tallies (gg_eval_counts_to_device): the per-slot confusion counts of many slots added into
caller-owned CUDA memory, ordered on the caller's stream.  Every tally is checked bit-exact against the same handle's
gg_eval_accumulate + gg_eval_read(reset=1), and for one slot per step against oracle/nextrows.py on the oracle's labels.
The ground truth travels in `ring`, as the KITTI player sends it."""
import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from oracle import Oracle, nextrows
from test_gpu_device_outputs import OTHER_CFGS, make_pair, torch_mod

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
KITTI_OFFSETS = (0, 4, 8, 12, 16)   # 18-byte records: x, y, z, intensity, label (scripts/kitti_data_publisher.py:117-150)


def label_steps(B, steps, seed):
    """[step][slot] -> (points with the SemanticKITTI id in `ring`, origin, ego xy, T, ego yaw).  A few points carry
    other ids, ids >= 1024 (dropped by the tallies) or are pushed below the ground (outliers)."""
    rng = np.random.default_rng(seed)
    scenes = [synth.make_scene(seed=seed + b, stream_len=10.0, undulation=0.2) for b in range(B)]
    out = []
    for k in range(steps):
        row = []
        for b in range(B):
            ex, ey, yaw = 0.8 * k + 0.05 * b, -0.35 * k * (b % 3), 0.04 * k * (1 + b % 2)
            pts, org, ids = synth.lidar_scan(scenes[b], ego_xy=(ex, ey), yaw=yaw, beams=64, az_steps=768, seed=seed + 100 * k + b,
                                             labels=True)
            idx = rng.choice(len(pts), len(pts) // 50, replace=False)
            ids[idx[: len(idx) // 2]] = rng.choice([0, 1, 44, 48, 52, 70, 71, 72, 80, 99, 252, 1023], len(idx) // 2)
            ids[idx[len(idx) // 2:]] = rng.choice([1024, 1025, 4096, 65535], len(idx) - len(idx) // 2)
            pts["ring"] = ids
            if k:
                down = rng.choice(len(pts), len(pts) // 200, replace=False)
                pts["z"][down] -= rng.uniform(0.3, 1.2, len(down)).astype(np.float32)
            row.append((pts, org, (ex, ey), synth.base_from_map(ex, ey, yaw, base_z=0.0, pitch=0.01), yaw))
        out.append(row)
    return out


def to_device(pts):
    torch = torch_mod()
    return torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).cuda()


def advance(g, k, row, slots):
    if k == 0:
        for b, r in enumerate(row):
            g.init_map(r[2][0], r[2][1], 0.0, slot=int(slots[b]))
    else:
        g.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))


def oracle_for(dim, res, slot, B):
    o = Oracle(dim, res)
    for s, kw in zip((1, B - 1), OTHER_CFGS):
        if slot == s:
            o.set_config(**kw)
    return o


def per_slot(g, slots):
    """The existing route: gg_eval_accumulate + gg_eval_read(reset=1), one slot at a time."""
    out = []
    for s in slots:
        g.eval_accumulate(int(s))
        out.append(g.eval_read(reset=True))
    return np.stack(out)


def batched(g, slots, **kw):
    torch = torch_mod()
    t = g.eval_counts_to_device(slots, **kw)
    assert t.dtype == torch.int64 and tuple(t.shape) == (len(slots), 1024, 2)
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("dim,res,B", [
    (99.0, 0.33, 4),      # N = 300, one slot per stream group
    (99.0, 0.33, 10),     # ten slots over the stream groups
    (33.33, 0.33, 10),    # N = 101
    (33.33, 0.33, 4),
])
def test_parity_over_a_rolling_stream(dim, res, B):
    """Permuted batches, every step of a rolling stream; slots 1 and B - 1 run their own configurations.  Slot 0 (the
    default configuration), 1 and B - 1 each follow an oracle with their own configuration."""
    g, _ = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    oracles = {s: oracle_for(dim, res, s, B) for s in (0, 1, B - 1)}
    rng = np.random.default_rng(8100 + B)
    steps = label_steps(B, 3, seed=8100 + B)
    for k, row in enumerate(steps):
        advance(g, k, row, slots)
        dev = [to_device(r[0]) for r in row]
        g.run_scans_to_device(dev, slots, [r[1] for r in row], 0.02 * k, labels=True, select=None)
        order = rng.permutation(B).astype(np.int32)
        got = batched(g, order)
        want = per_slot(g, order)
        assert np.array_equal(got, want), f"step {k}: batched != per-slot"
        for s, o in oracles.items():
            if k == 0:
                o.init_map(row[s][2][0], row[s][2][1], 0.0)
            else:
                o.update(row[s][2][0], row[s][2][1], row[s][3])
            lab_o, _, _ = o.filter_cloud(row[s][0], row[s][1], 0.02 * k, threads=1)
            k0 = int(np.flatnonzero(order == s)[0])
            assert np.array_equal(got[k0], nextrows.eval_counts(lab_o, row[s][0]["ring"])), f"step {k}: slot {s} != oracle"
            assert got[k0].sum() > 0
        sub = order[: max(1, B // 3)]
        assert np.array_equal(batched(g, sub), want[: len(sub)]), f"step {k}: subset"
    g.close()


def scan_inputs(g, route, row, slots, base_z):
    """Runs one scan per slot through `route`; returns what the caller must keep alive."""
    torch = torch_mod()
    B = len(slots)
    descs = g.make_descs([int(s) for s in slots], [len(r[0]) for r in row], [r[1] for r in row], [base_z] * B)
    if route == "filter_cloud":
        for s, r in zip(slots, row):
            g.filter_cloud(r[0], r[1], base_z, slot=int(s))
        return None
    if route in ("batch_packed", "batch_plain"):
        hp = [torch.from_numpy(np.ascontiguousarray(r[0]).view(np.uint8).copy()).pin_memory() for r in row]
        hl = [torch.zeros(len(r[0]), dtype=torch.uint8).pin_memory() for r in row]
        g.filter_cloud_batch_ptrs(descs, [t.data_ptr() for t in hp], [t.data_ptr() for t in hl])
        return hp, hl
    dev = [to_device(r[0]) for r in row]
    torch.cuda.synchronize()
    if route == "run_scans_device":
        g.run_scans_device(descs, [t.data_ptr() for t in dev])
    else:
        g.run_scans_to_device(dev, slots, [r[1] for r in row], base_z, labels=True, select="all")
    return dev


@pytest.mark.parametrize("route", ["filter_cloud", "batch_packed", "batch_plain", "run_scans_device", "run_scans_to_device"])
def test_every_input_route(monkeypatch, route):
    if route.startswith("batch"):
        monkeypatch.setenv("GG_HOST_PACK", "1" if route == "batch_packed" else "0")
        monkeypatch.setenv("GG_HOST_THREADS", "2")
    dim, res, B = 99.0, 0.33, 6
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536)
    o = Oracle(dim, res)
    slots = np.arange(B, dtype=np.int32)
    steps = label_steps(B, 2, seed=8200)
    for k, row in enumerate(steps):
        advance(g, k, row, slots)
        if k == 0:
            o.init_map(row[2][2][0], row[2][2][1], 0.0)
        else:
            o.update(row[2][2][0], row[2][2][1], row[2][3])
        keep = scan_inputs(g, route, row, slots, 0.02 * k)
        if route == "batch_packed":
            assert g.last_batch_transfer()[0] == B, "every scan was packed"
        if route == "batch_plain":
            assert g.last_batch_transfer()[1] == B, "every scan went as 32-byte records"
        lab_o, _, _ = o.filter_cloud(row[2][0], row[2][1], 0.02 * k, threads=1)
        order = slots[::-1].copy()
        got = batched(g, order)
        assert np.array_equal(got, per_slot(g, order)), f"{route} step {k}"
        assert np.array_equal(got[B - 1 - 2], nextrows.eval_counts(lab_o, row[2][0]["ring"])), f"{route} step {k}: oracle"
        del keep
    g.close()


def kitti_payload(pts_frame, ids):
    """18-byte records with the label at offset 16."""
    n = len(pts_frame)
    raw = np.zeros((n, 18), np.uint8)
    for name, off in (("x", 0), ("y", 4), ("z", 8), ("intensity", 12)):
        raw[:, off:off + 4] = np.ascontiguousarray(pts_frame[name]).view(np.uint8).reshape(n, 4)
    raw[:, 16:18] = np.ascontiguousarray(ids, np.uint16).view(np.uint8).reshape(n, 2)
    return raw


def test_cloud_msgs_ground_truth_survives_the_payload():
    """gg_run_cloud_msgs_to_device on 18-byte KITTI payloads, sensor-frame and map-frame mixed, each payload freed right
    after the call and its memory refilled: the tallies read the labels from the slot's own buffer."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 5
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536)
    o = Oracle(dim, res)
    slots = np.arange(B, dtype=np.int32)[::-1].copy()
    scenes = [synth.make_scene(seed=8300 + b, stream_len=10.0) for b in range(B)]
    for k in range(2):
        payloads, T, origins, clouds = [], [], [], []
        for b in range(B):
            ego, yaw = (0.8 * k + 0.1 * b, 0.2 * b), 0.05 * k * b
            sensor = b % 2 == 0
            pts, org, ids = synth.lidar_scan(scenes[b], ego_xy=ego, yaw=yaw, beams=64, az_steps=512, seed=8300 + 10 * k + b,
                                             frame="base" if sensor else "map", labels=True)
            if sensor:
                c, s = np.cos(yaw), np.sin(yaw)
                Tm = np.array([[c, -s, 0.0, ego[0]], [s, c, 0.0, ego[1]], [0.0, 0.0, 1.0, 0.0]], np.float64)
            else:
                Tm = None
            raw = kitti_payload(pts, ids)
            payloads.append(torch.from_numpy(raw.reshape(-1).copy()).cuda())
            T.append(Tm)
            origins.append(org)
            clouds.append(nextrows.unpack_transform(raw, len(pts), 18, KITTI_OFFSETS, Tm))
            if k == 0:
                g.init_map(ego[0], ego[1], 0.0, slot=int(slots[b]))
            else:
                g.update_pose(ego[0], ego[1], synth.base_from_map(ego[0], ego[1], yaw), slot=int(slots[b]))
            if b == 2:   # a sensor-frame payload
                if k == 0:
                    o.init_map(ego[0], ego[1], 0.0)
                else:
                    o.update(ego[0], ego[1], synth.base_from_map(ego[0], ego[1], yaw))
        torch.cuda.synchronize()
        sizes = [p.numel() for p in payloads]
        g.run_cloud_msgs_to_device(payloads, 18, KITTI_OFFSETS, T, slots, origins, 0.0, labels=True, select=None)
        del payloads
        refill = [torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda") for n in sizes]
        got = batched(g, slots)
        assert all(bool((r == 0xEE).all()) for r in refill)
        assert np.array_equal(got, per_slot(g, slots)), f"step {k}"
        lab_o, _, _ = o.filter_cloud(clouds[2], origins[2], 0.0, threads=1)
        assert np.array_equal(got[2], nextrows.eval_counts(lab_o, clouds[2]["ring"])), f"step {k}: oracle"
        assert got[2].sum() > 0
    g.close()


def test_semantics_add_drop_and_empty():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 3
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536)
    scene = synth.make_scene(seed=8400, n_boxes=8, rmin=4.0, rmax=14.0)
    pts, org, ids = synth.lidar_scan(scene, beams=32, az_steps=512, seed=8400, labels=True)
    n = len(pts)
    pts["ring"] = ids
    big = pts.copy()
    big["ring"][::7] = 1024 + np.arange(len(big[::7]), dtype=np.uint16) % 3000
    big["x"][::11] += np.float32(500.0)    # outside the map: absent (label 0)
    for s in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=s)
    g.filter_cloud(pts, org, 0.0, slot=0)
    lab_big = g.filter_cloud(big, org, 0.0, slot=1)
    g.filter_cloud(np.zeros(0, synth.POINT_DTYPE), org, 0.0, slot=2)   # an empty cloud
    g.synchronize()
    lab0 = g.download_labels(n, slot=0)
    g.synchronize()
    once = per_slot(g, [0, 1, 2])
    # the sum over ids is the number of labelled points; ids >= 1024 and absent points are not counted
    assert once[0].sum() == (lab0 != 0).sum() and (lab0 != 0).sum() > 0
    assert (lab_big[::11] == 0).all() and (big["ring"][lab_big != 0] >= 1024).sum() > 0
    assert once[1].sum() == ((lab_big != 0) & (big["ring"] < 1024)).sum()
    assert np.array_equal(once[1], nextrows.eval_counts(lab_big, big["ring"]))
    assert (once[2] == 0).all()
    # adds into a non-zero start; two calls double the tallies
    start = torch.full((3, 1024, 2), 5, dtype=torch.int64, device="cuda")
    out = g.eval_counts_to_device([0, 1, 2], out=start)
    assert out is start
    torch.cuda.synchronize()
    assert np.array_equal(start.cpu().numpy().view(np.uint64), once + 5)
    g.eval_counts_to_device([0, 1, 2], out=start)
    torch.cuda.synchronize()
    assert np.array_equal(start.cpu().numpy().view(np.uint64), 2 * once + 5)
    g.close()


@pytest.mark.parametrize("which", ["current", "side"])
def test_stream_order_without_host_waits(which):
    """(a) the call returns while the stream is still busy, (b) it sees the scans enqueued right before it, (c) a clone
    enqueued right after it sees the tallies, (d) the slot's next scan enqueued right after it does not change them."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 4
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536)
    slots = np.arange(B, dtype=np.int32)
    steps = label_steps(B, 3, seed=8500)
    stream = torch.cuda.current_stream() if which == "current" else torch.cuda.Stream()
    if which == "current":
        assert stream.cuda_stream == 0
    for b, r in enumerate(steps[0]):
        g.init_map(r[2][0], r[2][1], 0.0, slot=b)
    dev = [[to_device(r[0]) for r in row] for row in steps]
    torch.cuda.synchronize()
    # warm-up: module loads, allocator pools
    with torch.cuda.stream(stream):
        g.run_scans_to_device(dev[0], slots, [r[1] for r in steps[0]], 0.0, labels=True, select=None, stream=stream)
        g.eval_counts_to_device(slots, stream=stream)
    torch.cuda.synchronize()
    before = torch.cuda.Event()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(400_000_000)               # ~200 ms of device time ahead of everything below
        before.record(stream)
        out1 = g.run_scans_to_device(dev[1], slots, [r[1] for r in steps[1]], 0.0, labels=True, select=None, stream=stream)
        tally = g.eval_counts_to_device(slots, stream=stream)
        assert not before.query(), "gg_eval_counts_to_device waited on the host for the stream"
        clone = tally.clone()
        out2 = g.run_scans_to_device(dev[2], slots, [r[1] for r in steps[2]], 0.0, labels=True, select=None, stream=stream)
        assert not before.query(), "the next scan waited on the host"
    pending = not before.query()
    torch.cuda.synchronize()
    assert pending, "the sleep did not cover the calls"
    want = np.stack([nextrows.eval_counts(out1.labels[b].cpu().numpy(), steps[1][b][0]["ring"]) for b in range(B)])
    assert not np.array_equal(want, np.stack([nextrows.eval_counts(out2.labels[b].cpu().numpy(), steps[2][b][0]["ring"])
                                              for b in range(B)]))
    assert np.array_equal(tally.cpu().numpy().view(np.uint64), want), f"{which}: tallies of the scans before the call"
    assert np.array_equal(clone.cpu().numpy().view(np.uint64), want), f"{which}: clone"
    g.close()


def test_rejected_calls_enqueue_nothing():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 6
    g = capi.GroundGridB200(dim, res, n_slots=B + 1, max_points=65536)   # slot B is never initialised
    steps = label_steps(B, 2, seed=8600)
    row = steps[0]
    for b, r in enumerate(row):
        g.init_map(r[2][0], r[2][1], 0.0, slot=b)
    dev = [to_device(r[0]) for r in row]
    torch.cuda.synchronize()
    full = [0, 1, 2, 3]
    descs = g.make_descs(full, [len(row[b][0]) for b in full], [row[b][1] for b in full], [0.0] * 4)
    g.run_scans_device(descs, [dev[b].data_ptr() for b in full])
    d4 = g.make_descs([4], [len(row[4][0])], [row[4][1]], [0.0])
    g.run_scans_device(d4, [dev[4].data_ptr()], stop_after=1)     # slot 4: the last scan stopped early
    g.update_pose_batch(np.array([5], np.int32), np.array([steps[1][5][2]]), steps[1][5][3].reshape(1, 12))   # slot 5: rolled only
    g.synchronize()
    buf = torch.full((B + 2, 1024, 2), 0x3C3C, dtype=torch.int64, device="cuda")
    P = buf.data_ptr()
    arena = g.layer_device_ptr("ground", slot=0)
    sl = np.ascontiguousarray([0, 1], np.int32)

    def call(slots_=(0, 1), d=P):
        g.eval_counts_to_device_ptrs(list(slots_), d, None)

    def raw(h, count, slots_ptr, d):
        rc = g._l.gg_eval_counts_to_device(h, count, slots_ptr, d, None)
        if rc != 0:
            raise capi.GroundGridError(rc, g._l.gg_last_error().decode())

    cases = {
        "null handle": (ARG, lambda: raw(None, 2, sl.ctypes.data, P)),
        "null slots": (ARG, lambda: raw(g._h, 2, None, P)),
        "null dev_counts": (ARG, lambda: raw(g._h, 2, sl.ctypes.data, None)),
        "negative count": (ARG, lambda: raw(g._h, -1, sl.ctypes.data, P)),
        "misaligned dev_counts": (ARG, lambda: call(d=P + 4)),
        "dev_counts in the arena": (ARG, lambda: call(d=arena)),
        "dev_counts ends in the arena": (ARG, lambda: call(d=arena - 2 * 1024 * 2 * 8 + 8)),
        "count exceeds slots": (ARG, lambda: call(list(range(B + 1)) + [0])),
        "slot out of range": (ARG, lambda: call([0, B + 1])),
        "negative slot": (ARG, lambda: call([0, -1])),
        "repeated slot": (ARG, lambda: call([0, 2, 2])),
        "map not initialised": (STATE, lambda: call([0, B])),
        "stopped early": (STATE, lambda: call([0, 4])),
        "rolled only since gg_init_map": (STATE, lambda: call([1, 5])),
    }
    for name, (code, fn) in cases.items():
        l0 = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            fn()
        assert e.value.code == code, f"{name}: code {e.value.code}"
        assert g.kernel_launches == l0, f"{name}: something was launched"
    for s in (4, 5):
        with pytest.raises(capi.GroundGridError) as e:
            g.eval_accumulate(s)
        assert e.value.code == STATE
    l0 = g.kernel_launches
    call([])                                   # an empty batch is accepted and enqueues nothing
    raw(g._h, 0, None, None)
    assert g.kernel_launches == l0
    torch.cuda.synchronize()
    assert (buf == 0x3C3C).all(), "a rejected call wrote into the buffer"
    # the handle is still usable
    got = batched(g, full)
    assert np.array_equal(got, per_slot(g, full))
    g.close()

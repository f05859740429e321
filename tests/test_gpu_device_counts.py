"""Point counts from caller GPU memory (gg_set_point_counts_from_device + GG_SCAN_DEVICE_COUNT): scans whose size only
the device knows.  Every case runs against a twin handle that makes the same scans with the host count u on the same
first u records, and must be bit-identical to it: labels, index, cloud, dev_counts, layers, gg_get_output, point-info
codes and heights, evaluation tallies and gg_last_scan_points.  The records past u of the caller's cloud or payload
are poison: in-map points well above the terrain whose rings the tallies count, so a read past the count shows."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from oracle import Oracle
from test_gpu_cloud_msgs import cuda_bytes, map_from_sensor, payload
from test_gpu_device_outputs import LIVE, make_pair, to_device, torch_mod
from test_gpu_device_poses import device_poses, pose_steps

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
INT32_MIN, INT32_MAX = -(2 ** 31), 2 ** 31 - 1
MAX_POINTS = 40000
MSG32 = (32, (0, 4, 8, 16, 20))   # PointXYZIR records as a PointCloud2 payload in the map frame
MSG18 = (18, (0, 4, 8, 12, 16))   # the KITTI player's 18-byte points, in a sensor frame


def poison(pts, n, rng):
    """n in-map records 4-12 m above the scan's points, rings the tallies count (ids < 64 < max_ring)."""
    out = np.zeros(n, synth.POINT_DTYPE)
    if n == 0:
        return out
    k = rng.integers(0, len(pts), n)
    out["x"] = pts["x"][k] + rng.uniform(-0.2, 0.2, n).astype(np.float32)
    out["y"] = pts["y"][k] + rng.uniform(-0.2, 0.2, n).astype(np.float32)
    out["z"] = pts["z"][k] + rng.uniform(4.0, 12.0, n).astype(np.float32)
    out["intensity"] = 7.0
    out["ring"] = rng.integers(0, 64, n).astype(np.uint16)
    return out


def with_poison(pts, u, cap, rng):
    """The first u records of pts, then cap - u poison records."""
    out = np.zeros(cap, synth.POINT_DTYPE)   # not np.concatenate: it would drop the record's padding
    out[:u] = pts[:u]
    out[u:] = poison(pts, cap - u, rng)
    return out


def kinds(B, n):
    """(u, capacity) per slot: u == capacity, u < capacity, u == 0, capacity = max_points, then repeating."""
    out = []
    for b in range(B):
        m = n[b]
        out.append([(m, m), (m * 2 // 3, m), (0, m // 2 + 1), (m - 17, MAX_POINTS)][b % 4])
    return out


def point_info(h, slots, caps, torch):
    """codes and heights of each slot's last scan into capacity-sized buffers (the raw call: no host wait)."""
    codes = [torch.full((max(c, 1),), -7, dtype=torch.int32, device="cuda") for c in caps]
    height = [torch.full((max(c, 1),), -7.0, dtype=torch.float32, device="cuda") for c in caps]
    h.point_info_to_device_ptrs(slots, [t.data_ptr() for t in codes], [t.data_ptr() for t in height], torch.cuda.current_stream().cuda_stream or None)
    return codes, height


def assert_twin(g, twin, slots, us, caps, ctx, complete=True, names=LIVE):
    """Layers, last_scan_points, point classes, and (complete scans) labels, get_output, point info and tallies."""
    torch = torch_mod()
    slots = [int(s) for s in slots]
    for s, u in zip(slots, us):
        for name in names:
            assert np.array_equal(g.layer(name, slot=s).view(np.uint32), twin.layer(name, slot=s).view(np.uint32)), f"{ctx} slot {s}: {name}"
    if complete:
        gc, gh = point_info(g, slots, caps, torch)
        tc, th = twin.point_info_to_device(slots)
        gt = g.eval_counts_to_device(slots)
        tt = twin.eval_counts_to_device(slots)
        torch.cuda.synchronize()
        assert torch.equal(gt, tt), f"{ctx}: tallies"
        for j, (s, u, c) in enumerate(zip(slots, us, caps)):
            assert torch.equal(gc[j][:u], tc[j]) and torch.equal(gh[j][:u].view(torch.int32), th[j].view(torch.int32)), f"{ctx} slot {s}: point info"
            assert bool((gc[j][u:] == -7).all()) and bool((gh[j][u:] == -7.0).all()), f"{ctx} slot {s}: point info past u"
        for s, u in zip(slots, us):
            gi, gcl = g.get_output(slot=s, want_cloud=True)
            ti, tcl = twin.get_output(slot=s, want_cloud=True)
            assert np.array_equal(gi, ti) and gcl.tobytes() == tcl.tobytes(), f"{ctx} slot {s}: get_output"
            assert np.array_equal(g.download_labels(u, slot=s), twin.download_labels(u, slot=s)), f"{ctx} slot {s}: labels"
    for s, u in zip(slots, us):
        assert g.last_scan_points(slot=s) == u == twin.last_scan_points(slot=s), f"{ctx} slot {s}: last_scan_points"
        if u:
            assert np.array_equal(g.point_classes(u, slot=s), twin.point_classes(u, slot=s)), f"{ctx} slot {s}: point classes"
    g.synchronize()
    twin.synchronize()


def check_device_outputs(out_g, out_t, us, ctx):
    torch = torch_mod()
    torch.cuda.synchronize()
    assert torch.equal(out_g.counts, out_t.counts), f"{ctx}: dev_counts"
    gc, gi = out_g.trimmed()
    tc, ti = out_t.trimmed()
    for k, u in enumerate(us):
        assert torch.equal(out_g.labels[k][:u], out_t.labels[k]), f"{ctx} scan {k}: labels"
        assert torch.equal(gc[k], tc[k]) and torch.equal(gi[k], ti[k]), f"{ctx} scan {k}: cloud / index"


def set_counts(g, slots, us, stream=None):
    torch = torch_mod()
    g.set_point_counts_from_device(slots, torch.tensor(np.asarray(us, np.int64), device="cuda"), stream=stream)


ROUTES = ["device0", "device1", "device2", "device3", "to_device", "msgs32", "msgs18"]


@pytest.mark.parametrize("route", ROUTES)
def test_parity_on_every_honoured_route(route):
    """Three steps with rolls; per batch every capacity kind (u == capacity, u < capacity, u == 0, capacity =
    max_points); stop_after 0-3 on gg_run_scans_device."""
    torch = torch_mod()
    B = 8
    g, twin = make_pair(99.0, 0.33, B, max_points=MAX_POINTS)
    rng = np.random.default_rng(ROUTES.index(route))
    steps = pose_steps(B, 3, jump=0.0, seed=5100)
    slots = np.arange(B, dtype=np.int32)[::-1].copy()
    stop = int(route[-1]) if route.startswith("device") else 0
    for k, full in enumerate(steps):
        row = [full[s] for s in slots]
        for h in (g, twin):
            if k == 0:
                for s, r in zip(slots, row):
                    h.init_map(r[2][0], r[2][1], 0.0, slot=int(s))
            else:
                h.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))
        uc = kinds(B, [len(r[0]) for r in row])
        us, caps = [u for u, _ in uc], [c for _, c in uc]
        set_counts(g, slots, us)
        clouds = [with_poison(r[0], u, c, rng) for r, (u, c) in zip(row, uc)]
        origins, bz = [r[1] for r in row], [r[4] for r in row]
        ctx = f"{route} step {k}"
        if route.startswith("device"):
            dev_g = [to_device(c) for c in clouds]
            dev_t = [to_device(r[0][:u]) for r, u in zip(row, us)]
            g.run_scans_device(g.make_descs(slots, caps, origins, bz), [t.data_ptr() for t in dev_g], stop_after=stop, device_counts=True)
            twin.run_scans_device(twin.make_descs(slots, us, origins, bz), [t.data_ptr() if u else 0 for t, u in zip(dev_t, us)], stop_after=stop)
            assert_twin(g, twin, slots, us, caps, ctx, complete=stop == 0)
            del dev_g, dev_t
        elif route == "to_device":
            dev_g = [to_device(c) for c in clouds]
            dev_t = [to_device(r[0][:u]) for r, u in zip(row, us)]
            og = g.run_scans_to_device(dev_g, slots, origins, bz, labels=True, select="nonground", index=True, device_counts=True)
            ot = twin.run_scans_to_device(dev_t, slots, origins, bz, labels=True, select="nonground", index=True)
            check_device_outputs(og, ot, us, ctx)
            assert_twin(g, twin, slots, us, caps, ctx)
        else:
            step, offs = MSG32 if route == "msgs32" else MSG18
            Ts = [None if route == "msgs32" else map_from_sensor(r[2], 0.2 * b + 0.1 * k) for b, r in enumerate(row)]
            raw = [payload(c, step, offs, T, rng) for c, T in zip(clouds, Ts)]
            dev_g = [cuda_bytes(x) for x in raw]
            dev_t = [cuda_bytes(x[:u]) for x, u in zip(raw, us)]
            T = Ts if route == "msgs18" else None
            og = g.run_cloud_msgs_to_device(dev_g, step, offs, T, slots, origins, bz, labels=True, select="all", index=True, device_counts=True)
            ot = twin.run_cloud_msgs_to_device(dev_t, step, offs, T, slots, origins, bz, labels=True, select="all", index=True)
            check_device_outputs(og, ot, us, ctx)
            assert_twin(g, twin, slots, us, caps, ctx)


def test_rolling_stream_with_device_poses_and_mixed_flags():
    """24 steps on ten slots over the stream groups: counts vary every step, rolls and scan poses come from the device,
    and every batch mixes flagged and host-count scans.  The twin runs host poses and host counts; slot 0 is also
    checked against the CPU oracle on the truncated clouds."""
    torch = torch_mod()
    B, STEPS = 10, 24
    g, twin = make_pair(99.0, 0.33, B, max_points=MAX_POINTS)
    o = Oracle(99.0, 0.33)
    rng = np.random.default_rng(77)
    steps = pose_steps(B, STEPS, jump=60.0, seed=5200)
    oracle_checked = 0
    for k, full in enumerate(steps):
        slots = rng.permutation(B).astype(np.int32)
        row = [full[s] for s in slots]
        xy, T, origins, bz = device_poses(row, torch)
        i0 = int(np.nonzero(slots == 0)[0][0])
        if k == 0:
            for s, r in zip(slots, row):
                g.init_map(r[2][0], r[2][1], 0.0, slot=int(s))
                twin.init_map(r[2][0], r[2][1], 0.0, slot=int(s))
            o.init_map(row[i0][2][0], row[i0][2][1], 0.0)
            g.update_poses_from_device(slots, origins=origins, base_z=bz)
        else:
            g.update_poses_from_device(slots, xy, T, origins, bz)
            twin.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))
            o.update(row[i0][2][0], row[i0][2][1], row[i0][3])
        n = [len(r[0]) for r in row]
        us = [int(rng.integers(0, m + 1)) if rng.random() < 0.9 else m for m in n]
        flagged = rng.random(B) < 0.6
        flagged[i0] = True
        us[i0] = max(us[i0], 1)
        caps = [n[j] if flagged[j] else us[j] for j in range(B)]
        set_counts(g, slots[flagged], [u for u, f in zip(us, flagged) if f])
        clouds = [with_poison(r[0], u, c, rng) for r, u, c in zip(row, us, caps)]
        dev_g = [to_device(c) for c in clouds]
        dev_t = [to_device(r[0][:u]) for r, u in zip(row, us)]
        descs = g._device_descs(slots, caps, "device", None)
        descs["flags"][flagged] |= capi.SCAN_DEVICE_COUNT
        og, ptrs = g._device_outputs(torch, torch.device("cuda", 0), torch.cuda.current_stream(), caps, True, capi.SELECT["all"], True, [])
        g.run_scans_to_device_ptrs(descs, [t.data_ptr() for t in dev_g], ptrs, capi.SELECT["all"], og.counts.data_ptr(), None)
        ot = twin.run_scans_to_device(dev_t, slots, [r[1] for r in row], [r[4] for r in row], labels=True, select="all", index=True)
        check_device_outputs(og, ot, us, f"step {k}")
        if k % 6 == 5 or k == STEPS - 1:
            assert_twin(g, twin, slots, us, caps, f"step {k}")
        if k in (3, 11, STEPS - 1):
            r = row[i0]
            ref, _, _ = o.filter_cloud(r[0][:us[i0]], r[1], r[4], threads=1)
            torch.cuda.synchronize()
            assert np.array_equal(og.labels[i0][:us[i0]].cpu().numpy(), ref), f"step {k}: labels differ from the oracle"
            for name in ("ground", "groundpatch"):
                assert np.array_equal(g.layer(name, slot=0).view(np.uint32), o.layer(name).view(np.uint32)), f"step {k}: {name} vs oracle"
            oracle_checked += 1
        else:
            o.filter_cloud(row[i0][0][:us[i0]], row[i0][1], row[i0][4], threads=1)
        del xy, T, origins, bz
    assert oracle_checked == 3


@pytest.mark.parametrize("bad", [-1, INT32_MIN, "cap+1", INT32_MAX])
def test_invalid_counts_run_the_scan_empty(bad):
    """A stored count outside [0, capacity] is identical to an empty host scan: layers, dev_counts 0, get_output empty
    and gg_last_scan_points 0; nothing past the capacity is read."""
    torch = torch_mod()
    B = 3
    g, twin = make_pair(99.0, 0.33, B, max_points=MAX_POINTS)
    steps = pose_steps(B, 2, jump=0.0, seed=5300)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(3)
    for h in (g, twin):
        for s, r in zip(slots, steps[0]):
            h.init_map(r[2][0], r[2][1], 0.0, slot=int(s))
    for k, row in enumerate(steps):   # a full scan first, so the empty one runs on a populated map
        caps = [len(r[0]) for r in row]
        us = caps if k == 0 else [0] * B
        vals = caps if k == 0 else [(c + 1 if bad == "cap+1" else bad) for c in caps]
        set_counts(g, slots, vals)
        dev_g = [to_device(with_poison(r[0], c, c, rng)) for r, c in zip(row, caps)]
        dev_t = [to_device(r[0][:u]) for r, u in zip(row, us)]
        og = g.run_scans_to_device(dev_g, slots, [r[1] for r in row], [r[4] for r in row], labels=True, select="all", index=True,
                                   device_counts=True)
        ot = twin.run_scans_to_device(dev_t, slots, [r[1] for r in row], [r[4] for r in row], labels=True, select="all", index=True)
        check_device_outputs(og, ot, us, f"{bad} step {k}")
        assert_twin(g, twin, slots, us, caps, f"{bad} step {k}")
    assert og.counts.cpu().tolist() == [0] * B


def test_stream_contract():
    """Counts made by a torch op on a side stream passed as `stream`; the count tensor overwritten on that stream right
    after the call (the scan uses the earlier value); two set calls before one scan (the second wins); two flagged scans
    after one set (both use it)."""
    torch = torch_mod()
    B = 4
    g, twin = make_pair(99.0, 0.33, B, max_points=MAX_POINTS)
    steps = pose_steps(B, 4, jump=0.0, seed=5400)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(4)
    for h in (g, twin):
        for s, r in zip(slots, steps[0]):
            h.init_map(r[2][0], r[2][1], 0.0, slot=int(s))
    side = torch.cuda.Stream()
    for k, row in enumerate(steps):
        caps = [len(r[0]) for r in row]
        us = [c * (3 + b + k) // 9 for b, c in enumerate(caps)]
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)          # the counts are late: only stream order makes them visible
            base = torch.tensor(np.asarray(us, np.int32), device="cuda")
            counts = (base * 2 + 6) // 2 - 3       # computed on the side stream
        if k == 1:
            g.set_point_counts_from_device(slots, torch.zeros(B, dtype=torch.int32, device="cuda"), stream=side)   # overridden
        if k != 3:   # step 3 reuses step 2's counts
            g.set_point_counts_from_device(slots, counts, stream=side)
            with torch.cuda.stream(side):
                counts.fill_(INT32_MAX)            # overwritten right after the call
        else:
            us = prev_us
        dev_g = [to_device(with_poison(r[0], u, c, rng)) for r, u, c in zip(row, us, caps)]
        dev_t = [to_device(r[0][:u]) for r, u in zip(row, us)]
        og = g.run_scans_to_device(dev_g, slots, [r[1] for r in row], [r[4] for r in row], labels=True, select="nonground", index=True,
                                   stream=side, device_counts=True)
        ot = twin.run_scans_to_device(dev_t, slots, [r[1] for r in row], [r[4] for r in row], labels=True, select="nonground", index=True)
        side.synchronize()
        check_device_outputs(og, ot, us, f"step {k}")
        assert_twin(g, twin, slots, us, caps, f"step {k}")
        prev_us = us


def test_ownership_of_the_last_count():
    """After a flagged scan the count is the device's: point info, tallies (batched and per slot) and get_output use it
    without a host wait, gg_last_scan_points / gg_get_point_classes wait and return it.  A host-count scan or gg_init_map
    ends device ownership; gg_init_map also forgets the stored count."""
    torch = torch_mod()
    B = 2
    g, twin = make_pair(99.0, 0.33, B, max_points=MAX_POINTS)
    steps = pose_steps(B, 3, jump=0.0, seed=5500)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(5)
    for h in (g, twin):
        for s, r in zip(slots, steps[0]):
            h.init_map(r[2][0], r[2][1], 0.0, slot=int(s))
    row = steps[0]
    caps = [len(r[0]) for r in row]
    us = [c // 2 for c in caps]
    set_counts(g, slots, us)
    dev_g = [to_device(with_poison(r[0], u, c, rng)) for r, u, c in zip(row, us, caps)]
    dev_t = [to_device(r[0][:u]) for r, u in zip(row, us)]
    g.run_scans_to_device(dev_g, slots, [r[1] for r in row], [r[4] for r in row], labels=True, select=None, device_counts=True)
    twin.run_scans_to_device(dev_t, slots, [r[1] for r in row], [r[4] for r in row], labels=True, select=None)
    # no host wait: the calls return while the caller's stream is still busy (their staging is allocated first)
    g.point_info_to_device(slots[:1], height=False)
    g.eval_accumulate(slot=0)
    g.eval_read(reset=True)
    busy = torch.cuda.Stream()
    with torch.cuda.stream(busy):
        torch.cuda._sleep(200_000_000)
        codes = [torch.full((c,), -7, dtype=torch.int32, device="cuda") for c in caps]
        tallies = torch.zeros((B, 1024, 2), dtype=torch.int64, device="cuda")
    g.point_info_to_device_ptrs(slots, [t.data_ptr() for t in codes], None, busy.cuda_stream)
    g.eval_counts_to_device_ptrs(slots, tallies.data_ptr(), busy.cuda_stream)
    g.eval_accumulate(slot=0)
    assert not busy.query(), "a device-count call waited for the caller's stream"
    busy.synchronize()
    tc, _ = twin.point_info_to_device(slots, height=False)
    tt = twin.eval_counts_to_device(slots)
    twin.eval_accumulate(slot=0)
    torch.cuda.synchronize()
    assert torch.equal(tallies, tt)
    for j, u in enumerate(us):
        assert torch.equal(codes[j][:u], tc[j]) and bool((codes[j][u:] == -7).all())
    assert np.array_equal(g.eval_read(reset=True), twin.eval_read(reset=True))
    assert_twin(g, twin, slots, us, caps, "device-owned")
    # a host-count scan of slot 0 ends device ownership
    row = steps[1]
    n0 = len(row[0][0])
    host_clouds = [to_device(row[0][0]) for _ in range(2)]   # the tallies read them later
    for h, c in zip((g, twin), host_clouds):
        h.run_scans_device(h.make_descs([0], [n0], [row[0][1]], [row[0][4]]), [c.data_ptr()])
        h.synchronize()
    assert g.last_scan_points(slot=0) == n0 == twin.last_scan_points(slot=0)
    assert_twin(g, twin, [0], [n0], [n0], "host count again")
    # gg_init_map forgets the stored count: a flagged scan is then GG_E_STATE, with nothing enqueued
    g.init_map(0.0, 0.0, 0.0, slot=1)
    assert g.last_scan_points(slot=1) == 0
    before = g.kernel_launches
    d = g.make_descs([1], [caps[1]], [row[1][1]], [row[1][4]])
    with pytest.raises(capi.GroundGridError) as e:
        g.run_scans_device(d, [dev_g[1].data_ptr()], device_counts=True)
    assert e.value.code == STATE and g.kernel_launches == before


def test_rejections_enqueue_nothing():
    """GG_SCAN_DEVICE_COUNT on the calls whose counts are on the host is GG_E_ARG; every GG_E_ARG / GG_E_STATE case of
    gg_set_point_counts_from_device; count == 0 is GG_OK.  None enqueues anything."""
    torch = torch_mod()
    B = 3
    g = capi.GroundGridB200(99.0, 0.33, n_slots=B, max_points=MAX_POINTS)
    L = g._l
    for s in range(B - 1):
        g.init_map(0.0, 0.0, 0.0, slot=s)
    pts, org = synth.lidar_scan(synth.make_scene(seed=9), ego_xy=(0.0, 0.0), beams=32, az_steps=256, seed=9)
    counts = torch.tensor([len(pts)] * B, dtype=torch.int32, device="cuda")
    g.set_point_counts_from_device([0, 1], counts[:2])
    g.synchronize()
    before = g.kernel_launches

    def desc(slot=0):
        d = g.make_descs([slot], [len(pts)], [org], [0.0])
        d[0].flags = capi.SCAN_DEVICE_COUNT
        return d

    keep = g.upload_points(pts, slot=0)
    g.synchronize()
    before = g.kernel_launches
    hp = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).pin_memory()
    dev = cuda_bytes(np.ascontiguousarray(pts).view(np.uint8))
    n_parts_, parts_, Tarr = capi.cloud_parts([[dev.numel()]], [[dev.data_ptr()]], 32, MSG32[1], None)
    ticket = C.c_int(-1)
    pp = (C.c_void_p * 1)(hp.data_ptr())
    cases = {
        "gg_run_scans": lambda: L.gg_run_scans(g._h, 1, desc(), 0),
        "gg_filter_cloud_batch": lambda: L.gg_filter_cloud_batch(g._h, 1, desc(), pp, None),
        "gg_filter_cloud_batch_begin": lambda: L.gg_filter_cloud_batch_begin(g._h, 1, desc(), pp, None, C.byref(ticket)),
        "merged": lambda: L.gg_run_merged_cloud_msgs_to_device(g._h, 1, desc(), capi._ptr(n_parts_), capi._ptr(parts_), None, 0, None, None),
    }
    for name, fn in cases.items():
        assert fn() == ARG, name
        assert g.kernel_launches == before, name
    # flagged scan of a slot without a stored count (slot 2 after its init_map)
    g.init_map(0.0, 0.0, 0.0, slot=2)
    g.synchronize()
    before = g.kernel_launches
    d2 = desc(2)
    assert L.gg_run_scans_device(g._h, 1, d2, (C.c_void_p * 1)(dev.data_ptr()), 0) == STATE
    assert g.kernel_launches == before
    # the set call
    sl = np.array([0, 1], np.int32)
    p = counts.data_ptr()
    layer = g.layer_device_ptr("ground", slot=1)
    set_cases = {
        "null handle": (lambda: L.gg_set_point_counts_from_device(None, 2, capi._ptr(sl), p, None), ARG),
        "null slots": (lambda: L.gg_set_point_counts_from_device(g._h, 2, None, p, None), ARG),
        "null counts": (lambda: L.gg_set_point_counts_from_device(g._h, 2, capi._ptr(sl), None, None), ARG),
        "negative count": (lambda: L.gg_set_point_counts_from_device(g._h, -1, capi._ptr(sl), p, None), ARG),
        "count > n_slots": (lambda: L.gg_set_point_counts_from_device(g._h, B + 1, capi._ptr(np.arange(B + 1, dtype=np.int32)), p, None), ARG),
        "slot out of range": (lambda: L.gg_set_point_counts_from_device(g._h, 2, capi._ptr(np.array([0, B], np.int32)), p, None), ARG),
        "negative slot": (lambda: L.gg_set_point_counts_from_device(g._h, 1, capi._ptr(np.array([-1], np.int32)), p, None), ARG),
        "repeated slot": (lambda: L.gg_set_point_counts_from_device(g._h, 2, capi._ptr(np.array([1, 1], np.int32)), p, None), ARG),
        "misaligned": (lambda: L.gg_set_point_counts_from_device(g._h, 2, capi._ptr(sl), p + 2, None), ARG),
        "overlaps the layers": (lambda: L.gg_set_point_counts_from_device(g._h, 2, capi._ptr(sl), layer + 64, None), ARG),
        "map not initialised": (lambda: L.gg_set_point_counts_from_device(g2._h, 1, capi._ptr(np.array([0], np.int32)), p, None), STATE),
        "count 0": (lambda: L.gg_set_point_counts_from_device(g._h, 0, None, None, None), 0),
    }
    g2 = capi.GroundGridB200(99.0, 0.33, n_slots=1, max_points=MAX_POINTS)
    before2 = g2.kernel_launches
    for name, (fn, want) in set_cases.items():
        assert fn() == want, name
        assert g.kernel_launches == before and g2.kernel_launches == before2, name
    # the handle is still usable: the stored counts of slots 0 and 1 are intact
    d = g.make_descs([0, 1], [len(pts)] * 2, [org] * 2, [0.0] * 2)
    g.run_scans_device(d, [dev.data_ptr()] * 2, device_counts=True)
    assert g.last_scan_points(slot=0) == len(pts) == g.last_scan_points(slot=1)
    del keep, Tarr

"""Point classes and heights from caller GPU memory (gg_point_info_to_device): the class code and the height above the
terrain of every input point of many slots, written into caller-owned CUDA memory and ordered on the caller's stream.
Codes are checked bit for bit against the same handle's gg_get_point_classes after every scan path; heights against
np.float32(z) - np.float32(ground[cell]) with ground from gg_get_layer and z the map-frame z of the scan (the cloud
itself, or oracle.nextrows.unpack_transform of a payload, which the payload tests hold bit-identical to the device
unpack), and against z - sample_layers_to_device(nearest, "ground") for map-frame clouds."""
import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from oracle import nextrows
from test_gpu_cloud_msgs import cuda_bytes, map_from_sensor, payload
from test_gpu_device_outputs import OTHER_CFGS, advance, make_pair, make_steps, to_device, torch_mod
from test_gpu_merged_cloud_msgs import concat, make_scans, n_of, nested

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
QNAN = np.uint32(0x7FC00000)
MSG_LAYOUTS = {"msgs18": (18, (0, 4, 8, 12, 16)), "msgs32": (32, (0, 4, 8, 16, 20))}


def make_handle(dim, res, B):
    """A handle whose slots 1 and B - 1 run OTHER_CFGS (max_ring 48 / 40: ignored points)."""
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536)
    for slot, kw in zip((1, B - 1), OTHER_CFGS):
        g.set_config(slot=slot, **kw)
    return g


def expected(g, slot, z):
    """(codes, height bits) of the slot's last scan through the per-slot route: gg_get_point_classes, gg_get_layer and
    numpy float32 arithmetic on the map-frame z of the scan's points."""
    n = g.last_scan_points(slot)
    codes = g.point_classes(n, slot=slot)
    assert len(z) == n
    G = g.layer("ground", slot=slot).reshape(-1, order="F")
    cls, cell = codes >> 24, (codes & 0xFFFFFF).astype(np.int64)
    h = np.full(n, QNAN, np.uint32)
    has = cls != capi.PC_ABSENT
    h[has] = (np.asarray(z, np.float32)[has] - G[cell[has]]).astype(np.float32).view(np.uint32)
    return codes, h


def batched(g, slots, **kw):
    torch = torch_mod()
    codes, height = g.point_info_to_device(slots, **kw)
    torch.cuda.synchronize()
    return ([None if codes is None else c.cpu().numpy().view(np.uint32) for c in codes] if codes is not None else None,
            [None if height is None else t.cpu().numpy().view(np.uint32) for t in height] if height is not None else None)


def assert_matches(g, slots, zs, ctx, **kw):
    codes, height = batched(g, slots, **kw)
    seen = np.zeros(6, np.int64)
    for k, s in enumerate(slots):
        want_c, want_h = expected(g, int(s), zs[int(s)])
        assert np.array_equal(codes[k], want_c), f"{ctx}: codes of slot {s}"
        assert np.array_equal(height[k], want_h), f"{ctx}: heights of slot {s}"
        seen += np.bincount(want_c >> 24, minlength=6)[:6]
    return seen


def run_route(g, route, row, slots, base_z, rng, k):
    """One scan per slot through `route`.  Returns {slot: map-frame z of its input points} and what must stay alive until
    the next synchronisation (payloads of the device routes are freed, and their memory refilled, right away)."""
    torch = torch_mod()
    B = len(slots)
    zs = {int(s): np.ascontiguousarray(r[0]["z"]) for s, r in zip(slots, row)}
    descs = g.make_descs([int(s) for s in slots], [len(r[0]) for r in row], [r[1] for r in row], [base_z] * B)
    if route == "filter_cloud":
        for s, r in zip(slots, row):
            g.filter_cloud(r[0], r[1], base_z, slot=int(s))
        return zs, None
    if route in ("batch_packed", "batch_plain"):
        hp = [torch.from_numpy(np.ascontiguousarray(r[0]).view(np.uint8).copy()).pin_memory() for r in row]
        hl = [torch.zeros(len(r[0]), dtype=torch.uint8).pin_memory() for r in row]
        g.filter_cloud_batch_ptrs(descs, [t.data_ptr() for t in hp], [t.data_ptr() for t in hl])
        return zs, (hp, hl)
    if route == "run_scans":
        keep = [g.upload_points(r[0], slot=int(s)) for s, r in zip(slots, row)]
        g.run_scans(descs)
        return zs, keep
    if route == "run_scans_to_device":
        dev = [to_device(r[0]) for r in row]
        g.run_scans_to_device(dev, slots, [r[1] for r in row], base_z, labels=True, select=None)
        sizes = [t.numel() for t in dev]
        del dev
        return zs, [torch.full((n,), 7.5, device="cuda") for n in sizes]
    if route in MSG_LAYOUTS:
        step, offsets = MSG_LAYOUTS[route]
        raws, Ts = [], []
        for b, r in enumerate(row):
            T = map_from_sensor(r[2], 0.3 * b + 0.1 * k) if b % 3 != 1 else None
            raws.append(payload(r[0], step, offsets, T, rng))
            Ts.append(T)
            zs[int(slots[b])] = nextrows.unpack_transform(raws[-1], len(r[0]), step, offsets, T)["z"]
        dev = [cuda_bytes(raw) for raw in raws]
        g.run_cloud_msgs_to_device(dev, step, offsets, Ts, slots, [r[1] for r in row], base_z, labels=True, select=None)
        sizes = [t.numel() for t in dev]
        del dev
        return zs, [torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda") for n in sizes]
    assert route == "merged"
    scans = make_scans(row, k, rng)
    for s, parts in zip(slots, scans):
        zs[int(s)] = concat(parts)["z"]
    dev = [[cuda_bytes(p[0]) for p in parts] for parts in scans]
    g.run_merged_cloud_msgs_to_device(dev, nested(scans, 1), nested(scans, 2), nested(scans, 3), slots, [r[1] for r in row], base_z,
                                      labels=True, select=None)
    assert any(n_of(parts) == 0 or any(len(p[0]) == 0 for p in parts) for parts in scans), "an empty part"
    del dev
    return zs, None


ROUTES = ["filter_cloud", "batch_packed", "batch_plain", "run_scans", "run_scans_to_device", "msgs18", "msgs32", "merged"]


@pytest.mark.parametrize("dim,res", [(99.0, 0.33), (33.33, 0.33)])   # N = 300 (even), N = 101 (odd)
@pytest.mark.parametrize("route", ROUTES)
def test_every_scan_path(monkeypatch, route, dim, res):
    """Codes and heights of every slot after each scan path, over two steps with a roll between them; slots 1 and B - 1
    run their own configurations (max_ring 48 / 40: ignored points); the second step pushes a share of points below the
    ground (outliers)."""
    if route.startswith("batch"):
        monkeypatch.setenv("GG_HOST_PACK", "1" if route == "batch_packed" else "0")
        monkeypatch.setenv("GG_HOST_THREADS", "2")
    B = 6
    g = make_handle(dim, res, B)
    slots = np.arange(B, dtype=np.int32)[::-1].copy()
    rng = np.random.default_rng(9100)
    seen = np.zeros(6, np.int64)
    for k, row in enumerate(make_steps(B, 2, seed=9100)):
        advance([g], k, row, slots)
        zs, keep = run_route(g, route, row, slots, 0.02 * k, rng, k)
        if route == "batch_packed":
            assert g.last_batch_transfer()[0] == B, "every scan was packed"
        if route == "batch_plain":
            assert g.last_batch_transfer()[1] == B, "every scan went as 32-byte records"
        order = np.random.default_rng(k).permutation(B).astype(np.int32)
        seen += assert_matches(g, order, zs, f"{route} step {k}")
        del keep
    for c in (capi.PC_KEPT, capi.PC_IGNORED, capi.PC_OUTLIER) + ((capi.PC_ABSENT,) if dim < 50 else ()):
        assert seen[c] > 0, f"{route}: class {c} never occurred"
    g.close()


def test_heights_match_sampled_ground_and_outputs_are_optional():
    """For map-frame clouds, height == z - sample_layers_to_device(nearest, "ground") at every point inside the map; codes
    only, heights only, preallocated outputs and an empty scan."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 4
    g = make_handle(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    for k, row in enumerate(make_steps(B, 2, seed=9200)):
        advance([g], k, row, slots)
        dev = [to_device(r[0]) for r in row]
        dev[2] = dev[2][:0] if k else dev[2]          # an empty scan in the second step
        g.run_scans_to_device(dev, slots, [r[1] for r in row], 0.0, labels=True, select=None)
        codes, height = g.point_info_to_device(slots)
        vals, cells = g.sample_layers_to_device(slots, [d.reshape(-1, 8) for d in dev], ("ground",), cells=True)
        for b in range(B):
            inside = cells[b] >= 0
            assert bool((cells[b][inside] == (codes[b][inside] & 0xFFFFFF)).all()), "a point's code names the sampled cell"
            want = dev[b][:, 2] - vals[b][0]
            assert torch.equal(height[b][inside].view(torch.int32), want[inside].view(torch.int32)), f"step {k} slot {b}"
            assert bool(((codes[b] >> 24) == 0).eq(~inside).all()), "absent points are the points outside the map"
            assert bool((height[b][~inside].view(torch.int32) == 0x7FC00000).all())
        assert len(codes[2]) == len(dev[2]) and (k == 0 or len(codes[2]) == 0)
        c_only, h_none = g.point_info_to_device(slots, height=False)
        h_none2, h_only = g.point_info_to_device(slots, codes=False)
        assert h_none is None and h_none2 is None
        pre = ([torch.full_like(c, -5) for c in codes], [torch.full_like(h, 3.0) for h in height])
        got = g.point_info_to_device(slots, out=pre)
        assert all(a is b for a, b in zip(got[0], pre[0]))
        torch.cuda.synchronize()
        for b in range(B):
            assert torch.equal(c_only[b], codes[b]) and torch.equal(pre[0][b], codes[b])
            assert torch.equal(h_only[b].view(torch.int32), height[b].view(torch.int32))
            assert torch.equal(pre[1][b].view(torch.int32), height[b].view(torch.int32))
    g.close()


@pytest.mark.parametrize("which", ["current", "side"])
def test_stream_order_without_host_waits(which):
    """(a) the call returns while the stream is still busy, (b) it sees the scan enqueued right before it, (c) a clone
    enqueued right after it sees the outputs, (d) a roll and the slot's next scan enqueued right after it change neither.
    The expected values come from a twin that ran the same first two steps only."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 4
    g, twin = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    steps = make_steps(B, 3, seed=9300)
    stream = torch.cuda.current_stream() if which == "current" else torch.cuda.Stream()
    if which == "current":
        assert stream.cuda_stream == 0
    dev = [[to_device(r[0]) for r in row] for row in steps]
    torch.cuda.synchronize()
    for k in range(2):
        advance([twin], k, steps[k], slots)
        twin.run_scans_to_device(dev[k], slots, [r[1] for r in steps[k]], 0.0, labels=True, select=None)
    want = [expected(twin, b, steps[1][b][0]["z"]) for b in range(B)]
    twin.close()
    advance([g], 0, steps[0], slots)
    with torch.cuda.stream(stream):   # warm-up: module loads, allocator pools
        g.run_scans_to_device(dev[0], slots, [r[1] for r in steps[0]], 0.0, labels=True, select=None, stream=stream)
        g.point_info_to_device(slots, stream=stream)
    torch.cuda.synchronize()
    before = torch.cuda.Event()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(400_000_000)               # ~200 ms of device time ahead of everything below
        before.record(stream)
        advance([g], 1, steps[1], slots)
        g.run_scans_to_device(dev[1], slots, [r[1] for r in steps[1]], 0.0, labels=True, select=None, stream=stream)
        codes, height = g.point_info_to_device(slots, stream=stream)
        assert not before.query(), "gg_point_info_to_device waited on the host for the stream"
        clone = [h.clone() for h in height]
        advance([g], 2, steps[2], slots)
        g.run_scans_to_device(dev[2], slots, [r[1] for r in steps[2]], 0.0, labels=True, select=None, stream=stream)
        assert not before.query(), "the next roll and scan waited on the host"
    pending = not before.query()
    torch.cuda.synchronize()
    assert pending, "the sleep did not cover the calls"
    for b in range(B):
        assert np.array_equal(codes[b].cpu().numpy().view(np.uint32), want[b][0]), f"{which}: codes of slot {b}"
        assert np.array_equal(height[b].cpu().numpy().view(np.uint32), want[b][1]), f"{which}: heights of slot {b}"
        assert np.array_equal(clone[b].cpu().numpy().view(np.uint32), want[b][1]), f"{which}: clone of slot {b}"
    g.close()


def test_rejected_calls_enqueue_nothing():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 7
    g = capi.GroundGridB200(dim, res, n_slots=B + 1, max_points=65536)   # slot B is never initialised
    steps = make_steps(B, 1, seed=9400)
    row = steps[0]
    for b, r in enumerate(row):
        g.init_map(r[2][0], r[2][1], 0.0, slot=b)
    dev = [to_device(r[0]) for r in row]
    torch.cuda.synchronize()
    full = [0, 1, 2, 3, 6]
    descs = g.make_descs(full, [len(row[b][0]) for b in full], [row[b][1] for b in full], [0.0] * len(full))
    g.run_scans_device(descs, [dev[b].data_ptr() for b in full])
    g.run_scans_device(g.make_descs([4], [len(row[4][0])], [row[4][1]], [0.0]), [dev[4].data_ptr()], stop_after=1)   # stopped early
    T = row[5][3].reshape(1, 12)
    g.update_pose_batch(np.array([5], np.int32), np.array([row[5][2]]), T)          # slot 5: no scan, a roll only
    x, y = g.position(slot=3)
    g.update_pose_batch(np.array([3], np.int32), np.array([[x + 2.0, y]]), T)        # slot 3: moved after its scan
    x, y = g.position(slot=6)
    g.update_pose_batch(np.array([6], np.int32), np.array([[x, y]]), T)              # slot 6: a roll that does not move
    g.synchronize()
    n = max(g.last_scan_points(b) for b in range(B))
    buf = torch.full((8, n + 64), 0x3C3C3C3C, dtype=torch.int32, device="cuda")
    P = [buf[j].data_ptr() for j in range(8)]
    arena = g.layer_device_ptr("ground", slot=0)
    sl = np.ascontiguousarray([0, 1], np.int32)
    outs = np.zeros(2, capi.POINT_INFO_DTYPE)
    outs["codes"], outs["height"] = P[0], P[1]

    def call(slots_=(0, 1), codes=None, height=None):
        slots_ = list(slots_)
        codes = P[:len(slots_)] if codes is None else codes
        height = P[4:4 + len(slots_)] if height is None else height
        g.point_info_to_device_ptrs(slots_, codes, height, None)

    def raw(h, count, slots_ptr, outs_ptr):
        rc = g._l.gg_point_info_to_device(h, count, slots_ptr, outs_ptr, None)
        if rc != 0:
            raise capi.GroundGridError(rc, g._l.gg_last_error().decode())

    n1 = g.last_scan_points(1)
    cases = {
        "null handle": (ARG, lambda: raw(None, 2, sl.ctypes.data, outs.ctypes.data)),
        "null slots": (ARG, lambda: raw(g._h, 2, None, outs.ctypes.data)),
        "null outs": (ARG, lambda: raw(g._h, 2, sl.ctypes.data, None)),
        "negative count": (ARG, lambda: raw(g._h, -1, sl.ctypes.data, outs.ctypes.data)),
        "misaligned codes": (ARG, lambda: call(codes=[P[0], P[1] + 2])),
        "misaligned height": (ARG, lambda: call(height=[P[4] + 1, P[5]])),
        "codes in the arena": (ARG, lambda: call(codes=[arena, P[1]])),
        "height ends in the arena": (ARG, lambda: call(height=[P[4], arena - 4 * n1 + 4])),
        "codes of one slot over the height of another": (ARG, lambda: call(codes=[P[0], P[4] + 4])),
        "codes and height of one slot overlap": (ARG, lambda: call(codes=[P[0], P[1]], height=[P[4], P[1] + 8])),
        "count exceeds slots": (ARG, lambda: call(list(range(B + 1)) + [0], codes=[0] * (B + 2), height=[0] * (B + 2))),
        "slot out of range": (ARG, lambda: call([0, B + 1])),
        "negative slot": (ARG, lambda: call([0, -1])),
        "repeated slot": (ARG, lambda: call([0, 2, 2])),
        "map not initialised": (STATE, lambda: call([0, B])),
        "stopped early": (STATE, lambda: call([0, 4])),
        "rolled only since gg_init_map": (STATE, lambda: call([1, 5])),
        "moved since the scan": (STATE, lambda: call([1, 3])),
    }
    for name, (code, fn) in cases.items():
        l0 = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            fn()
        assert e.value.code == code, f"{name}: code {e.value.code}"
        assert g.kernel_launches == l0, f"{name}: something was launched"
    l0 = g.kernel_launches
    call([])                                   # an empty batch is accepted and enqueues nothing
    raw(g._h, 0, None, None)
    g.point_info_to_device_ptrs([0, 1], None, None, None)   # nothing to write: accepted, nothing enqueued
    assert g.kernel_launches == l0
    torch.cuda.synchronize()
    assert (buf == 0x3C3C3C3C).all(), "a rejected call wrote into the buffers"
    # the handle is still usable; a roll that does not move keeps the slot readable
    zs = {b: row[b][0]["z"] for b in full}
    assert_matches(g, [6, 0, 2], zs, "after the rejections")
    g.close()


def test_rolling_stream_of_100_scans():
    """100 scans with rolls between them on three slots (N = 101), each step checked against the per-slot route and
    against the sampled ground; the slots' batch order changes every step."""
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 3
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536)
    g.set_config(slot=1, **OTHER_CFGS[0])
    slots = np.arange(B, dtype=np.int32)
    scenes = [synth.make_scene(seed=9500 + b, stream_len=90.0, undulation=0.2) for b in range(B)]
    rng = np.random.default_rng(9500)
    seen = np.zeros(6, np.int64)
    for k in range(100):
        row = []
        for b in range(B):
            ex, ey, yaw = 0.8 * k + 0.1 * b, 0.3 * np.sin(0.1 * k + b), 0.02 * np.sin(0.05 * k)
            pts, org = synth.lidar_scan(scenes[b], ego_xy=(ex, ey), yaw=yaw, beams=64, az_steps=192, seed=9500 + 10 * k + b)
            if k:
                idx = rng.choice(len(pts), len(pts) // 100, replace=False)
                pts["z"][idx] -= rng.uniform(0.3, 1.2, len(idx)).astype(np.float32)
            row.append((pts, org, (ex, ey), synth.base_from_map(ex, ey, yaw, base_z=0.0, pitch=0.01)))
        advance([g], k, row, slots)
        dev = [to_device(r[0]) for r in row]
        g.run_scans_to_device(dev, slots, [r[1] for r in row], 0.0, labels=True, select=None)
        order = rng.permutation(B).astype(np.int32)
        seen += assert_matches(g, order, {b: row[b][0]["z"] for b in range(B)}, f"step {k}")
        _, height = g.point_info_to_device(slots, codes=False)
        vals, cells = g.sample_layers_to_device(slots, [d.reshape(-1, 8) for d in dev], ("ground",), cells=True)
        for b in range(B):
            inside = cells[b] >= 0
            want = dev[b][:, 2] - vals[b][0]
            assert torch.equal(height[b][inside].view(torch.int32), want[inside].view(torch.int32)), f"step {k} slot {b}: sampled"
    assert seen[capi.PC_OUTLIER] > 0 and seen[capi.PC_IGNORED] > 0 and seen[capi.PC_KEPT_BORDER] > 0
    g.close()

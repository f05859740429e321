"""Poses from caller GPU memory (gg_update_poses_from_device): rolls resolved on the device and scan poses stored per
slot, used by scans flagged GG_SCAN_DEVICE_POSE.  Every case runs against a twin handle driven by the host calls
(gg_update_pose_batch, host origins / base_z) on the same clouds, and must be bit-identical to it: labels, output
clouds, layers, the moved flags and the map positions read back afterwards."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from test_gpu_cloud_msgs import cuda_bytes
from test_gpu_device_outputs import LIVE, make_pair, to_device, torch_mod
import cloud_orders

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
MSG = (32, (0, 4, 8, 16, 20))   # a 32-byte PointXYZIR record as a PointCloud2 payload in the map frame
ROUTES = ["run_scans", "run_scans_device", "run_scans_to_device", "msgs", "merged", "batch_packed", "batch_plain"]
STEPS = 32
_STEP_CACHE = {}


def pose_steps(B, steps, jump, seed=4200):
    """[step][slot] -> (points, origin, ego xy, T, base_z): yaw, a pitched base frame, a step without movement every
    seventh step and one jump of `jump` metres (a whole-map shift) half way."""
    key = (B, steps, jump, seed)
    if key in _STEP_CACHE:
        return _STEP_CACHE[key]
    scenes = [synth.make_scene(seed=seed + b, stream_len=10.0, undulation=0.2) for b in range(B)]
    ego = [[0.05 * b, 0.0] for b in range(B)]
    out = []
    for k in range(steps):
        row = []
        for b in range(B):
            if k == steps // 2:
                ego[b] = [ego[b][0] + jump, ego[b][1] - 0.5 * jump]
            elif k and k % 7 != 3:
                ego[b] = [ego[b][0] + 0.8 + 0.05 * b, ego[b][1] - 0.35 * (b % 3)]
            yaw = 0.04 * k * (1 + b % 2)
            pts, org = synth.lidar_scan(scenes[b], ego_xy=tuple(ego[b]), yaw=yaw, beams=32, az_steps=512, seed=seed + 100 * k + b)
            row.append((pts, org, tuple(ego[b]), synth.base_from_map(ego[b][0], ego[b][1], yaw, base_z=0.0, pitch=0.01), 0.02 * k + 0.001 * b))
        out.append(row)
    _STEP_CACHE[key] = out
    return out


def device_poses(row, torch):
    """The poses of a row as CUDA tensors (xy, T, origins, base_z)."""
    return (torch.tensor(np.array([r[2] for r in row], np.float64), device="cuda"),
            torch.tensor(np.stack([r[3].reshape(12) for r in row]), dtype=torch.float64, device="cuda"),
            torch.tensor(np.array([r[1] for r in row], np.float32), device="cuda"),
            torch.tensor(np.array([r[4] for r in row], np.float64), device="cuda"))


def run_route(h, route, slots, row, origins, keep):
    """One scan per slot through `route`; origins is the list of host origins (base_z from the row) or "device"."""
    torch = torch_mod()
    slots = [int(s) for s in slots]
    n = [len(r[0]) for r in row]
    base_z = [r[4] for r in row]
    if route == "run_scans":
        keep += [h.upload_points(r[0], slot=s) for s, r in zip(slots, row)]
        h.run_scans(h.make_descs(slots, n, origins, base_z))
    elif route == "run_scans_device":
        dev = [to_device(r[0]) for r in row]
        keep += dev
        h.run_scans_device(h.make_descs(slots, n, origins, base_z), [t.data_ptr() for t in dev])
    elif route == "run_scans_to_device":
        dev = [to_device(r[0]) for r in row]
        keep += dev
        keep.append(h.run_scans_to_device(dev, slots, origins, base_z, labels=True, select="all", index=True))
    elif route == "msgs":
        dev = [cuda_bytes(np.ascontiguousarray(r[0]).view(np.uint8)) for r in row]
        h.run_cloud_msgs_to_device(dev, MSG[0], MSG[1], None, slots, origins, base_z, labels=True, select=None)
    elif route == "merged":
        dev = []
        for j, r in enumerate(row):
            raw = np.ascontiguousarray(r[0]).view(np.uint8)
            cut = 32 * ((len(r[0]) * (j + 1)) // (len(row) + 1))
            dev.append([cuda_bytes(raw[:cut]), cuda_bytes(raw[cut:])])
        h.run_merged_cloud_msgs_to_device(dev, MSG[0], MSG[1], None, slots, origins, base_z, labels=True, select=None)
    else:
        hp = [torch.from_numpy(np.ascontiguousarray(r[0]).view(np.uint8).copy()).pin_memory() for r in row]
        keep += hp
        h.filter_cloud_batch_ptrs(h.make_descs(slots, n, origins, base_z), [t.data_ptr() for t in hp], None)


def labels_of(h, slots, row):
    out = [h.download_labels(len(r[0]), slot=int(s)) for s, r in zip(slots, row)]
    h.synchronize()
    return out


def assert_same_state(g, twin, slots, ctx, names=LIVE, output=True, cloud=True):
    for s in slots:
        s = int(s)
        for name in names:
            assert np.array_equal(g.layer(name, slot=s).view(np.uint32), twin.layer(name, slot=s).view(np.uint32)), f"{ctx} slot {s}: {name}"
        if output:
            gi, gc = g.get_output(slot=s, want_cloud=cloud)
            ti, tc = twin.get_output(slot=s, want_cloud=cloud)
            assert np.array_equal(gi, ti) and (not cloud or gc.tobytes() == tc.tobytes()), f"{ctx} slot {s}: get_output"
        assert g.position(slot=s).view(np.uint64).tolist() == twin.position(slot=s).view(np.uint64).tolist(), f"{ctx} slot {s}: position"


@pytest.mark.parametrize("dim,res,B", [(99.0, 0.33, 4), (33.33, 0.33, 10)])   # N = 300, 101
@pytest.mark.parametrize("route", ROUTES)
def test_rolling_streams_through_every_scan_path(monkeypatch, route, dim, res, B):
    """32 steps of device rolls and device scan poses on permuted batches over several stream groups (two slots on
    their own configuration); the twin runs the same steps with host poses.  dev_moved equals the host's moved flags
    every step (including steps that do not move and the whole-map jump); labels are equal every step; layers,
    gg_get_output and positions at the jump and at the end."""
    torch = torch_mod()
    if route.startswith("batch"):
        monkeypatch.setenv("GG_HOST_PACK", "1" if route == "batch_packed" else "0")
        monkeypatch.setenv("GG_HOST_THREADS", "2")
    g, twin = make_pair(dim, res, B)
    rng = np.random.default_rng(B)
    steps = pose_steps(B, STEPS, jump=1.5 * dim)
    moved_seen = set()
    for k, full_row in enumerate(steps):
        slots = rng.permutation(B).astype(np.int32)
        row = [full_row[s] for s in slots]
        xy, T, origins, bz = device_poses(row, torch)
        if k == 0:
            for s, r in zip(slots, row):
                g.init_map(r[2][0], r[2][1], 0.0, slot=int(s))
                twin.init_map(r[2][0], r[2][1], 0.0, slot=int(s))
            assert g.update_poses_from_device(slots, origins=origins, base_z=bz) is None
        else:
            moved = g.update_poses_from_device(slots, xy, T, origins, bz, moved=True)
            want = twin.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))
            got = moved.cpu().numpy()
            assert np.array_equal(got, want.astype(np.int32)), f"step {k}: dev_moved {got} != {want}"
            moved_seen.update(got.tolist())
        del xy, T, origins, bz
        keep = []
        run_route(g, route, slots, row, "device", keep)
        run_route(twin, route, slots, row, [r[1] for r in row], keep)
        for s, a, b in zip(slots, labels_of(g, slots, row), labels_of(twin, slots, row)):
            assert np.array_equal(a, b), f"{route} step {k} slot {s}: labels"
        if k in (STEPS // 2, STEPS - 1):
            assert_same_state(g, twin, slots, f"{route} step {k}", cloud=route != "batch_packed")
            # position() took the positions back to the host: the next device roll starts from them
    assert moved_seen == {0, 1}


@pytest.mark.parametrize("position", [(1.2e5, -3.4e5), (4.1e5, 5.6e6)])
def test_far_from_the_origin_with_lookups_and_heights(position):
    """Device rolls around map positions far from the origin (float32 clouds are coarse there), then terrain lookups at
    the scan's points and per-point heights, bit-identical to the twin's."""
    torch = torch_mod()
    B = 3
    g, twin = make_pair(99.0, 0.33, B)
    scene = cloud_orders.far_scene(position, seed=77)
    slots = np.arange(B, dtype=np.int32)
    for h in (g, twin):
        for s in slots:
            h.init_map(position[0], position[1], 0.0, slot=int(s))
    for k in range(6):
        row = []
        for b in range(B):
            ego = (position[0] + 0.7 * k + 0.1 * b, position[1] - 0.4 * k)
            pts, org = synth.lidar_scan(scene, ego_xy=ego, yaw=0.03 * k, beams=32, az_steps=512, seed=500 + 10 * k + b)
            row.append((pts, org, ego, synth.base_from_map(ego[0], ego[1], 0.03 * k, pitch=0.01), 0.01 * k))
        xy, T, origins, bz = device_poses(row, torch)
        moved = g.update_poses_from_device(slots, xy, T, origins, bz, moved=True)
        want = twin.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))
        assert np.array_equal(moved.cpu().numpy(), want.astype(np.int32)), f"step {k}: moved"
        keep = []
        run_route(g, "run_scans_to_device", slots, row, "device", keep)
        run_route(twin, "run_scans_to_device", slots, row, [r[1] for r in row], keep)
        queries = [to_device(r[0]) for r in row]
        gs, gc = g.sample_layers_to_device(slots, queries, names=("ground", "groundpatch"), mode="linear", cells=True)
        ts, tc = twin.sample_layers_to_device(slots, queries, names=("ground", "groundpatch"), mode="linear", cells=True)
        gh = g.point_info_to_device(slots)
        th = twin.point_info_to_device(slots)
        torch.cuda.synchronize()
        for j in range(B):
            assert torch.equal(gs[j].view(torch.int32), ts[j].view(torch.int32)) and torch.equal(gc[j], tc[j]), f"step {k}: lookups"
            assert torch.equal(gh[0][j], th[0][j]) and torch.equal(gh[1][j].view(torch.int32), th[1][j].view(torch.int32)), f"step {k}: heights"
        for s, a, b in zip(slots, labels_of(g, slots, row), labels_of(twin, slots, row)):
            assert np.array_equal(a, b), f"step {k} slot {s}: labels"
    assert_same_state(g, twin, slots, "far")


def test_mixing_host_and_device_calls():
    """Device rolls, then gg_get_map_position and a host roll; gg_set_map_position and gg_init_map after device rolls;
    terrain lookups after a device roll whose position the host never read back."""
    torch = torch_mod()
    B = 4
    g, twin = make_pair(99.0, 0.33, B)
    steps = pose_steps(B, 9, jump=150.0, seed=4300)
    slots = np.arange(B, dtype=np.int32)

    alive = []   # the callers' clouds, which gg_get_output reads

    def scan(k, host_slots=()):
        row = steps[k]
        keep = alive
        for s in slots:
            origins = [row[s][1]] if s in host_slots else "device"
            run_route(g, "run_scans_to_device", [s], [row[s]], origins, keep)
        run_route(twin, "run_scans_to_device", slots, row, [r[1] for r in row], keep)
        for s, a, b in zip(slots, labels_of(g, slots, row), labels_of(twin, slots, row)):
            assert np.array_equal(a, b), f"step {k} slot {s}: labels"

    def device_roll(k, sl):
        row = [steps[k][s] for s in sl]
        xy, T, origins, bz = device_poses(row, torch)
        g.update_poses_from_device(sl, xy, T, origins, bz)
        twin.update_pose_batch(sl, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))

    for h in (g, twin):
        for s in slots:
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=int(s))
    device_roll(0, slots)        # scan poses (and rolls that do not move)
    scan(0)
    for k in (1, 2):
        device_roll(k, slots)
        scan(k)
    # gg_get_map_position after device rolls, then a host roll of the same slot
    assert g.position(slot=0).tolist() == twin.position(slot=0).tolist()
    r = steps[3][0]
    assert g.update_pose(r[2][0], r[2][1], r[3], slot=0) == twin.update_pose(r[2][0], r[2][1], r[3], slot=0)
    device_roll(3, slots[1:])
    g.update_poses_from_device([0], origins=torch.tensor(np.array([r[1]], np.float32), device="cuda"),
                               base_z=torch.tensor([r[4]], dtype=torch.float64, device="cuda"))
    scan(3)
    # gg_set_map_position on slot 1 and gg_init_map on slot 2 right after device rolls (no read back in between)
    device_roll(4, slots)
    for h in (g, twin):
        h.set_position(steps[4][1][2][0] + 0.9, steps[4][1][2][1] - 0.4, slot=1)
        h.init_map(steps[4][2][2][0], steps[4][2][2][1], 0.1, slot=2)
    with pytest.raises(capi.GroundGridError) as e:   # gg_init_map dropped the slot's device scan pose
        g.run_scans(g.make_descs([2], [len(steps[4][2][0])], "device", None))
    assert e.value.code == STATE
    scan(4, host_slots=(2,))
    assert_same_state(g, twin, slots, "after set_map_position / init_map")
    # lookups after a device roll the host never read back
    device_roll(5, slots)
    queries = [to_device(steps[6][s][0]) for s in slots]
    for mode in ("nearest", "linear"):
        gs, gc = g.sample_layers_to_device(slots, queries, mode=mode, cells=True)
        ts, tc = twin.sample_layers_to_device(slots, queries, mode=mode, cells=True)
        torch.cuda.synchronize()
        for j in range(B):
            assert torch.equal(gs[j].view(torch.int32), ts[j].view(torch.int32)) and torch.equal(gc[j], tc[j]), f"{mode} lookups slot {j}"
    scan(5)
    assert_same_state(g, twin, slots, "end")


def test_scan_poses_without_a_roll_and_mixed_flags():
    """Scan poses only (xy NULL), host rolls on both handles; a batch mixing flagged and unflagged scans."""
    torch = torch_mod()
    B = 6
    g, twin = make_pair(33.33, 0.33, B)
    steps = pose_steps(B, 5, jump=50.0, seed=4400)
    slots = np.arange(B, dtype=np.int32)[::-1].copy()
    for k, full_row in enumerate(steps):
        row = [full_row[s] for s in slots]
        for h in (g, twin):
            if k == 0:
                for s, r in zip(slots, row):
                    h.init_map(r[2][0], r[2][1], 0.0, slot=int(s))
            else:
                h.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))
        _, _, origins, bz = device_poses(row, torch)
        moved = g.update_poses_from_device(slots, origins=origins, base_z=bz, moved=True)
        assert moved.cpu().tolist() == [0] * B
        descs = g.make_descs(slots, [len(r[0]) for r in row], [r[1] for r in row], [r[4] for r in row])
        for j in range(B):
            if (j + k) % 2:
                descs[j].flags = capi.SCAN_DEVICE_POSE
                descs[j].origin[0] = descs[j].origin[1] = descs[j].origin[2] = 1.0e4   # ignored
                descs[j].base_z = -50.0
        keep = [g.upload_points(r[0], slot=int(s)) for s, r in zip(slots, row)]
        g.run_scans(descs)
        run_route(twin, "run_scans", slots, row, [r[1] for r in row], keep)
        for s, a, b in zip(slots, labels_of(g, slots, row), labels_of(twin, slots, row)):
            assert np.array_equal(a, b), f"step {k} slot {s}: labels"
    assert_same_state(g, twin, slots, "scan poses")


def test_invalid_poses_leave_map_and_position_untouched():
    torch = torch_mod()
    B = 5
    g, twin = make_pair(99.0, 0.33, B)
    steps = pose_steps(B, 3, jump=10.0, seed=4500)
    slots = np.arange(B, dtype=np.int32)
    for h in (g, twin):
        for s in slots:
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=int(s))
    keep = []
    run_route(g, "run_scans", slots, steps[0], [r[1] for r in steps[0]], keep)
    run_route(twin, "run_scans", slots, steps[0], [r[1] for r in steps[0]], keep)
    g.synchronize()
    twin.synchronize()
    row = steps[1]
    xy = np.array([r[2] for r in row], np.float64)
    bad = {0: (np.nan, 0.0), 1: (0.0, np.inf), 2: (-np.inf, np.nan), 3: (1.0e12, 0.0)}   # slot 3: a shift outside int32
    for s, v in bad.items():
        xy[s] = v
    T = np.stack([r[3].reshape(12) for r in row])
    moved = g.update_poses_from_device(slots, torch.tensor(xy, device="cuda"), torch.tensor(T, device="cuda"), moved=True)
    want4 = twin.update_pose_batch([4], xy[4:], T[4:])
    assert moved.cpu().tolist() == [-1, -1, -1, -1, int(want4[0])]
    assert_same_state(g, twin, slots, "invalid poses", names=("ground", "groundpatch"), output=False)
    # a valid device roll afterwards continues from the untouched positions
    r2 = steps[2]
    xy2 = np.array([r[2] for r in r2], np.float64)
    T2 = np.stack([r[3].reshape(12) for r in r2])
    moved = g.update_poses_from_device(slots, torch.tensor(xy2, device="cuda"), torch.tensor(T2, device="cuda"), moved=True)
    assert moved.cpu().tolist() == twin.update_pose_batch(slots, xy2, T2).astype(int).tolist()
    assert_same_state(g, twin, slots, "after a valid roll", names=("ground", "groundpatch"), output=False)


@pytest.mark.parametrize("which", ["legacy", "side"])
def test_stream_order_without_host_waits(which):
    """Poses written by torch kernels on the caller's stream right before each call (behind a sleep kernel), freed and
    their memory refilled with NaN right after it, dev_moved cloned right after it, scans on the same stream; no host
    wait until the end."""
    torch = torch_mod()
    B = 4
    g, twin = make_pair(99.0, 0.33, B)
    steps = pose_steps(B, 8, jump=12.0, seed=4600)
    slots = np.arange(B, dtype=np.int32)
    for h in (g, twin):
        for s in slots:
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=int(s))
    src = [device_poses(row, torch) for row in steps]
    clouds = [[to_device(r[0]) for r in row] for row in steps]
    torch.cuda.synchronize()
    stream = torch.cuda.Stream() if which == "side" else torch.cuda.default_stream()
    moved_copies, labels = [], []
    with torch.cuda.stream(stream):
        for k in range(len(steps)):
            torch.cuda._sleep(20_000_000)
            poses = [torch.empty_like(t).copy_(t) for t in src[k]]
            moved = g.update_poses_from_device(slots, *poses, moved=True, stream=stream)
            sizes = [t.numel() for t in poses]
            del poses
            refill = [torch.full((n,), float("nan"), dtype=torch.float64) for n in sizes]
            moved_copies.append(moved.clone())
            out = g.run_scans_to_device(clouds[k], slots, "device", None, labels=True, select=None, stream=stream)
            labels.append(out.labels)
            del refill
    stream.synchronize()
    for k, row in enumerate(steps):
        want = twin.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))
        assert moved_copies[k].cpu().tolist() == want.astype(int).tolist(), f"step {k}: dev_moved"
        keep = []
        run_route(twin, "run_scans_device", slots, row, [r[1] for r in row], keep)
        for j, (s, b) in enumerate(zip(slots, labels_of(twin, slots, row))):
            assert np.array_equal(labels[k][j].cpu().numpy(), b), f"step {k} slot {s}: labels"
    assert_same_state(g, twin, slots, which, output=False)


def test_rejections_enqueue_nothing_and_state_rules():
    torch = torch_mod()
    B = 4
    g = capi.GroundGridB200(33.33, 0.33, n_slots=B, max_points=65536)
    for s in range(3):
        g.init_map(0.0, 0.0, 0.0, slot=s)
    xy = torch.zeros((B, 2), dtype=torch.float64, device="cuda")
    T = torch.tensor(np.tile(synth.base_from_map(0.0, 0.0).reshape(12), (B, 1)), device="cuda")
    org = torch.zeros((B, 3), dtype=torch.float32, device="cuda")
    bz = torch.zeros(B, dtype=torch.float64, device="cuda")
    moved = torch.zeros(2 * B, dtype=torch.int32, device="cuda")
    L = g._l

    def call(count, slots, poses, moved_ptr=None):
        sl = None if slots is None else np.ascontiguousarray(slots, np.int32)
        p = None if poses is None else C.byref(capi.DevicePoses(*poses))
        return L.gg_update_poses_from_device(g._h, count, capi._ptr(sl), p, moved_ptr, None)

    full = (xy.data_ptr(), T.data_ptr(), org.data_ptr(), bz.data_ptr())
    layer = g.layer_device_ptr("ground", slot=1)
    cases = [
        ("null handle", lambda: L.gg_update_poses_from_device(None, 1, None, None, None, None), ARG),
        ("null slots", lambda: call(1, None, full), ARG),
        ("null poses", lambda: call(1, [0], None), ARG),
        ("count > n_slots", lambda: call(B + 1, list(range(B + 1)), full), ARG),
        ("slot out of range", lambda: call(1, [B], full), ARG),
        ("repeated slot", lambda: call(2, [1, 1], full), ARG),
        ("xy without T", lambda: call(1, [0], (full[0], None, None, None)), ARG),
        ("T without xy", lambda: call(1, [0], (None, full[1], None, None)), ARG),
        ("origin without base_z", lambda: call(1, [0], (None, None, full[2], None)), ARG),
        ("base_z without origin", lambda: call(1, [0], (None, None, None, full[3])), ARG),
        ("misaligned xy", lambda: call(1, [0], (full[0] + 4, full[1], None, None)), ARG),
        ("misaligned base_z", lambda: call(1, [0], (None, None, full[2], full[3] + 4)), ARG),
        ("misaligned origin", lambda: call(1, [0], (None, None, full[2] + 2, full[3])), ARG),
        ("misaligned dev_moved", lambda: call(1, [0], full, moved.data_ptr() + 2), ARG),
        ("dev_moved over xy", lambda: call(2, [0, 1], full, full[0] + 8), ARG),
        ("dev_moved over T", lambda: call(2, [0, 1], full, full[1] + 96), ARG),
        ("dev_moved over origin", lambda: call(1, [0], full, full[2]), ARG),
        ("dev_moved over base_z", lambda: call(2, [0, 1], full, full[3] + 4), ARG),
        ("dev_moved over the layers", lambda: call(1, [0], full, layer), ARG),
        ("map not initialised", lambda: call(2, [0, 3], full), STATE),
    ]
    before = g.kernel_launches
    for name, fn, code in cases:
        assert fn() == code, name
        assert g.kernel_launches == before, f"{name}: something was enqueued"
    assert call(0, None, full) == 0 and call(2, [0, 1], (None, None, None, None), moved.data_ptr()) == 0
    assert g.kernel_launches == before
    # a flagged scan needs a device scan pose since gg_init_map
    pts, org0 = synth.lidar_scan(synth.make_scene(seed=3), beams=32, az_steps=512, seed=3)
    g.upload_points(pts, slot=0)
    with pytest.raises(capi.GroundGridError) as e:
        g.run_scans(g.make_descs([0], [len(pts)], "device", None))
    assert e.value.code == STATE and g.kernel_launches == before
    g.update_poses_from_device([0], origins=org[:1], base_z=bz[:1])
    g.run_scans(g.make_descs([0], [len(pts)], "device", None))
    g.synchronize()
    # gg_point_info_to_device: accepted after the scan, refused after a device roll (even one that does not move)
    g.point_info_to_device([0])
    g.update_poses_from_device([0], xy[:1], T[:1])
    with pytest.raises(capi.GroundGridError) as e:
        g.point_info_to_device([0])
    assert e.value.code == STATE
    g.run_scans(g.make_descs([0], [len(pts)], "device", None))
    g.point_info_to_device([0])
    g.synchronize()
    # inputs may share memory: poses whose arrays overlap each other are accepted
    before = g.kernel_launches
    assert call(1, [2], (full[0], full[1], full[1] + 8, full[0])) == 0
    assert g.kernel_launches > before
    g.synchronize()


def test_launch_counts(monkeypatch):
    """An all-host flow launches exactly the kernels it launches on a handle that never used device poses; the device
    flow adds k_pose_resolve per stream group of a roll and k_stage_poses per group of a staged launch with device
    poses."""
    torch = torch_mod()
    monkeypatch.setenv("GG_STREAMS", "3")   # slots 0-1, 2-3, 4-5
    g, fresh = (capi.GroundGridB200(33.33, 0.33, n_slots=6, max_points=65536) for _ in range(2))
    pts, org = synth.lidar_scan(synth.make_scene(seed=5), beams=32, az_steps=512, seed=5)
    for h in (g, fresh):
        for s in range(6):
            h.init_map(0.0, 0.0, 0.0, slot=s)
    T = synth.base_from_map(3.0, 1.0)

    def delta(h, fn):
        before = h.kernel_launches
        fn(h)
        h.synchronize()
        return h.kernel_launches - before

    def host_flow(h):
        h.update_pose_batch([3, 4, 5], [(3.0, 1.0)] * 3, np.stack([T.reshape(12)] * 3))
        for s in (3, 4, 5):
            h.upload_points(pts, slot=s)
        h.run_scans(h.make_descs([3, 4, 5], [len(pts)] * 3, [org] * 3, [0.0] * 3))
        h.get_layers_to_device([3, 5])

    xy = torch.tensor([[3.0, 1.0]] * 3, dtype=torch.float64, device="cuda")
    Td = torch.tensor(np.stack([T.reshape(12)] * 3), device="cuda")
    o = torch.tensor(np.array([org] * 3, np.float32), device="cuda")
    bz = torch.zeros(3, dtype=torch.float64, device="cuda")
    assert delta(g, lambda h: h.update_poses_from_device([0, 1, 2], xy, Td, o, bz)) == 2 * 3   # 2 groups: resolve + roll
    assert delta(g, lambda h: h.update_poses_from_device([0, 1, 2], origins=o, base_z=bz)) == 2   # resolve only

    def device_scans(h):
        for s in (0, 1, 2):
            h.upload_points(pts, slot=s)
        h.run_scans(h.make_descs([0, 1, 2], [len(pts)] * 3, "device", None))

    assert delta(g, device_scans) == 2 * (1 + 8)   # k_stage_poses + the pipeline per group
    assert delta(g, host_flow) == delta(fresh, host_flow) == 2 * 2 + 2 * 8 + 2   # slot 3 shares a group with device slot 2
    g.profile_enable(True)
    device_scans(g)
    prof = g.profile_read()
    assert prof["k_stage_poses"][1] == 2 and prof["k_rasterize"][1] == 2

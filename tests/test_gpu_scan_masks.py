"""Scan masks from caller GPU memory (gg_set_scan_masks_from_device + GG_SCAN_DEVICE_MASK): a skipped scan leaves its
map untouched.  Handle A runs masked, flagged calls over every slot; its twin B runs the same sequence with the skipped
slots simply left out of each call.  Both must agree bit for bit (NaN-aware): every layer, the positions, the scanned
slots' outputs, and for a skipped slot a zero count, output buffers that come back byte-unchanged, and an empty last
scan (last_scan_points 0, no tallies, no point info, an empty get_output)."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from oracle import Oracle
from test_gpu_device_outputs import DEAD, make_pair, to_device, torch_mod
from test_gpu_device_poses import pose_steps
from test_gpu_spiral_layouts import dim_of, layout_id

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
NAMES = ("ground", "groundpatch", "variance", "minGroundHeight", "count", "obstacles")   # every layer by its fixed name
MSG32 = (32, (0, 4, 8, 16, 20))   # PointXYZIR records as a PointCloud2 payload in the map frame
POISON = 0xA5


def with_outliers(pts, rng):
    """The scan with 40 of its points pushed 3 m under the terrain (below-ground outliers) and kept in padded records."""
    out = pts.copy()
    k = rng.choice(len(out), min(40, len(out)), replace=False)
    out["z"][k] -= 3.0
    return out


def mask_steps(pattern, B, steps, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(steps):
        if pattern == "on":
            m = np.ones(B, np.int32)
        elif pattern == "off":
            m = np.zeros(B, np.int32)
        elif pattern == "alternating":
            m = ((np.arange(B) + k) % 2).astype(np.int32)
        else:
            m = rng.integers(0, 2, B).astype(np.int32)
        out.append(m)
    return out


def set_masks(h, slots, mask, stream=None):
    torch = torch_mod()
    # nonzero values other than 1 scan as well
    h.set_scan_masks_from_device(slots, torch.tensor(np.where(mask != 0, np.arange(1, len(mask) + 1) * 7, 0), dtype=torch.int32, device="cuda"),
                                 stream=stream)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def assert_maps_equal(a, b, slots, names, ctx):
    for s in slots:
        s = int(s)
        for name in names:
            assert np.array_equal(bits(a.layer(name, slot=s)), bits(b.layer(name, slot=s))), f"{ctx} slot {s}: {name}"
        assert a.position(slot=s).tobytes() == b.position(slot=s).tobytes(), f"{ctx} slot {s}: position"


class Outs:
    """Poisoned output buffers of one masked call: labels / index / cloud per scan at capacity, and dev_counts."""

    def __init__(self, torch, caps):
        self.labels = [torch.full((max(c, 1),), POISON, dtype=torch.uint8, device="cuda") for c in caps]
        self.index = [torch.full((max(c, 1),), -5, dtype=torch.int32, device="cuda") for c in caps]
        self.cloud = [torch.full((max(c, 1) * 32,), POISON, dtype=torch.uint8, device="cuda") for c in caps]
        self.counts = torch.full((len(caps),), -9, dtype=torch.int32, device="cuda")
        self.ptrs = np.array([[l.data_ptr(), i.data_ptr(), c.data_ptr()] for l, i, c in zip(self.labels, self.index, self.cloud)], np.uint64)


def check_outputs(torch, outs, twin_out, mask, us, ctx):
    """Scanned scans equal the twin's; skipped ones count 0 and leave their buffers byte-unchanged."""
    torch.cuda.synchronize()
    counts = outs.counts.cpu().numpy()
    j = 0
    tc, ti = twin_out.trimmed() if twin_out is not None else ([], [])
    for k, on in enumerate(mask):
        if not on:
            assert counts[k] == 0, f"{ctx} scan {k}: dev_counts of a skipped scan"
            assert bool((outs.labels[k] == POISON).all()) and bool((outs.index[k] == -5).all()) and bool((outs.cloud[k] == POISON).all()), \
                f"{ctx} scan {k}: a skipped scan wrote its outputs"
            continue
        n = int(twin_out.counts[j])
        assert counts[k] == n, f"{ctx} scan {k}: dev_counts"
        u = us[k]
        assert torch.equal(outs.labels[k][:u], twin_out.labels[j][:u]), f"{ctx} scan {k}: labels"
        assert torch.equal(outs.index[k][:n], ti[j]), f"{ctx} scan {k}: index"
        assert torch.equal(outs.cloud[k][:n * 32], tc[j].reshape(-1).view(torch.uint8)), f"{ctx} scan {k}: cloud"
        j += 1


def check_last_scans(torch, a, b, slots, mask, us, ctx, tallies=True):
    """last_scan_points, get_output, point info and tallies: the twin's for scanned slots, empty for skipped ones."""
    on = [int(s) for s, m in zip(slots, mask) if m]
    ta = a.eval_counts_to_device([int(s) for s in slots]) if tallies else None
    tb = b.eval_counts_to_device(on) if tallies and on else None
    pa = a.point_info_to_device([int(s) for s in slots]) if tallies else None
    pb = b.point_info_to_device(on) if tallies and on else None
    torch.cuda.synchronize()
    j = 0
    for k, (s, m) in enumerate(zip(slots, mask)):
        s = int(s)
        if not m:
            assert a.last_scan_points(slot=s) == 0, f"{ctx} slot {s}: last_scan_points after a skip"
            if tallies:
                assert int(ta[k].abs().sum()) == 0, f"{ctx} slot {s}: tallies of a skipped scan"
                assert pa[0][k].numel() == 0 and pa[1][k].numel() == 0, f"{ctx} slot {s}: point info of a skipped scan"
                idx, cl = a.get_output(slot=s, want_cloud=True)
                assert len(idx) == 0 and len(cl) == 0, f"{ctx} slot {s}: get_output of a skipped scan"
            continue
        assert a.last_scan_points(slot=s) == us[k] == b.last_scan_points(slot=s), f"{ctx} slot {s}: last_scan_points"
        if tallies:
            assert torch.equal(ta[k], tb[j]), f"{ctx} slot {s}: tallies"
            assert torch.equal(pa[0][k], pb[0][j]) and torch.equal(pa[1][k].view(torch.int32), pb[1][j].view(torch.int32)), f"{ctx} slot {s}: point info"
            ia, ca = a.get_output(slot=s, want_cloud=True)
            ib, cb = b.get_output(slot=s, want_cloud=True)
            assert np.array_equal(ia, ib) and ca.tobytes() == cb.tobytes(), f"{ctx} slot {s}: get_output"
        j += 1


def two_parts(cloud):
    """A scan split into a front and a back part, each 32-byte records in the map frame."""
    h = len(cloud) // 3
    return [cloud[:h], cloud[h:]]


# route, stop_after, GG_SCAN_DEVICE_COUNT, GG_SCAN_DEVICE_POSE, full layers
CASES = [
    ("device", 0, True, True, False),
    ("device", 0, False, False, True),
    ("device", 1, True, False, False),
    ("device", 2, False, True, True),
    ("to_device", 0, False, False, True),
    ("to_device", 0, True, True, False),
    ("msgs", 0, True, False, False),
    ("msgs", 0, False, True, True),
    ("merged", 0, True, True, True),
    ("merged", 0, False, False, False),
]
PATTERNS = ["on", "off", "alternating", "random"]


def case_id(c):
    route, stop, cnt, pose, full = c
    return f"{route}-stop{stop}" + ("-count" if cnt else "") + ("-pose" if pose else "") + ("-full" if full else "")


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_masked_batches_match_the_twin_that_leaves_skipped_slots_out(case, pattern):
    """10 steps with rolls, yaw and outliers; the slots in reverse order over every stream group."""
    route, stop, dev_count, dev_pose, full = case
    torch = torch_mod()
    B, STEPS = 6, 10
    a, b = make_pair(60.0, 0.33, B, full_layers=full, max_points=40000)
    names = NAMES + (DEAD if full else ())
    rng = np.random.default_rng(CASES.index(case) * 10 + PATTERNS.index(pattern))
    steps = pose_steps(B, STEPS, jump=0.0, seed=7300)
    masks = mask_steps(pattern, B, STEPS, seed=CASES.index(case))
    slots = np.arange(B, dtype=np.int32)[::-1].copy()
    for k in range(STEPS):
        row = [steps[k][s] for s in slots]
        for h in (a, b):
            if k == 0:
                for s, r in zip(slots, row):
                    h.init_map(r[2][0], r[2][1], 0.0, slot=int(s))
            else:
                h.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))
        mask = masks[k]
        on = np.flatnonzero(mask)
        clouds = [with_outliers(r[0], rng) for r in row]
        caps = [len(c) for c in clouds]
        us = [c * 3 // 4 for c in caps] if dev_count else caps
        origins, bz = [r[1] for r in row], [r[4] for r in row]
        if dev_pose:
            for h in (a, b):
                h.update_poses_from_device(slots, origins=torch.tensor(np.array(origins, np.float32), device="cuda"),
                                           base_z=torch.tensor(np.array(bz, np.float64), device="cuda"))
        org = "device" if dev_pose else origins
        if dev_count:
            cnt = torch.tensor(us, dtype=torch.int32, device="cuda")
            if route == "merged":
                # each part runs on its own first u_p records: u_p = 3/4 of the part, the scan on their sum
                parts_u = np.array([[len(p) * 3 // 4 for p in two_parts(c)] for c in clouds], np.int32)
                us = [int(x) for x in parts_u.sum(axis=1)]
                pc = torch.tensor(parts_u, device="cuda")
                a.set_part_counts_from_device(slots, pc)
                b.set_part_counts_from_device(slots, pc)
            else:
                a.set_point_counts_from_device(slots, cnt)
                b.set_point_counts_from_device(slots, cnt)
        set_masks(a, slots, mask)
        ctx = f"{case_id(case)} {pattern} step {k}"
        sub = lambda xs: [xs[i] for i in on]   # noqa: E731
        bo = None if dev_pose else np.array(origins)
        if route == "device":
            dev = [to_device(c) for c in clouds]
            a.run_scans_device(a.make_descs(slots, caps, org, bz), [t.data_ptr() for t in dev], stop_after=stop, device_counts=dev_count,
                               device_masks=True)
            if len(on):
                b.run_scans_device(b.make_descs(slots[on], sub(caps), "device" if dev_pose else sub(origins), sub(bz)),
                                   [dev[i].data_ptr() for i in on], stop_after=stop, device_counts=dev_count)
            assert_maps_equal(a, b, slots, names, ctx)
            check_last_scans(torch, a, b, slots, mask, us, ctx, tallies=stop == 0)
            continue
        outs = Outs(torch, caps)
        st = torch.cuda.current_stream().cuda_stream or None
        if route == "to_device":
            dev = [to_device(c) for c in clouds]
            descs = a._device_descs(slots, caps, org, bz, dev_count, True)
            a.run_scans_to_device_ptrs(descs, [t.data_ptr() for t in dev], outs.ptrs, capi.SELECT["all"], outs.counts.data_ptr(), st)
            tw = b.run_scans_to_device(sub(dev), slots[on], org if dev_pose else bo[on], np.array(bz)[on], select="all", index=True,
                                       device_counts=dev_count) if len(on) else None
        elif route == "msgs":
            dev = [to_device(c).view(torch.uint8) for c in clouds]
            descs = a._device_descs(slots, caps, org, bz, dev_count, True)
            a.run_cloud_msgs_to_device_ptrs(descs, [t.data_ptr() for t in dev], MSG32[0], MSG32[1], None, outs.ptrs, capi.SELECT["all"],
                                            outs.counts.data_ptr(), st)
            tw = b.run_cloud_msgs_to_device(sub(dev), MSG32[0], MSG32[1], None, slots[on], org if dev_pose else bo[on], np.array(bz)[on],
                                            select="all", index=True, device_counts=dev_count) if len(on) else None
        else:
            # device part counts: both parts at capacity, the stored counts pick the first u records of the scan
            parts = [[to_device(p).view(torch.uint8) for p in two_parts(c)] for c in clouds]
            if dev_count:
                ta = a.run_merged_cloud_msgs_to_device(parts, MSG32[0], MSG32[1], None, slots, org, bz, select="all", index=True,
                                                       device_counts=True, device_masks=True)
            else:
                ta = a.run_merged_cloud_msgs_to_device(parts, MSG32[0], MSG32[1], None, slots, org, bz, select="all", index=True,
                                                       device_masks=True)
            tw = b.run_merged_cloud_msgs_to_device(sub(parts), MSG32[0], MSG32[1], None, slots[on], org if dev_pose else bo[on],
                                                   np.array(bz)[on], select="all", index=True, device_counts=dev_count) if len(on) else None
            # the merged route's outputs are the binding's own: a skipped scan counts 0, the scanned ones equal the twin's
            torch.cuda.synchronize()
            outs.counts.copy_(ta.counts)
            ac, ai = ta.trimmed()
            for k2 in range(B):
                if mask[k2]:
                    outs.labels[k2][:caps[k2]].copy_(ta.labels[k2])
                    outs.index[k2][:len(ai[k2])].copy_(ai[k2])
                    outs.cloud[k2][:len(ac[k2]) * 32].copy_(ac[k2].reshape(-1).view(torch.uint8))
                else:
                    assert len(ai[k2]) == 0 and len(ac[k2]) == 0, f"{ctx} scan {k2}: output of a skipped merged scan"
        check_outputs(torch, outs, tw, mask, us, ctx)
        assert_maps_equal(a, b, slots, names, ctx)
        check_last_scans(torch, a, b, slots, mask, us, ctx)


@pytest.mark.parametrize("n", [12, 300, 468, 1200, 1600], ids=layout_id)
def test_every_spiral_path(n):
    """Alternating masks over three slots on every spiral path (pipe, skew one and two phases, pipe 1024, plain)."""
    B = 3
    a, b = (capi.GroundGridB200(dim_of(n), 0.33, n_slots=B, max_points=20000) for _ in range(2))
    scene = synth.make_scene(seed=n, stream_len=10.0, undulation=0.2)
    slots = np.arange(B, dtype=np.int32)
    for h in (a, b):
        for s in range(B):
            h.init_map(0.0, 0.0, 0.0, slot=s)
    for k in range(4):
        pts, org = synth.lidar_scan(scene, ego_xy=(0.4 * k, 0.0), yaw=0.05 * k, beams=16, az_steps=512, seed=n + k)
        pts = pts[:20000]
        dev = to_device(pts)
        mask = ((np.arange(B) + k) % 2).astype(np.int32)
        set_masks(a, slots, mask)
        a.run_scans_device(a.make_descs(slots, [len(pts)] * B, [org] * B, [0.1] * B), [dev.data_ptr()] * B, device_masks=True)
        on = slots[mask != 0]
        b.run_scans_device(b.make_descs(on, [len(pts)] * len(on), [org] * len(on), [0.1] * len(on)), [dev.data_ptr()] * len(on))
        assert_maps_equal(a, b, slots, NAMES, f"N {n} step {k}")


def test_slot_zero_follows_the_oracle_that_scans_only_when_its_mask_is_on():
    """Slot 0 against the oracle, which rolls every step and scans only when the mask is on.  The rolled prior ("ground",
    "groundpatch") is compared after every step.  The per-scan layers are compared after the steps that scan; after a
    skipped step they must hold exactly what the slot's last scan left.  (A roll moves only the prior here: the
    reference's map move also shifts the per-scan layers, which its next scan overwrites before reading them.)"""
    B = 2
    g = capi.GroundGridB200(60.0, 0.33, n_slots=B, max_points=40000)
    o = Oracle(60.0, 0.33)
    steps = pose_steps(B, 8, jump=0.0, seed=7400)
    pattern = [1, 0, 0, 1, 1, 0, 1, 0]
    slots = np.arange(B, dtype=np.int32)
    last_scan = {}
    for k, row in enumerate(steps):
        if k == 0:
            for s in range(B):
                g.init_map(row[s][2][0], row[s][2][1], 0.0, slot=s)
            o.init_map(row[0][2][0], row[0][2][1], 0.0)
        else:
            g.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))
            o.update(row[0][2][0], row[0][2][1], row[0][3])
        mask = np.array([pattern[k], 1], np.int32)
        set_masks(g, slots, mask)
        dev = [to_device(r[0]) for r in row]
        out = g.run_scans_to_device(dev, slots, [r[1] for r in row], [r[4] for r in row], select="all", device_masks=True)
        if pattern[k]:
            want, _, _ = o.filter_cloud(row[0][0], row[0][1], row[0][4], threads=1)
            assert np.array_equal(out.labels[0].cpu().numpy(), want), f"step {k}: labels"
        else:
            torch_mod().cuda.synchronize()
            assert int(out.counts[0]) == 0
        for name in ("ground", "groundpatch"):
            assert np.array_equal(bits(g.layer(name, slot=0)), bits(o.layer(name))), f"step {k}: {name}"
        for name in ("variance", "minGroundHeight", "points"):
            if pattern[k]:
                assert np.array_equal(bits(g.layer(name, slot=0)), bits(o.layer(name))), f"step {k}: {name}"
                last_scan[name] = g.layer(name, slot=0).copy()
            else:
                assert np.array_equal(bits(g.layer(name, slot=0)), bits(last_scan[name])), f"step {k}: {name} changed by a skipped scan"


def test_a_skipped_scan_is_not_an_empty_scan():
    """After one step, a count-0 scan decays groundpatch; a skipped scan leaves it as it was."""
    torch = torch_mod()
    g = capi.GroundGridB200(60.0, 0.33, n_slots=2, max_points=40000)
    scene = synth.make_scene(seed=3, stream_len=10.0, undulation=0.2)
    pts, org = synth.lidar_scan(scene, beams=32, az_steps=512, seed=3)
    slots = np.arange(2, dtype=np.int32)
    for s in range(2):
        g.init_map(0.0, 0.0, 0.0, slot=s)
    dev = to_device(pts)
    g.run_scans_device(g.make_descs(slots, [len(pts)] * 2, [org] * 2, [0.0] * 2), [dev.data_ptr()] * 2)
    before = [g.layer("groundpatch", slot=s).copy() for s in range(2)]
    g.set_point_counts_from_device(slots, torch.tensor([0, len(pts)], dtype=torch.int32, device="cuda"))
    set_masks(g, slots, np.array([1, 0], np.int32))
    g.run_scans_device(g.make_descs(slots, [len(pts)] * 2, [org] * 2, [0.0] * 2), [dev.data_ptr()] * 2, device_counts=True, device_masks=True)
    assert not np.array_equal(bits(g.layer("groundpatch", slot=0)), bits(before[0])), "a count-0 scan must run the spiral"
    assert np.array_equal(bits(g.layer("groundpatch", slot=1)), bits(before[1])), "a skipped scan must leave the map alone"
    assert g.last_scan_points(slot=0) == 0 == g.last_scan_points(slot=1)


def test_state_rules_and_rejections():
    torch = torch_mod()
    B = 3
    g = capi.GroundGridB200(40.0, 0.33, n_slots=B, max_points=4096)
    L = g._l
    slots = np.arange(B, dtype=np.int32)
    for s in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=s)
    pts, org = synth.lidar_scan(synth.make_scene(seed=5), beams=8, az_steps=256, seed=5)
    pts = pts[:4096]
    dev = to_device(pts)
    descs = lambda sl: g.make_descs(sl, [len(pts)] * len(sl), [org] * len(sl), [0.0] * len(sl))   # noqa: E731
    ptrs = lambda sl: [dev.data_ptr()] * len(sl)   # noqa: E731

    def expect(code, fn):
        before = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            fn()
        assert e.value.code == code, str(e.value)
        assert g.kernel_launches == before

    expect(STATE, lambda: g.run_scans_device(descs(slots), ptrs(slots), device_masks=True))   # nothing stored yet
    m = torch.ones(B, dtype=torch.int32, device="cuda")
    sl = np.ascontiguousarray(slots)
    st = torch.cuda.current_stream().cuda_stream or None
    before = g.kernel_launches
    raw = lambda count, s_, p_: L.gg_set_scan_masks_from_device(g._h, count, s_, p_, st)   # noqa: E731
    for rc, ctx in ((raw(1, None, m.data_ptr()), "null slots"), (raw(1, capi._ptr(sl), None), "null mask"),
                    (raw(1, capi._ptr(sl), m.data_ptr() + 2), "misaligned"), (raw(B + 1, capi._ptr(np.arange(B + 1, dtype=np.int32)), m.data_ptr()), "count"),
                    (raw(2, capi._ptr(np.array([1, 1], np.int32)), m.data_ptr()), "repeated"),
                    (raw(1, capi._ptr(np.array([B], np.int32)), m.data_ptr()), "out of range"),
                    (raw(1, capi._ptr(sl), g.layer_device_ptr("ground", slot=0)), "over the layers"),
                    (L.gg_set_scan_masks_from_device(None, 1, capi._ptr(sl), m.data_ptr(), st), "null handle")):
        assert rc == ARG, ctx
    assert g.kernel_launches == before
    g.set_scan_masks_from_device(slots, m)
    # the host-label paths reject the flag
    d = descs(slots)
    for x in d:
        x.flags |= capi.SCAN_DEVICE_MASK
    expect(ARG, lambda: g.run_scans(d))
    lp = [torch.zeros(len(pts), dtype=torch.uint8, device="cuda") for _ in range(B)]
    expect(ARG, lambda: g.filter_cloud_batch_ptrs(d, [pts.ctypes.data] * B, [t.data_ptr() for t in lp]))
    g.run_scans_device(descs(slots), ptrs(slots), device_masks=True)
    # init_maps_from_device and restore keep the stored mask; init_map forgets it
    g.init_maps_from_device(slots, torch.zeros((B, 3), dtype=torch.float64, device="cuda"))
    pool = g.save_maps_to_device(slots)
    g.restore_maps_from_device(slots, pool)
    g.run_scans_device(descs(slots), ptrs(slots), device_masks=True)
    g.init_map(0.0, 0.0, 0.0, slot=1)
    expect(STATE, lambda: g.run_scans_device(descs(slots), ptrs(slots), device_masks=True))
    g.run_scans_device(descs(slots[[0, 2]]), ptrs([0, 2]), device_masks=True)
    g.synchronize()


def test_stream_contract_with_the_mask_overwritten_right_after_the_call():
    torch = torch_mod()
    B = 4
    a, b = make_pair(40.0, 0.33, B, max_points=20000)
    slots = np.arange(B, dtype=np.int32)
    for h in (a, b):
        for s in range(B):
            h.init_map(0.0, 0.0, 0.0, slot=s)
    pts, org = synth.lidar_scan(synth.make_scene(seed=9), beams=16, az_steps=512, seed=9)
    pts = pts[:20000]
    dev = to_device(pts)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        m = torch.tensor([1, 0, 1, 0], dtype=torch.int32, device="cuda")
        torch.cuda._sleep(20_000_000)   # the call's kernels queue behind this
        a.set_scan_masks_from_device(slots, m, stream=side)
        m.fill_(0)                     # a refill on the stream right after the call
    a.run_scans_device(a.make_descs(slots, [len(pts)] * B, [org] * B, [0.0] * B), [dev.data_ptr()] * B, device_masks=True)
    on = slots[[0, 2]]
    b.run_scans_device(b.make_descs(on, [len(pts)] * 2, [org] * 2, [0.0] * 2), [dev.data_ptr()] * 2)
    assert_maps_equal(a, b, slots, NAMES, "stream")


def plan_inputs(torch, B, caps):
    return dict(clouds=[torch.zeros((c, 8), dtype=torch.float32, device="cuda") for c in caps],
                counts=torch.zeros(B, dtype=torch.int32, device="cuda"), xy=torch.zeros((B, 2), dtype=torch.float64, device="cuda"),
                T=torch.zeros((B, 12), dtype=torch.float64, device="cuda"), org=torch.zeros((B, 3), dtype=torch.float32, device="cuda"),
                bz=torch.zeros(B, dtype=torch.float64, device="cuda"), mask=torch.zeros(B, dtype=torch.int32, device="cuda"))


def write_step(torch, inp, row, us, mask):
    for c, r, u in zip(inp["clouds"], row, us):
        c.zero_()
        c[:u].copy_(to_device(r[0][:u]).view(torch.float32).reshape(u, 8))
    inp["counts"].copy_(torch.tensor(us, dtype=torch.int32))
    inp["xy"].copy_(torch.tensor(np.array([r[2] for r in row]), dtype=torch.float64))
    inp["T"].copy_(torch.tensor(np.stack([r[3].reshape(12) for r in row]), dtype=torch.float64))
    inp["org"].copy_(torch.tensor(np.array([r[1] for r in row], np.float32)))
    inp["bz"].copy_(torch.tensor([r[4] for r in row], dtype=torch.float64))
    inp["mask"].copy_(torch.tensor(mask, dtype=torch.int32))


def twin_step(torch, b, inp, slots, mask, tallies):
    """The plan's call sequence on the twin, with the skipped slots left out of the scan and the tallies."""
    b.set_point_counts_from_device(slots, inp["counts"])
    b.update_poses_from_device(slots, xy=inp["xy"], T=inp["T"], origins=inp["org"], base_z=inp["bz"])
    on = slots[np.asarray(mask) != 0]
    if len(on):
        b.run_scans_to_device([inp["clouds"][s] for s in on], on, "device", None, select="all", index=True, device_counts=True)
        t = b.eval_counts_to_device(on)
        tallies[torch.tensor(on, device="cuda")] += t


@pytest.mark.parametrize("graph", [False, True], ids=["launch", "torch_graph"])
def test_plan_with_the_mask_rewritten_between_replays(graph):
    """A plan with resets (mask all zero), configs, snapshots and tallies: each replay equals the twin's sequence, and
    the tallies grow only by the scanned slots."""
    torch = torch_mod()
    B, STEPS = 8, 8
    a, b = make_pair(60.0, 0.33, B, max_points=40000)
    steps = pose_steps(B, STEPS + 1, jump=0.0, seed=7500)
    slots = np.arange(B, dtype=np.int32)
    for h in (a, b):
        for s in range(B):
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    caps = [max(len(steps[k][s][0]) for k in range(STEPS + 1)) for s in range(B)]
    inp = plan_inputs(torch, B, caps)
    reset_xyz = torch.zeros((B, 3), dtype=torch.float64, device="cuda")
    reset_mask = torch.zeros(B, dtype=torch.int32, device="cuda")
    cfgs = capi.config_tensor([a.get_config(slot=s) for s in range(B)])
    ta = torch.zeros((B, 1024, 2), dtype=torch.int64, device="cuda")
    tb = torch.zeros_like(ta)
    plan = a.step_plan(slots, clouds=inp["clouds"], counts=inp["counts"], xy=inp["xy"], T_base_from_map=inp["T"], pose_origins=inp["org"],
                       pose_base_z=inp["bz"], select="all", index=True, reset_xyz=reset_xyz, reset_mask=reset_mask, configs=cfgs,
                       save=True, tallies=ta, scan_mask=inp["mask"])
    b.set_configs_from_device(slots, cfgs)
    tg = None
    if graph:
        tg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(tg):
            plan.launch()
    masks = mask_steps("random", B, STEPS, seed=11)
    masks[0][:] = 1
    for k in range(1, STEPS + 1):
        row = steps[k]
        us = [len(r[0]) * 4 // 5 for r in row]
        mask = masks[k - 1]
        write_step(torch, inp, row, us, mask)
        (tg.replay() if graph else plan.launch())
        twin_step(torch, b, inp, slots, mask, tb)
        torch.cuda.synchronize()
        ctx = f"plan step {k}"
        assert torch.equal(ta, tb), f"{ctx}: tallies"
        outs = plan.outputs
        counts = outs.counts.cpu().numpy()
        assert all(counts[s] == 0 for s in range(B) if not mask[s]), f"{ctx}: counts of skipped scans"
        assert_maps_equal(a, b, slots, NAMES, ctx)
    plan.close()


def test_standalone_masks_reach_a_plan_and_the_stage_costs_one_kernel_per_group(monkeypatch):
    """The mask stage adds one kernel per stream group.  A plan without the stage whose scans are flagged reads the masks
    that standalone calls store on its bound slots before each replay."""
    torch = torch_mod()
    B = 8
    a, b = make_pair(60.0, 0.33, B, max_points=40000)
    steps = pose_steps(B, 4, jump=0.0, seed=7600)
    slots = np.arange(B, dtype=np.int32)
    for h in (a, b):
        for s in range(B):
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    caps = [max(len(steps[k][s][0]) for k in range(4)) for s in range(B)]
    inp = plan_inputs(torch, B, caps)
    kw = dict(clouds=inp["clouds"], counts=inp["counts"], xy=inp["xy"], T_base_from_map=inp["T"], pose_origins=inp["org"],
              pose_base_z=inp["bz"], select="all", save=True)
    p0 = a.step_plan(slots, **kw)
    k0 = p0.kernels
    p0.close()
    p1 = a.step_plan(slots, scan_mask=inp["mask"], **kw)
    groups = len({s * a.n_streams // B for s in range(B)})
    assert p1.kernels == k0 + groups
    p1.close()
    # a plan without the stage whose scans are flagged: masks come from standalone calls, also on the bound slots
    inp["mask"].fill_(1)
    a.set_scan_masks_from_device(slots, inp["mask"])
    # step_plan flags the scans only with a mask stage: flag them here, for a plan without one
    descs = capi.GroundGridB200._device_descs
    monkeypatch.setattr(capi.GroundGridB200, "_device_descs", staticmethod(lambda sl, n, o, bz, dc=False, dm=False: descs(sl, n, o, bz, dc, True)))
    plan = a.step_plan(slots, **kw)
    monkeypatch.undo()
    assert plan.kernels == k0
    tb = torch.zeros((B, 1024, 2), dtype=torch.int64, device="cuda")
    for k in range(1, 4):
        row = steps[k]
        us = [len(r[0]) * 4 // 5 for r in row]
        mask = ((np.arange(B) + k) % 3 != 0).astype(np.int32)
        write_step(torch, inp, row, us, mask)
        a.set_scan_masks_from_device(slots, inp["mask"])   # accepted on bound slots
        plan.launch()
        twin_step(torch, b, inp, slots, mask, tb)
        torch.cuda.synchronize()
        assert_maps_equal(a, b, slots, NAMES, f"standalone masks step {k}")
        assert all(int(plan.outputs.counts[s]) == 0 for s in range(B) if not mask[s])
    plan.close()

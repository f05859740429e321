"""Step plans (gg_step_plan_create / gg_step_plan_launch): a batch's counts, roll and scans recorded once as a CUDA graph
and replayed from caller GPU memory.  Every case runs against a twin handle that makes the literal call sequence --
gg_set_point_counts_from_device, gg_update_poses_from_device, gg_run_scans_to_device / gg_run_cloud_msgs_to_device --
on the same tensors, and must be bit-identical to it: labels, index, cloud, dev_counts, dev_moved every step; layers,
positions, gg_get_output, point info, tallies and gg_last_scan_points at the end.  Records past each scan's count are
poison (test_gpu_device_counts), so a read past the count shows."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi
from oracle import Oracle, nextrows
from test_gpu_cloud_msgs import map_from_sensor, payload
from test_gpu_device_counts import MAX_POINTS, assert_twin, with_poison
from test_gpu_device_outputs import make_pair, torch_mod
from test_gpu_device_poses import pose_steps

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
B, STEPS, GROUPS = 8, 24, 3
PLAN_SLOTS = ([7, 0, 3, 5], [1, 2, 4, 6])      # each plan spans the three stream groups (slot * 3 // 8)
PLAN_SELECTS = ("all", "nonground")
CAPS = [MAX_POINTS, 12000, 20000, MAX_POINTS, 9000, 30000, MAX_POINTS, 15000]   # fixed per slot: the buffers are the plan's
MSG32 = (32, (0, 4, 8, 16, 20))   # PointXYZIR records as a PointCloud2 payload in the map frame
MSG18 = (18, (0, 4, 8, 12, 16))   # the KITTI player's 18-byte points, in a sensor frame


def handles(monkeypatch):
    monkeypatch.setenv("GG_STREAMS", str(GROUPS))
    g, twin = make_pair(99.0, 0.33, B, max_points=MAX_POINTS)
    assert g.n_streams == GROUPS == twin.n_streams
    return g, twin


def count_of(kind, m, cap):
    """u per capacity kind: u == capacity (the whole buffer, poison included), u < capacity, u == 0, capacity - 17."""
    return [cap, min(m, cap) * 2 // 3, 0, min(m, cap) - 17][kind]


class Inputs:
    """The fixed CUDA tensors of one plan: clouds or payloads at capacity, counts, poses and (msgs18) transforms."""

    def __init__(self, torch, slots, route):
        self.slots = slots
        self.route = route
        n = len(slots)
        self.step = 32 if route == "records" else (MSG32 if route == "msgs32" else MSG18)[0]
        self.offs = (MSG32 if route != "msgs18" else MSG18)[1]
        self.buf = [torch.zeros(CAPS[s] * self.step, dtype=torch.uint8, device="cuda") for s in slots]
        self.counts = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.xy = torch.zeros((n, 2), dtype=torch.float64, device="cuda")
        self.T = torch.zeros((n, 12), dtype=torch.float64, device="cuda")
        self.origins = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
        self.base_z = torch.zeros(n, dtype=torch.float64, device="cuda")
        self.Tmap = torch.zeros((n, 12), dtype=torch.float64, device="cuda") if route == "msgs18" else None
        self.Thost = [None] * n

    def plan(self, g, select):
        kw = dict(counts=self.counts, xy=self.xy, T_base_from_map=self.T, pose_origins=self.origins, pose_base_z=self.base_z, moved=True,
                  labels=True, select=select, index=True)
        if self.route == "records":
            return g.step_plan(self.slots, clouds=self.buf, **kw)
        return g.step_plan(self.slots, payloads=self.buf, point_step=self.step, field_offsets=self.offs,
                           T=None if self.Tmap is None else list(self.Tmap), **kw)

    def write(self, torch, row, xy, rng, kinds):
        """The next step's inputs, written into the tensors on the current stream.  Returns (us, raw) per scan."""
        us, raws = [], []
        for j, s in enumerate(self.slots):
            pts, cap = row[s][0], CAPS[s]
            u = count_of(kinds[j], len(pts), cap)
            cloud = with_poison(pts, min(len(pts), cap), cap, rng)
            if self.route == "msgs18":
                self.Thost[j] = map_from_sensor(row[s][2], 0.2 * s + 0.01 * len(us))
                raw = payload(cloud, self.step, self.offs, self.Thost[j], rng)
            elif self.route == "msgs32":
                raw = payload(cloud, self.step, self.offs, None, rng)
            else:
                raw = np.ascontiguousarray(cloud).view(np.uint8)
            self.buf[j].copy_(torch.from_numpy(np.ascontiguousarray(raw).reshape(-1)))
            us.append(u)
            raws.append(raw)
        self.counts.copy_(torch.tensor(us, dtype=torch.int32))
        self.xy.copy_(torch.tensor(np.array([xy[s] for s in self.slots], np.float64)))
        self.T.copy_(torch.tensor(np.stack([row[s][3].reshape(12) for s in self.slots])))
        self.origins.copy_(torch.tensor(np.array([row[s][1] for s in self.slots], np.float32)))
        self.base_z.copy_(torch.tensor(np.array([row[s][4] for s in self.slots], np.float64)))
        if self.Tmap is not None:
            self.Tmap.copy_(torch.tensor(np.stack([t.reshape(12) for t in self.Thost])))
        return us, raws

    def twin_step(self, twin, select, stream=None):
        """The literal call sequence on the same tensors: (DeviceOutputs, dev_moved)."""
        twin.set_point_counts_from_device(self.slots, self.counts, stream=stream)
        moved = twin.update_poses_from_device(self.slots, self.xy, self.T, self.origins, self.base_z, moved=True, stream=stream)
        kw = dict(labels=True, select=select, index=True, stream=stream, device_counts=True)
        if self.route == "records":
            out = twin.run_scans_to_device(self.buf, self.slots, "device", None, **kw)
        else:
            out = twin.run_cloud_msgs_to_device(self.buf, self.step, self.offs, None if self.Tmap is None else list(self.Thost), self.slots,
                                                "device", None, **kw)
        return out, moved


def check_step(plan, out_t, moved_t, us, ctx):
    torch = torch_mod()
    torch.cuda.synchronize()
    out_g = plan.outputs
    assert torch.equal(plan.moved, moved_t), f"{ctx}: dev_moved {plan.moved.tolist()} vs {moved_t.tolist()}"
    assert torch.equal(out_g.counts, out_t.counts), f"{ctx}: dev_counts"
    gc, gi = out_g.trimmed()
    tc, ti = out_t.trimmed()
    for k, u in enumerate(us):
        assert torch.equal(out_g.labels[k][:u], out_t.labels[k][:u]), f"{ctx} scan {k}: labels"
        assert torch.equal(gi[k], ti[k]) and torch.equal(gc[k].view(torch.int32), tc[k].view(torch.int32)), f"{ctx} scan {k}: index / cloud"


def assert_positions(g, twin, slots, ctx):
    for s in slots:
        assert g.position(slot=s).view(np.uint64).tolist() == twin.position(slot=s).view(np.uint64).tolist(), f"{ctx} slot {s}: position"


def step_xy(row, k, prev):
    """The rolls of step k: the row's odometry (moves on most steps), the previous position for one slot (a roll that
    does not move) and NaN for another (dev_moved = -1; never slot 0, which the oracle follows)."""
    xy = {s: np.array(row[s][2], np.float64) for s in range(B)}
    if k:
        xy[(k + 1) % B] = prev[(k + 1) % B].copy()
    nan = 1 + (3 * k) % (B - 1)
    if nan == (k + 1) % B:
        nan = 1 + (nan % (B - 1))
    xy[nan] = np.array([np.nan, row[nan][2][1]])
    return xy, nan


@pytest.mark.parametrize("route", ["records", "msgs32", "msgs18"])
def test_rolling_sequence_matches_the_call_sequence(monkeypatch, route):
    """24 steps on 8 slots over 3 stream groups, two plans (select "all" and "nonground"): rolls that move and that do
    not, one non-finite xy per step, every capacity kind with poisoned records past the count; slot 0 is also checked
    against the CPU oracle at three steps."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, STEPS, jump=60.0, seed=6100)
    rng = np.random.default_rng(["records", "msgs32", "msgs18"].index(route))
    o = Oracle(99.0, 0.33)
    for h in (g, twin):
        for s in range(B):
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    o.init_map(steps[0][0][2][0], steps[0][0][2][1], 0.0)
    inputs = [Inputs(torch, list(sl), route) for sl in PLAN_SLOTS]
    plans = [inp.plan(g, sel) for inp, sel in zip(inputs, PLAN_SELECTS)]
    extra = sum(len({s * GROUPS // B for s in sl}) for sl in PLAN_SLOTS) if route == "msgs18" else 0   # k_stage_transforms per branch
    prev = {s: np.array(steps[0][s][2], np.float64) for s in range(B)}
    checked = 0
    for k, row in enumerate(steps):
        xy, nan = step_xy(row, k, prev)
        ctx = f"{route} step {k}"
        written = [inp.write(torch, row, xy, rng, [(s + k) % 4 for s in inp.slots]) for inp in inputs]
        g0, t0 = g.kernel_launches, twin.kernel_launches
        for p in plans:
            p.launch()
        twin_out = [inp.twin_step(twin, sel) for inp, sel in zip(inputs, PLAN_SELECTS)]
        assert g.kernel_launches - g0 == sum(p.kernels for p in plans) == twin.kernel_launches - t0 + extra, ctx
        for p, inp, (us, _), (out_t, moved_t) in zip(plans, inputs, written, twin_out):
            check_step(p, out_t, moved_t, us, ctx)
            if nan in inp.slots:
                assert p.moved[inp.slots.index(nan)].item() == -1, ctx
        # the oracle follows slot 0 (plan 0, scan 1)
        j0 = inputs[0].slots.index(0)
        us0, raws0 = written[0]
        u0 = us0[j0]
        if route == "msgs18":
            pts0 = nextrows.unpack_transform(raws0[j0][:u0], u0, MSG18[0], MSG18[1], inputs[0].Thost[j0])
        else:
            pts0 = nextrows.unpack_transform(np.ascontiguousarray(raws0[j0]).reshape(-1, inputs[0].step)[:u0], u0, inputs[0].step,
                                             inputs[0].offs, None)
        o.update(xy[0][0], xy[0][1], row[0][3])
        ref, _, _ = o.filter_cloud(pts0, row[0][1], row[0][4], threads=1)
        if k in (3, 11, STEPS - 1):
            assert u0 > 0, ctx
            assert np.array_equal(plans[0].outputs.labels[j0][:u0].cpu().numpy(), ref), f"{ctx}: labels differ from the oracle"
            for name in ("ground", "groundpatch"):
                assert np.array_equal(g.layer(name, slot=0).view(np.uint32), o.layer(name).view(np.uint32)), f"{ctx}: {name} vs oracle"
            checked += 1
        prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
    assert checked == 3
    torch.cuda.synchronize()
    slots = [s for sl in PLAN_SLOTS for s in sl]
    us = [u for us_, _ in written for u in us_]
    assert_twin(g, twin, slots, us, [CAPS[s] for s in slots], f"{route} end")
    assert_positions(g, twin, range(B), f"{route} end")
    for p in plans:
        p.close()


def test_plan_inside_a_torch_graph(monkeypatch):
    """plan.launch() captured in torch.cuda.graph, then 10 replays of the torch graph with new inputs written between
    them: each replay equals the twin's call sequence on the same tensors."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 11, jump=0.0, seed=6200)
    rng = np.random.default_rng(21)
    for h in (g, twin):
        for s in range(B):
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    inp = Inputs(torch, list(range(B))[::-1], "records")
    plan = inp.plan(g, "all")
    graph = torch.cuda.CUDAGraph()
    before = g.kernel_launches
    with torch.cuda.graph(graph):
        plan.launch()
    assert g.kernel_launches - before == plan.kernels
    prev = {s: np.array(steps[0][s][2], np.float64) for s in range(B)}
    for k in range(1, 11):
        row = steps[k]
        xy, nan = step_xy(row, k, prev)
        us, _ = inp.write(torch, row, xy, rng, [(s + k) % 4 for s in inp.slots])
        graph.replay()
        out_t, moved_t = inp.twin_step(twin, "all")
        check_step(plan, out_t, moved_t, us, f"replay {k}")
        prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
    torch.cuda.synchronize()   # the captured step has no fences with the handle's streams
    assert_twin(g, twin, inp.slots, us, [CAPS[s] for s in inp.slots], "torch graph")
    assert_positions(g, twin, range(B), "torch graph")
    del graph
    plan.close()


def test_stream_contract(monkeypatch):
    """Inputs made by a torch op on a side stream right before the launch and outputs consumed right after; a sleep
    ahead of the launch shows that gg_step_plan_launch returns before the stream reaches the replay; layer exports and
    terrain lookups of bound slots, and gg_get_output on the slots' own stream groups, interleaved with launches, see the
    right step."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 4, jump=0.0, seed=6300)
    rng = np.random.default_rng(31)
    for h in (g, twin):
        for s in range(B):
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    inp = Inputs(torch, list(range(B)), "records")
    plan = inp.plan(g, "nonground")
    side = torch.cuda.Stream()
    names = ("ground", "groundpatch", "points")
    prev = {s: np.array(steps[0][s][2], np.float64) for s in range(B)}
    for k in range(4):
        row = steps[k]
        xy, _ = step_xy(row, k, prev)
        us, _ = inp.write(torch, row, xy, rng, [(s + k) % 4 for s in inp.slots])
        want = inp.counts.clone()
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(100_000_000)
            inp.counts.copy_((want * 2 + 6) // 2 - 3)      # produced on the side stream just before the launch
        plan.launch(side)
        assert not side.query(), "gg_step_plan_launch waited for the stream"
        with torch.cuda.stream(side):
            labels = [t.clone() for t in plan.outputs.labels]   # consumed right after
            counts = plan.outputs.counts.clone()
            moved = plan.moved.clone()
            pos = [t[:200].clone() for t in plan.outputs.cloud]
        layers = g.get_layers_to_device(inp.slots, names, stream=side)
        samples = g.sample_layers_to_device(inp.slots, pos, names[:2], stream=side)
        s0 = inp.slots[k % B]
        gi, gcl = g.get_output(slot=s0, want_cloud=True)   # the slot's stream group waits for the replay
        side.synchronize()
        out_t, moved_t = inp.twin_step(twin, "nonground")
        t_layers = twin.get_layers_to_device(inp.slots, names)
        t_samples = twin.sample_layers_to_device(inp.slots, pos, names[:2])
        ti, tcl = twin.get_output(slot=s0, want_cloud=True)
        torch.cuda.synchronize()
        ctx = f"step {k}"
        assert np.array_equal(gi, ti) and gcl.tobytes() == tcl.tobytes(), f"{ctx}: get_output"
        assert torch.equal(counts, out_t.counts) and torch.equal(moved, moved_t), ctx
        for j, u in enumerate(us):
            assert torch.equal(labels[j][:u], out_t.labels[j][:u]), f"{ctx} scan {j}: labels"
        assert torch.equal(layers.view(torch.int32), t_layers.view(torch.int32)), f"{ctx}: layers"
        for a, b in zip(samples, t_samples):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"{ctx}: samples"
        prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
    plan.close()


def test_rejections_enqueue_nothing_and_bound_slots(monkeypatch):
    """Each GG_E_ARG / GG_E_STATE of gg_step_plan_create, each GG_E_STATE of a bound slot, a slot bound twice: none
    enqueues anything.  gg_get_map_position of a bound slot returns the device position; gg_kernel_launches grows by the
    plan's kernel count per launch; after destroy the slots accept every call again."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    L = g._l
    steps = pose_steps(B, 2, jump=0.0, seed=6400)
    for h in (g, twin):
        for s in range(B - 1):             # slot B - 1 stays uninitialised
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    rng = np.random.default_rng(41)
    inp = Inputs(torch, [0, 3, 6], "msgs18")
    xy = {s: np.array(steps[1][s][2]) for s in range(B)}
    inp.write(torch, steps[1], xy, rng, [0, 1, 3])
    out, ptrs = g._device_outputs(torch, torch.device("cuda", 0), torch.cuda.current_stream(), [CAPS[s] for s in inp.slots], True, 3, True, [])
    T = torch.zeros((4, 12), dtype=torch.float64, device="cuda")
    g.synchronize()
    before = g.kernel_launches

    def desc(slots=(0, 3, 6), **over):
        n = len(slots)
        descs = g._device_descs(list(slots), [CAPS[s] if s < B else 100 for s in slots], "device", None, True)
        msgs = np.zeros(max(n, 1), capi.CLOUD_MSG_DTYPE)
        msgs["data"][:n] = [b.data_ptr() for b in inp.buf[:n]] if n <= 3 else inp.buf[0].data_ptr()
        msgs["point_step"] = 18
        msgs["field_offsets"] = MSG18[1]
        tp = np.array([T[j % 4].data_ptr() for j in range(max(n, 1))], np.uint64)
        keep = [descs, msgs, tp]
        d = capi.StepDesc()
        d.count = n
        d.scans = descs.ctypes.data
        d.msgs = msgs.ctypes.data
        d.dev_T_map_from_frame = tp.ctypes.data
        d.dev_n_points = inp.counts.data_ptr()
        d.poses = capi.DevicePoses(inp.xy.data_ptr(), inp.T.data_ptr(), inp.origins.data_ptr(), inp.base_z.data_ptr())
        d.outs = ptrs.ctypes.data
        d.select = 3
        d.dev_counts = out.counts.data_ptr()
        for k, v in over.items():
            if callable(v):
                v(d, descs, msgs, tp, keep)
            else:
                setattr(d, k, v)
        return d, keep

    def create(d):
        p = C.c_void_p()
        return L.gg_step_plan_create(g._h, C.byref(d[0]), C.byref(p)), p

    def host_T(d, descs, msgs, tp, keep):
        Th = np.zeros(12, np.float64)
        keep.append(Th)
        msgs["T_map_from_frame"][1] = Th.ctypes.data

    def no_pose(d, descs, msgs, tp, keep):
        d.poses = capi.DevicePoses(None, None, None, None)

    cases = {
        "count 0": (desc(count=0), ARG),
        "count > n_slots": (desc(count=B + 1), ARG),
        "null scans": (desc(scans=None), ARG),
        "null msgs (neither)": (desc(msgs=None), ARG),
        "both dev_points and msgs": (desc(dev_points=inp.buf[0].data_ptr()), ARG),
        "dev_T without msgs": (desc(msgs=None, dev_points=inp.buf[0].data_ptr()), ARG),
        "misaligned dev_T": (desc(fn=lambda d, de, m, tp, k: tp.__setitem__(0, tp[0] + 4)), ARG),
        "overlapping dev_T": (desc(fn=lambda d, de, m, tp, k: tp.__setitem__(1, tp[0] + 48)), ARG),
        "device and host T": (desc(fn=host_T), ARG),
        "repeated slot": (desc(slots=(0, 3, 3)), ARG),
        "slot out of range": (desc(slots=(0, B, 6)), ARG),
        "misaligned dev_n_points": (desc(dev_n_points=inp.counts.data_ptr() + 2), ARG),
        "xy without T": (desc(fn=lambda d, de, m, tp, k: setattr(d, "poses", capi.DevicePoses(inp.xy.data_ptr(), None, None, None))), ARG),
        "unknown select bits": (desc(select=4), ARG),
        "index without dev_counts": (desc(dev_counts=None), ARG),
        "point_step < 12": (desc(fn=lambda d, de, m, tp, k: m.__setitem__("point_step", 8)), ARG),
        "capacity above max_points": (desc(fn=lambda d, de, m, tp, k: de.__setitem__("n_points", MAX_POINTS + 1000)), ARG),
        "map not initialised": (desc(slots=(0, 3, B - 1)), STATE),
        "device pose without step 2": (desc(fn=no_pose), STATE),
    }
    for name, (d, want) in cases.items():
        rc, p = create(d)
        assert rc == want and not p.value, f"{name}: {rc}"
        assert g.kernel_launches == before, name
    # a valid plan, then a slot bound twice
    plan = inp.plan(g, "all")
    assert g.kernel_launches == before
    rc, p = create(desc(slots=(1, 6)))
    assert rc == STATE and not p.value, "slot 6 bound twice"
    other = g.step_plan([1, 2], clouds=[torch.zeros((100, 8), device="cuda"), torch.zeros((100, 8), device="cuda")],
                        origins=[[0, 0, 0]] * 2, base_z=[0.0, 0.0])   # unbound slots may have their own plan
    other.close()
    g.synchronize()
    before = g.kernel_launches
    # the calls a bound slot refuses
    Tb = steps[1][0][3]
    pts = steps[1][0][0]
    sd = g.make_descs([3], [len(pts)], [steps[1][0][1]], [0.0])
    pp = (C.c_void_p * 1)(pts.ctypes.data)
    ticket = C.c_int(-1)
    cfg = g.get_config(slot=3)
    refused = {
        "gg_update_pose": lambda: L.gg_update_pose(g._h, 3, 1.0, 2.0, capi._ptr(np.ascontiguousarray(Tb.reshape(12))), None),
        "gg_update_pose_batch": lambda: L.gg_update_pose_batch(g._h, 2, capi._ptr(np.array([1, 6], np.int32)), capi._ptr(np.zeros(4)),
                                                              capi._ptr(np.zeros(24)), None),
        "gg_set_map_position": lambda: L.gg_set_map_position(g._h, 0, 1.0, 2.0),
        "gg_init_map": lambda: L.gg_init_map(g._h, 6, 0.0, 0.0, 0.0),
        "gg_set_slot_config": lambda: L.gg_set_slot_config(g._h, 3, C.byref(cfg)),
        "gg_set_config": lambda: L.gg_set_config(g._h, C.byref(g.get_config())),
        "gg_filter_cloud": lambda: L.gg_filter_cloud(g._h, 0, capi._ptr(pts), len(pts), capi._ptr(np.zeros(3, np.float32)), 0.0, None, None,
                                                     None, None),
        "gg_filter_cloud_batch": lambda: L.gg_filter_cloud_batch(g._h, 1, sd, pp, None),
        "gg_filter_cloud_batch_begin": lambda: L.gg_filter_cloud_batch_begin(g._h, 1, sd, pp, None, C.byref(ticket)),
    }
    for name, fn in refused.items():
        assert fn() == STATE, name
        assert g.kernel_launches == before, name
    # launches: the plan's kernel count each, and a bound slot's position is the device's and stays device-owned
    for k in range(2):
        plan.launch()
        assert g.kernel_launches == before + (k + 1) * plan.kernels
        out_t, moved_t = inp.twin_step(twin, "all")
    check_step(plan, out_t, moved_t, [count_of(kk, len(steps[1][s][0]), CAPS[s]) for kk, s in zip([0, 1, 3], inp.slots)], "two launches")
    assert_positions(g, twin, inp.slots, "bound")
    assert L.gg_set_map_position(g._h, 0, 1.0, 2.0) == STATE, "get_map_position left the slot host-owned"
    plan.close()
    # after destroy the slots accept the calls again
    g.synchronize()
    assert g.update_pose(steps[1][0][2][0], steps[1][0][2][1], Tb, slot=3) in (True, False)
    g.set_config(slot=3, max_ring=64)
    g.set_config(max_ring=1024)
    g.init_map(0.0, 0.0, 0.0, slot=6)
    g.set_position(5.0, 6.0, slot=0)
    assert g.position(slot=0).tolist() == [5.0, 6.0]
    assert L.gg_filter_cloud_batch(g._h, 1, sd, pp, None) == 0
    plan2 = inp.plan(g, "nonground")   # the slots can be bound again
    plan2.close()
    del T

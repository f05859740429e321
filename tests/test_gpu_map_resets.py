"""Map resets from caller GPU memory (gg_init_maps_from_device, gg_step_plan_create_with_resets): initGroundGrid of the
slots a device mask picks, at device poses.  Every case runs against a twin handle that calls the host gg_init_map for
the masked slots at the same point of the sequence, and must be bit-identical to it: every layer, the map positions,
and the outputs of the scans that follow.  Slots the mask leaves out must come out bit-unchanged."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi
from oracle import Oracle
from test_gpu_device_counts import MAX_POINTS, assert_twin, with_poison
from test_gpu_device_outputs import DEAD, LIVE, make_pair, to_device, torch_mod
from test_gpu_device_poses import pose_steps
from test_gpu_step_plans import CAPS, Inputs, check_step, step_xy

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
B, GROUPS = 8, 3


def handles(monkeypatch, full_layers=False):
    monkeypatch.setenv("GG_STREAMS", str(GROUPS))
    g, twin = make_pair(99.0, 0.33, B, full_layers=full_layers, max_points=MAX_POINTS)
    assert g.n_streams == GROUPS == twin.n_streams
    return g, twin


def reset_poses(rng, centres):
    """Odometry x, y, z per slot near the given centres; z values that round in fp32."""
    c = np.asarray(centres, np.float64).reshape(-1, 2)
    xyz = np.empty((len(c), 3), np.float64)
    xyz[:, :2] = c + rng.uniform(-4.0, 4.0, c.shape)
    xyz[:, 2] = rng.uniform(-3.0, 3.0, len(c)) + 1e-9
    assert np.any(xyz[:, 2] != xyz[:, 2].astype(np.float32).astype(np.float64))
    return xyz


def twin_resets(twin, slots, xyz, mask):
    """The host path the device call must equal: gg_init_map of every masked slot."""
    for k, s in enumerate(slots):
        if mask is None or mask[k]:
            twin.init_map(float(xyz[k][0]), float(xyz[k][1]), float(xyz[k][2]), slot=int(s))


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint64)


def assert_layers(g, twin, slots, names, ctx):
    for s in slots:
        for name in names:
            assert np.array_equal(bits(g.layer(name, slot=int(s))), bits(twin.layer(name, slot=int(s)))), f"{ctx} slot {s}: {name}"


def assert_positions(g, twin, slots, ctx):
    for s in slots:
        assert bits(g.position(slot=int(s))).tolist() == bits(twin.position(slot=int(s))).tolist(), f"{ctx} slot {s}: position"


def same_outputs(out_g, out_t, us, ctx):
    torch = torch_mod()
    torch.cuda.synchronize()
    assert torch.equal(out_g.counts, out_t.counts), f"{ctx}: dev_counts"
    gc, gi = out_g.trimmed()
    tc, ti = out_t.trimmed()
    for k, u in enumerate(us):
        assert torch.equal(out_g.labels[k][:u], out_t.labels[k][:u]), f"{ctx} scan {k}: labels"
        assert torch.equal(gi[k], ti[k]) and torch.equal(gc[k].view(torch.int32), tc[k].view(torch.int32)), f"{ctx} scan {k}: index / cloud"


def device_step(h, slots, row, clouds, counts, stream=None):
    """counts -> device poses (roll and scan pose) -> scans on the device counts and poses."""
    torch = torch_mod()
    h.set_point_counts_from_device(slots, torch.tensor(np.asarray(counts, np.int32), device="cuda"), stream=stream)
    moved = h.update_poses_from_device(slots, torch.tensor(np.array([row[s][2] for s in slots], np.float64), device="cuda"),
                                       torch.tensor(np.stack([row[s][3].reshape(12) for s in slots]), device="cuda"),
                                       torch.tensor(np.array([row[s][1] for s in slots], np.float32), device="cuda"),
                                       torch.tensor(np.array([row[s][4] for s in slots], np.float64), device="cuda"), moved=True, stream=stream)
    out = h.run_scans_to_device(clouds, slots, "device", None, labels=True, select="all", index=True, stream=stream, device_counts=True)
    return out, moved


def poisoned_clouds(row, slots, rng, extra=300):
    """Per slot the row's points, then `extra` poison records; (CUDA clouds, counts, capacities)."""
    us = [len(row[s][0]) for s in slots]
    caps = [u + extra for u in us]
    return [to_device(with_poison(row[s][0], u, c, rng)) for s, u, c in zip(slots, us, caps)], us, caps


def mid_sequence(g, twin, steps, slots):
    """init_map at step 0, then one device-pose, device-count scan (step 1) on both handles."""
    rng = np.random.default_rng(5)
    for h in (g, twin):
        for s in slots:
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    clouds, us, caps = poisoned_clouds(steps[1], slots, rng)
    out_g, mv_g = device_step(g, slots, steps[1], clouds, us)
    out_t, mv_t = device_step(twin, slots, steps[1], clouds, us)
    same_outputs(out_g, out_t, us, "mid-sequence")
    return clouds, us, caps


MASKS = {"zero": [0] * B, "one": [1] * B, "sparse": [1, 0, 0, 1, 0, 1, 0, 0], "null": None}


@pytest.mark.parametrize("full_layers", [False, True])
def test_single_call_every_mask(monkeypatch, full_layers):
    """8 slots over 3 stream groups, mid-sequence, some positions host-owned and some device-owned: all-zero, all-one,
    sparse and NULL masks, each checked layer by layer and position by position against host gg_init_map."""
    torch = torch_mod()
    g, twin = handles(monkeypatch, full_layers)
    names = LIVE + DEAD if full_layers else LIVE
    steps = pose_steps(B, 2, jump=0.0, seed=7100)
    slots = list(range(B))[::-1]
    mid_sequence(g, twin, steps, slots)
    rng = np.random.default_rng(71)
    device_owned = [0, 2, 3, 5, 7]
    for case, mask in MASKS.items():
        # a roll to the current position moves nothing and leaves these positions device-owned
        pos = {s: g.position(slot=s) for s in range(B)}
        for h in (g, twin):
            xy = torch.tensor(np.array([pos[s] for s in device_owned]), device="cuda")
            T = torch.tensor(np.stack([steps[1][s][3].reshape(12) for s in device_owned]), device="cuda")
            assert h.update_poses_from_device(device_owned, xy, T, moved=True).tolist() == [0] * len(device_owned)
        before = {(s, n): g.layer(n, slot=s) for s in range(B) for n in names}
        xyz = reset_poses(rng, [pos[s] for s in slots])
        m = None if mask is None else torch.tensor(mask, dtype=torch.int32, device="cuda")
        g.init_maps_from_device(slots, torch.tensor(xyz, device="cuda"), m)
        twin_resets(twin, slots, xyz, mask)
        ctx = f"mask {case}"
        assert_layers(g, twin, range(B), names, ctx)
        assert_positions(g, twin, range(B), ctx)
        for k, s in enumerate(slots):
            if mask is not None and not mask[k]:
                for n in names:
                    assert np.array_equal(bits(g.layer(n, slot=s)), bits(before[(s, n)])), f"{ctx} slot {s}: {n} changed"
                assert bits(g.position(slot=s)).tolist() == bits(pos[s]).tolist(), f"{ctx} slot {s}: position changed"
            else:
                assert bits(g.position(slot=s)).tolist() == bits(xyz[k][:2]).tolist(), f"{ctx} slot {s}: position"


def test_rolling_sequence(monkeypatch):
    """12 steps of seeded resets -> counts -> device poses -> scans on 8 slots over 3 stream groups; the twin resets with
    host gg_init_map.  Outputs every step, layers and positions at the end; slot 0 against the CPU oracle re-initialised
    at its reset steps."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    STEPS = 12
    steps = pose_steps(B, STEPS, jump=0.0, seed=7200)
    slots = [3, 0, 6, 1, 4, 7, 2, 5]
    rng = np.random.default_rng(72)
    o = Oracle(99.0, 0.33)
    for h in (g, twin):
        for s in slots:
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    o.init_map(steps[0][0][2][0], steps[0][0][2][1], 0.0)
    j0 = slots.index(0)
    checked = 0
    for k in range(1, STEPS):
        row = steps[k]
        ctx = f"step {k}"
        mask = (rng.random(B) < 0.3).astype(np.int32)
        mask[j0] = 1 if k in (2, 3, 7) else 0
        xyz = reset_poses(rng, [row[s][2] for s in slots])
        g.init_maps_from_device(slots, torch.tensor(xyz, device="cuda"), torch.tensor(mask, device="cuda"))
        twin_resets(twin, slots, xyz, mask)
        clouds, us, caps = poisoned_clouds(row, slots, rng)
        out_g, mv_g = device_step(g, slots, row, clouds, us)
        out_t, mv_t = device_step(twin, slots, row, clouds, us)
        same_outputs(out_g, out_t, us, ctx)
        assert torch.equal(mv_g, mv_t), f"{ctx}: dev_moved"
        if mask[j0]:
            o.init_map(float(xyz[j0][0]), float(xyz[j0][1]), float(xyz[j0][2]))
        o.update(row[0][2][0], row[0][2][1], row[0][3])
        ref, _, _ = o.filter_cloud(row[0][0], row[0][1], row[0][4], threads=1)
        if k in (2, 3, 7, STEPS - 1):
            assert np.array_equal(out_g.labels[j0][:us[j0]].cpu().numpy(), ref), f"{ctx}: labels differ from the oracle"
            for name in ("ground", "groundpatch"):
                assert np.array_equal(bits(g.layer(name, slot=0)), bits(o.layer(name))), f"{ctx}: {name} vs oracle"
            checked += 1
    assert checked == 4
    assert_twin(g, twin, slots, us, caps, "end")
    assert_positions(g, twin, slots, "end")


def plan_kw(inp, select):
    return dict(counts=inp.counts, xy=inp.xy, T_base_from_map=inp.T, pose_origins=inp.origins, pose_base_z=inp.base_z, moved=True,
                labels=True, select=select, index=True)


def make_plan(g, inp, select, **extra):
    kw = dict(plan_kw(inp, select), **extra)
    if inp.route == "records":
        return g.step_plan(inp.slots, clouds=inp.buf, **kw)
    return g.step_plan(inp.slots, payloads=inp.buf, point_step=inp.step, field_offsets=inp.offs,
                       T=None if inp.Tmap is None else list(inp.Tmap), **kw)


def plan_masks(steps):
    """Per step: all zero, all one, then slot index 2 reset on two consecutive steps among seeded masks."""
    rng = np.random.default_rng(73)
    out = []
    for k in range(steps):
        if k == 0:
            m = np.zeros(B, np.int32)
        elif k == 1:
            m = np.ones(B, np.int32)
        else:
            m = (rng.random(B) < 0.3).astype(np.int32)
            m[2] = 1 if k in (3, 4) else 0
        out.append(m)
    return out


@pytest.mark.parametrize("capture", [False, True])
@pytest.mark.parametrize("route", ["records", "msgs18"])
def test_plan_with_resets(monkeypatch, route, capture):
    """step_plan(..., reset_xyz, reset_mask) with the mask rewritten before every replay, plain or captured in
    torch.cuda.graph: each replay equals the twin's host resets + literal call sequence on the same tensors."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    STEPS = 8
    steps = pose_steps(B, STEPS + 1, jump=0.0, seed=7300)
    rng = np.random.default_rng(74)
    for h in (g, twin):
        for s in range(B):
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    inp = Inputs(torch, [5, 2, 7, 0, 3, 6, 1, 4], route)
    rx = torch.zeros((B, 3), dtype=torch.float64, device="cuda")
    rm = torch.zeros(B, dtype=torch.int32, device="cuda")
    plain = make_plan(g, inp, "all")
    k_plain = plain.kernels
    plain.close()
    plan = make_plan(g, inp, "all", reset_xyz=rx, reset_mask=rm)
    assert plan.kernels == k_plain + GROUPS
    graph = None
    if capture:
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            plan.launch()
    masks = plan_masks(STEPS)
    prev = {s: np.array(steps[0][s][2], np.float64) for s in range(B)}
    for k in range(STEPS):
        row = steps[k + 1]
        ctx = f"{route} capture={capture} step {k}"
        xy, _ = step_xy(row, k + 1, prev)
        us, _ = inp.write(torch, row, xy, rng, [(s + k) % 4 for s in inp.slots])
        xyz = reset_poses(rng, [row[s][2] for s in inp.slots])
        rx.copy_(torch.tensor(xyz))
        rm.copy_(torch.tensor(masks[k]))
        g0 = g.kernel_launches
        if capture:
            graph.replay()
        else:
            plan.launch()
            assert g.kernel_launches - g0 == plan.kernels, ctx
        torch.cuda.synchronize()
        twin_resets(twin, inp.slots, xyz, masks[k])
        out_t, moved_t = inp.twin_step(twin, "all")
        check_step(plan, out_t, moved_t, us, ctx)
        prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
    torch.cuda.synchronize()
    assert_twin(g, twin, inp.slots, us, [CAPS[s] for s in inp.slots], f"{route} end")
    assert_positions(g, twin, range(B), f"{route} end")
    del graph
    plan.close()


def test_state_rules(monkeypatch):
    """After a reset: point info refused until the next scan, get_output and tallies unchanged, a flagged scan uses the
    kept scan pose and count, position() gives the reset doubles; mask=None gives an uninitialised slot a map; a slot
    bound to a plan accepts the call."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 3, jump=0.0, seed=7400)
    slots = list(range(B - 1))            # slot B - 1 stays uninitialised
    clouds, us, caps = mid_sequence(g, twin, steps, slots)
    outputs = {s: g.get_output(slot=s, want_cloud=True) for s in slots}
    tallies = g.eval_counts_to_device(slots)
    g.position(slot=4)                    # host-owned again; the others stay device-owned
    rng = np.random.default_rng(75)
    mask = np.array([1, 0, 1, 1, 0, 0, 1], np.int32)
    xyz = reset_poses(rng, [steps[2][s][2] for s in slots])
    g.init_maps_from_device(slots, torch.tensor(xyz, device="cuda"), torch.tensor(mask, device="cuda"))
    twin_resets(twin, slots, xyz, mask)
    for s in slots:
        with pytest.raises(capi.GroundGridError) as e:
            g.point_info_to_device([s])
        assert e.value.code == STATE, f"slot {s}: point info after a reset"
    for s in slots:
        gi, gc = g.get_output(slot=s, want_cloud=True)
        assert np.array_equal(gi, outputs[s][0]) and gc.tobytes() == outputs[s][1].tobytes(), f"slot {s}: get_output changed"
    assert torch.equal(g.eval_counts_to_device(slots), tallies), "tallies changed"
    assert_layers(g, twin, slots, LIVE, "after the reset")
    for k, s in enumerate(slots):
        if mask[k]:
            assert bits(g.position(slot=s)).tolist() == bits(xyz[k][:2]).tolist(), f"slot {s}: position"
    assert_positions(g, twin, slots, "after the reset")

    # a flagged scan right after the reset runs on the kept scan pose and count; the twin's gg_init_map forgot them
    row1, row2 = steps[1], steps[2]
    cap2 = [max(u, len(row2[s][0])) + 200 for s, u in zip(slots, us)]
    clouds2 = [to_device(with_poison(row2[s][0], min(len(row2[s][0]), c), c, rng)) for s, c in zip(slots, cap2)]
    out_g = g.run_scans_to_device(clouds2, slots, "device", None, labels=True, select="all", index=True, device_counts=True)
    twin.set_point_counts_from_device(slots, torch.tensor(np.asarray(us, np.int32), device="cuda"))
    twin.update_poses_from_device(slots, origins=torch.tensor(np.array([row1[s][1] for s in slots], np.float32), device="cuda"),
                                  base_z=torch.tensor(np.array([row1[s][4] for s in slots], np.float64), device="cuda"))
    out_t = twin.run_scans_to_device(clouds2, slots, "device", None, labels=True, select="all", index=True, device_counts=True)
    same_outputs(out_g, out_t, us, "flagged scan after the reset")
    assert_twin(g, twin, slots, us, cap2, "flagged scan after the reset")

    # mask=None on a slot without a map
    last = B - 1
    xyz7 = reset_poses(rng, [steps[2][last][2]])
    g.init_maps_from_device([last], torch.tensor(xyz7, device="cuda"))
    twin_resets(twin, [last], xyz7, None)
    pts, org = steps[2][last][0], steps[2][last][1]
    outs = [h.run_scans_to_device([to_device(pts)], [last], [org], 0.1, labels=True, select="all", index=True) for h in (g, twin)]
    same_outputs(outs[0], outs[1], [len(pts)], "uninitialised slot")
    assert_layers(g, twin, [last], LIVE, "uninitialised slot")
    assert bits(g.position(slot=last)).tolist() == bits(xyz7[0][:2]).tolist() == bits(twin.position(slot=last)).tolist()

    # a slot bound to a step plan accepts the call
    inp = Inputs(torch, [0, 3], "records")
    plan = make_plan(g, inp, "all")
    xyz_b = reset_poses(rng, [steps[2][s][2] for s in (3, 5)])
    g.init_maps_from_device([3, 5], torch.tensor(xyz_b, device="cuda"), torch.ones(2, dtype=torch.int32, device="cuda"))
    twin_resets(twin, [3, 5], xyz_b, [1, 1])
    assert_layers(g, twin, [3, 5], LIVE, "bound slot")
    assert_positions(g, twin, [3, 5], "bound slot")
    plan.close()


def test_stream_contract(monkeypatch):
    """xyz and mask produced on a side stream behind a sleep, the call on that stream returning before it gets there,
    and both overwritten on the stream right after the call: the reset uses the values of the call."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 2, jump=0.0, seed=7500)
    slots = list(range(B))
    mid_sequence(g, twin, steps, slots)
    rng = np.random.default_rng(76)
    xyz = reset_poses(rng, [steps[1][s][2] for s in slots])
    mask = np.array([0, 1, 1, 0, 1, 0, 0, 1], np.int32)
    rx = torch.zeros((B, 3), dtype=torch.float64, device="cuda")
    rm = torch.zeros(B, dtype=torch.int32, device="cuda")
    want_x, want_m = torch.tensor(xyz, device="cuda"), torch.tensor(mask, device="cuda")
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        rx.copy_(want_x)
        rm.copy_(want_m)
    g.init_maps_from_device(slots, rx, rm, stream=side)
    assert not side.query(), "gg_init_maps_from_device waited for the stream"
    with torch.cuda.stream(side):
        rx.fill_(1.0e6)
        rm.copy_(1 - want_m)
    side.synchronize()
    twin_resets(twin, slots, xyz, mask)
    assert_layers(g, twin, slots, LIVE, "stream contract")
    assert_positions(g, twin, slots, "stream contract")


def test_rejections_enqueue_nothing(monkeypatch):
    """Every GG_E_ARG / GG_E_STATE of gg_init_maps_from_device and of gg_step_plan_create_with_resets without xyz leaves
    gg_kernel_launches unchanged; count 0 succeeds and enqueues nothing."""
    torch = torch_mod()
    g, _ = handles(monkeypatch)
    L = g._l
    for s in range(B - 1):                # slot B - 1 stays uninitialised
        g.init_map(0.0, 0.0, 0.0, slot=s)
    rx = torch.zeros((B + 1, 3), dtype=torch.float64, device="cuda")
    rm = torch.ones(B + 1, dtype=torch.int32, device="cuda")
    ground = g.layer_device_ptr("ground", slot=2)
    g.synchronize()
    before = g.kernel_launches

    def call(slots=(0, 3, 5), xyz=rx.data_ptr(), mask=rm.data_ptr(), h=g._h, resets=True, null_slots=False, count=None):
        sl = np.ascontiguousarray(slots, np.int32)
        r = capi.DeviceResets(xyz, mask)
        return L.gg_init_maps_from_device(h, len(sl) if count is None else count, None if null_slots else capi._ptr(sl),
                                          C.byref(r) if resets else None, None)

    cases = {
        "null handle": (dict(h=None), ARG),
        "null slots": (dict(null_slots=True), ARG),
        "null resets": (dict(resets=False), ARG),
        "null xyz": (dict(xyz=None), ARG),
        "count > n_slots": (dict(slots=list(range(B + 1))), ARG),
        "slot out of range": (dict(slots=(0, B, 5)), ARG),
        "negative slot": (dict(slots=(0, -1, 5)), ARG),
        "repeated slot": (dict(slots=(0, 3, 3)), ARG),
        "misaligned xyz": (dict(xyz=rx.data_ptr() + 4), ARG),
        "misaligned mask": (dict(mask=rm.data_ptr() + 2), ARG),
        "xyz overlapping the layers": (dict(xyz=ground), ARG),
        "mask overlapping the layers": (dict(mask=ground), ARG),
        "map not initialised with a mask": (dict(slots=(0, B - 1)), STATE),
    }
    for name, (kw, want) in cases.items():
        assert call(**kw) == want, name
        assert g.kernel_launches == before, name
    assert call(count=0) == 0 and call(count=0, null_slots=True, resets=False) == 0
    assert g.kernel_launches == before, "count 0"
    p = C.c_void_p()
    rc = L.gg_step_plan_create_with_resets(g._h, C.byref(capi.StepDesc()), C.byref(capi.DeviceResets(None, rm.data_ptr())), C.byref(p))
    assert rc == ARG and not p.value
    assert g.kernel_launches == before
    # the same call with valid arguments launches one kernel per stream group with slots in it
    assert call() == 0
    assert g.kernel_launches == before + len({s * GROUPS // B for s in (0, 3, 5)})
    g.synchronize()
    # inputs may share memory: a mask inside xyz is accepted (its zero words reset no slot)
    assert call(mask=rx.data_ptr() + 8) == 0
    assert g.kernel_launches == before + 2 * len({s * GROUPS // B for s in (0, 3, 5)})
    g.synchronize()

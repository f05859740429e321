"""Per-slot configurations from caller GPU memory (gg_set_slot_configs_from_device, gg_step_plan_create_with_configs).
Every case runs against a twin handle that calls the host gg_set_slot_config for the masked slots at the same point of
the sequence, and must be bit-identical to it: labels, index, cloud, dev_counts, every layer, map positions, point info
and tallies.  Slot 0 is also followed by the CPU oracle with the same configuration."""
import math

import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from oracle import Oracle
from test_gpu_device_counts import assert_twin
from test_gpu_device_outputs import DEAD, LIVE, torch_mod
from test_gpu_device_poses import pose_steps
from test_gpu_map_resets import B, GROUPS, assert_layers, assert_positions, device_step, handles, make_plan, poisoned_clouds, same_outputs
from test_gpu_slot_config import CFGS, full
from test_gpu_step_plans import CAPS, Inputs, check_step, step_xy

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
DOUBLES = [name for name, t in capi.Config._fields_ if t is capi.C.c_double]
# NaN and +-inf in every double field, ring cut-offs of 0 and below, the largest variance threshold, decay factors of 0
# and 0.5, and patch-size distances on both sides of the centre cells of an N = 300 map
EDGE = ([{f: v} for f in DOUBLES for v in (math.nan, math.inf, -math.inf)]
        + [dict(max_ring=0), dict(max_ring=-7), dict(point_count_cell_variance_threshold=2**31 - 1),
           dict(occupied_cells_decrease_factor=0.0), dict(occupied_cells_decrease_factor=0.5),
           dict(patch_size_change_distance=0.33), dict(patch_size_change_distance=35.0), dict(patch_size_change_distance=-4.0)])
MASKS = {"zero": [0] * B, "one": [1] * B, "sparse": [1, 0, 0, 1, 0, 1, 0, 0], "null": None}


def cfg_bytes(kw):
    return capi.config_tensor([full(kw)], device="cpu")[0].numpy().tobytes()


def twin_configs(twin, slots, kws, mask):
    """The host path the device call must equal: gg_set_slot_config of every masked slot."""
    for k, s in enumerate(slots):
        if mask is None or mask[k]:
            twin.set_config(slot=int(s), **full(kws[k]))


def both_configs(g, twin, slots, kws, mask=None, stream=None):
    torch = torch_mod()
    m = None if mask is None else torch.tensor(np.asarray(mask, np.int32), device="cuda")
    g.set_configs_from_device(slots, capi.config_tensor([full(kw) for kw in kws]), m, stream=stream)
    twin_configs(twin, slots, kws, mask)


def start(g, twin, steps, slots):
    for h in (g, twin):
        for s in slots:
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)


def step_both(g, twin, row, slots, rng, ctx, names=LIVE):
    clouds, us, caps = poisoned_clouds(row, slots, rng)
    out_g, mv_g = device_step(g, slots, row, clouds, us)
    out_t, mv_t = device_step(twin, slots, row, clouds, us)
    same_outputs(out_g, out_t, us, ctx)
    assert torch_mod().equal(mv_g, mv_t), f"{ctx}: dev_moved"
    assert_twin(g, twin, slots, us, caps, ctx, names=names)
    return out_g, us


@pytest.mark.parametrize("full_layers", [False, True])
def test_every_mask_mid_sequence(monkeypatch, full_layers):
    """8 slots over 3 stream groups: all-zero, all-one, sparse and NULL masks between rolling device steps, each followed
    by a roll and a scan; masked-off slots keep their configuration bytes; slot 0 against the oracle."""
    g, twin = handles(monkeypatch, full_layers)
    names = LIVE + DEAD if full_layers else LIVE
    steps = pose_steps(B, 2 + len(MASKS), jump=0.0, seed=8100)
    slots = list(range(B))[::-1]
    start(g, twin, steps, slots)
    rng = np.random.default_rng(81)
    o = Oracle(99.0, 0.33)   # slot 0 starts with the default configuration
    o.init_map(steps[0][0][2][0], steps[0][0][2][1], 0.0)
    j0 = slots.index(0)
    for k, (case, mask) in enumerate([(None, [0] * B)] + list(MASKS.items())):
        row = steps[k + 1]
        ctx = f"mask {case} step {k + 1}"
        kws = [CFGS[(s + k) % 4] for s in slots]
        before = {s: bytes(g.get_config(slot=s)) for s in slots}
        if case is not None:
            both_configs(g, twin, slots, kws, mask)
            for j, s in enumerate(slots):
                want = cfg_bytes(kws[j]) if mask is None or mask[j] else before[s]
                assert bytes(g.get_config(slot=s)) == want, f"{ctx} slot {s}: stored configuration"
            if mask is None or mask[j0]:
                o.set_config(**full(kws[j0]))
        out_g, us = step_both(g, twin, row, slots, rng, ctx, names)
        o.update(row[0][2][0], row[0][2][1], row[0][3])
        ref, _, _ = o.filter_cloud(row[0][0], row[0][1], row[0][4], threads=1)
        assert np.array_equal(out_g.labels[j0][:us[j0]].cpu().numpy(), ref), f"{ctx}: labels differ from the oracle"
        for name in ("ground", "groundpatch"):
            assert np.array_equal(g.layer(name, slot=0).view(np.uint32), o.layer(name).view(np.uint32)), f"{ctx}: {name} vs oracle"
    assert_positions(g, twin, range(B), "end")


def test_edge_configurations(monkeypatch):
    """NaN and +-inf in each double field, max_ring 0 and negative, INT_MAX variance threshold, decay factors 0 and 0.5,
    patch-size distances that move the 3x3 / 5x5 boundary: eight at a time, each followed by a roll and a scan."""
    g, twin = handles(monkeypatch, full_layers=True)
    batches = [EDGE[i:i + B] for i in range(0, len(EDGE), B)]
    steps = pose_steps(B, 1 + len(batches), jump=0.0, seed=8200)
    slots = list(range(B))
    start(g, twin, steps, slots)
    rng = np.random.default_rng(82)
    for k, batch in enumerate(batches):
        kws = [batch[j % len(batch)] for j in range(B)]
        both_configs(g, twin, slots, kws)
        for j, s in enumerate(slots):
            assert bytes(g.get_config(slot=s)) == cfg_bytes(kws[j]), f"batch {k} slot {s}: stored bytes"
        step_both(g, twin, steps[k + 1], slots, rng, f"edge batch {k}", LIVE + DEAD)


def test_every_flow_on_device_configured_slots():
    """gg_filter_cloud, gg_filter_cloud_batch, gg_run_scans, gg_run_scans_device, gg_run_scans_to_device,
    gg_run_cloud_msgs_to_device, gg_run_merged_cloud_msgs_to_device, the per-phase entries, gg_detect_ground_patch and
    gg_interpolate_cell on slots configured from the device, against the twin's host configurations."""
    torch = torch_mod()
    dim, res, n = 33.33, 0.33, 4
    g, twin = [capi.GroundGridB200(dim, res, n_slots=n, max_points=40000, full_layers=True) for _ in range(2)]
    slots = list(range(n))
    kws = [CFGS[(s + 1) % 4] for s in slots]
    both_configs(g, twin, slots, kws)
    scene = synth.make_scene(seed=23, n_boxes=8, rmin=4.0, rmax=14.0)
    for h in (g, twin):
        for s in slots:
            h.init_map(0.0, 0.0, 0.0, slot=s)

    def cloud(k):
        pts, org = synth.lidar_scan(scene, beams=64, az_steps=512, seed=230 + k)
        pts["z"][:: 37 + k] -= 0.8
        return pts, org

    def same(ctx, names=LIVE + DEAD):
        g.synchronize()
        twin.synchronize()
        assert_layers(g, twin, slots, names, ctx)

    pts, org = cloud(0)
    for s in slots:
        assert np.array_equal(g.filter_cloud(pts, org, 0.1, slot=s), twin.filter_cloud(pts, org, 0.1, slot=s)), f"filter_cloud slot {s}"
    same("filter_cloud")
    pts, org = cloud(1)
    labels = {}
    for h in (g, twin):
        descs = h.make_descs(slots, [len(pts)] * n, [org] * n, [0.2] * n)
        hp = [torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).pin_memory() for _ in slots]
        hl = [torch.zeros(len(pts), dtype=torch.uint8).pin_memory() for _ in slots]
        h.filter_cloud_batch_ptrs(descs, [t.data_ptr() for t in hp], [t.data_ptr() for t in hl])
        labels[h] = [t.numpy().copy() for t in hl]
    assert all(np.array_equal(a, b) for a, b in zip(labels[g], labels[twin])), "filter_cloud_batch labels"
    same("filter_cloud_batch")
    pts, org = cloud(2)
    for h in (g, twin):
        keep = [h.upload_points(pts, slot=s) for s in slots]
        h.run_scans(h.make_descs(slots, [len(pts)] * n, [org] * n, [0.0] * n))
        h.synchronize()
        del keep
    same("run_scans")
    pts, org = cloud(3)
    dev = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).cuda()
    for h in (g, twin):
        h.run_scans_device(h.make_descs(slots, [len(pts)] * n, [org] * n, [0.0] * n), [dev.data_ptr()] * n)
    same("run_scans_device")
    pts, org = cloud(4)
    dev = torch.from_numpy(np.ascontiguousarray(pts).view(np.float32).reshape(-1, 8).copy()).cuda()
    outs = [h.run_scans_to_device([dev] * n, slots, [org] * n, [0.0] * n, labels=True, select="all", index=True) for h in (g, twin)]
    same_outputs(outs[0], outs[1], [len(pts)] * n, "run_scans_to_device")
    same("run_scans_to_device")
    pts, org = cloud(5)
    raw = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).cuda()
    outs = [h.run_cloud_msgs_to_device([raw] * n, 32, (0, 4, 8, 16, 20), None, slots, [org] * n, [0.0] * n, labels=True, select="all",
                                       index=True) for h in (g, twin)]
    same_outputs(outs[0], outs[1], [len(pts)] * n, "run_cloud_msgs_to_device")
    same("run_cloud_msgs_to_device")
    pts, org = cloud(6)
    half = len(pts) // 2
    parts = [torch.from_numpy(np.ascontiguousarray(pts[a:b]).view(np.uint8).copy()).cuda() for a, b in ((0, half), (half, len(pts)))]
    outs = [h.run_merged_cloud_msgs_to_device([parts] * n, 32, (0, 4, 8, 16, 20), None, slots, [org] * n, [0.0] * n, labels=True,
                                              select="all", index=True) for h in (g, twin)]
    same_outputs(outs[0], outs[1], [len(pts)] * n, "run_merged_cloud_msgs_to_device")
    same("run_merged_cloud_msgs_to_device")
    pts, org = cloud(7)
    for h in (g, twin):
        for s in slots:
            h.run_single(pts, org, 0.25, slot=s, stop_after=1)
            h.detect_ground_patches(slot=s)
            h.spiral_ground_interpolation(0.25, slot=s)
    same("per-phase entries")
    pts, org = cloud(8)
    N = g.n
    for h in (g, twin):
        for s in slots:
            h.run_single(pts, org, 0.0, slot=s, stop_after=1)
            for S in (3, 5):
                for i in range(N // 2 - 10, N // 2 + 10, 3):
                    h.detect_ground_patch(S, i, i + 1, slot=s)
            for x, y in ((5, 7), (N // 2, N // 2 - 1), (1, 1), (N - 2, N - 2)):
                h.interpolate_cell(x, y, slot=s)
    same("detect_ground_patch / interpolate_cell", ("ground", "groundpatch"))


def test_host_state_rules(monkeypatch):
    """get_config returns the stored bytes; set_config(slot) and set_config() make slots host-configured again and a
    later device call works; init_map and init_maps_from_device keep the configuration; a slot that was in a call only
    with mask 0 behaves as before."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 6, jump=0.0, seed=8300)
    slots = list(range(B))
    start(g, twin, steps, slots)
    rng = np.random.default_rng(83)
    nan_cfg = dict(CFGS[1], outlier_tolerance=math.nan)
    mask = [0, 1] * (B // 2)
    both_configs(g, twin, slots, [nan_cfg] * B, mask)
    for s in slots:
        assert bytes(g.get_config(slot=s)) == bytes(twin.get_config(slot=s)), f"slot {s}: get_config"
    step_both(g, twin, steps[1], slots, rng, "mask 0 / 1")
    g.set_config(slot=1, **full(CFGS[3]))
    twin.set_config(slot=1, **full(CFGS[3]))
    assert bytes(g.get_config(slot=1)) == cfg_bytes(CFGS[3])
    step_both(g, twin, steps[2], slots, rng, "slot 1 host-configured again")
    both_configs(g, twin, [1, 2], [CFGS[2], CFGS[0]])
    step_both(g, twin, steps[3], slots, rng, "device call after the revert")
    for h in (g, twin):   # init_map keeps the configuration
        h.init_map(steps[3][5][2][0], steps[3][5][2][1], 0.5, slot=5)
    xyz = np.array([[steps[3][s][2][0], steps[3][s][2][1], 0.25] for s in (2, 3)], np.float64)
    g.init_maps_from_device([2, 3], torch.tensor(xyz, device="cuda"))
    for j, s in enumerate((2, 3)):
        twin.init_map(*map(float, xyz[j]), slot=s)
    step_both(g, twin, steps[4], slots, rng, "after init_map / init_maps_from_device")
    g.set_config(**full(CFGS[1]))
    twin.set_config(**full(CFGS[1]))
    for s in slots:
        assert bytes(g.get_config(slot=s)) == cfg_bytes(CFGS[1])
    step_both(g, twin, steps[5], slots, rng, "handle-wide revert")
    assert_positions(g, twin, slots, "end")


def test_stream_contract(monkeypatch):
    """The call on a side stream, its configuration buffer overwritten with poison on that stream right after the call,
    the scans that follow on the same stream: the poison has no effect."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 3, jump=0.0, seed=8400)
    slots = [4, 1, 6, 0, 7, 2, 5, 3]
    start(g, twin, steps, slots)
    rng = np.random.default_rng(84)
    side = torch.cuda.Stream()
    for k in (1, 2):
        kws = [CFGS[(j + k) % 4] for j in range(B)]
        mask = (np.arange(B) % 3 != k).astype(np.int32)
        with torch.cuda.stream(side):
            t = capi.config_tensor([full(kw) for kw in kws])
            m = torch.tensor(mask, device="cuda")
            torch.cuda._sleep(20_000_000)   # the call returns long before its kernels run
            g.set_configs_from_device(slots, t, m, stream=side)
            t.fill_(0x7f)
            m.fill_(1)
            clouds, us, caps = poisoned_clouds(steps[k], slots, rng)
            out_g, _ = device_step(g, slots, steps[k], clouds, us, stream=side)
        side.synchronize()
        twin_configs(twin, slots, kws, mask)
        out_t, _ = device_step(twin, slots, steps[k], clouds, us)
        same_outputs(out_g, out_t, us, f"step {k}")
        assert_twin(g, twin, slots, us, caps, f"step {k}")


@pytest.mark.parametrize("capture", [False, True])
def test_plan_with_configs(monkeypatch, capture):
    """step_plan(..., configs, config_mask) with both rewritten before every replay, plain or captured in
    torch.cuda.graph: each replay equals the twin's host gg_set_slot_config + literal call sequence."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    STEPS = 6
    steps = pose_steps(B, STEPS + 1, jump=0.0, seed=8500)
    rng = np.random.default_rng(85)
    start(g, twin, steps, range(B))
    inp = Inputs(torch, [5, 2, 7, 0, 3, 6, 1, 4], "records")
    plain = make_plan(g, inp, "all")
    k_plain = plain.kernels
    plain.close()
    ct = capi.config_tensor([full(CFGS[0])] * B)
    cm = torch.zeros(B, dtype=torch.int32, device="cuda")
    plan = make_plan(g, inp, "all", configs=ct, config_mask=cm)
    assert plan.kernels == k_plain + 2 * GROUPS
    graph = None
    if capture:
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            plan.launch()
    prev = {s: np.array(steps[0][s][2], np.float64) for s in range(B)}
    for k in range(STEPS):
        row = steps[k + 1]
        ctx = f"capture={capture} step {k}"
        xy, _ = step_xy(row, k + 1, prev)
        us, _ = inp.write(torch, row, xy, rng, [(s + k) % 4 for s in inp.slots])
        kws = [CFGS[(j + k) % 4] if k % 3 else EDGE[(5 * k + j) % len(EDGE)] for j in range(B)]
        mask = [1] * B if k == 0 else (rng.random(B) < 0.5).astype(np.int32).tolist()
        ct.copy_(capi.config_tensor([full(kw) for kw in kws]))
        capi.config_field(ct, "outlier_tolerance")[::3].fill_(0.17)   # written on the GPU
        for j in range(0, B, 3):
            kws[j] = dict(kws[j], outlier_tolerance=0.17)
        cm.copy_(torch.tensor(mask, dtype=torch.int32))
        if capture:
            graph.replay()
        else:
            plan.launch()
        torch.cuda.synchronize()
        twin_configs(twin, inp.slots, kws, mask)
        out_t, moved_t = inp.twin_step(twin, "all")
        check_step(plan, out_t, moved_t, us, ctx)
        prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
    torch.cuda.synchronize()
    assert_twin(g, twin, inp.slots, us, [CAPS[s] for s in inp.slots], "end")
    for s in range(B):
        assert bytes(g.get_config(slot=s)) == bytes(twin.get_config(slot=s)), f"slot {s}: stored configuration"
    # a standalone call on the bound, device-configured slots is accepted and reaches the next replay
    g.set_configs_from_device([0, 3], capi.config_tensor([full(CFGS[2]), full(CFGS[1])]))
    twin_configs(twin, [0, 3], [CFGS[2], CFGS[1]], None)
    cm.zero_()
    row = steps[STEPS]
    us, _ = inp.write(torch, row, {s: np.array(row[s][2], np.float64) for s in range(B)}, rng, [0] * B)
    if capture:
        graph.replay()
    else:
        plan.launch()
    torch.cuda.synchronize()
    out_t, moved_t = inp.twin_step(twin, "all")
    check_step(plan, out_t, moved_t, us, "standalone call on bound slots")
    for code_call in (lambda: g.set_config(slot=0, **full(CFGS[0])), lambda: g.set_config(**full(CFGS[0]))):
        with pytest.raises(capi.GroundGridError) as e:
            code_call()
        assert e.value.code == STATE
    del graph
    plan.close()


def test_rejections_enqueue_nothing(monkeypatch):
    """Every GG_E_ARG and GG_E_STATE of the call and of the plan entry point: no launch, no layer or state change; a
    rejected plan leaves no plan, no bound slot and no device-configured slot."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 1, jump=0.0, seed=8600)
    start(g, twin, steps, range(B))
    ct = capi.config_tensor([full(CFGS[1])] * B)
    m = torch.ones(B, dtype=torch.int32, device="cuda")
    layer = g.layer_device_ptr("ground", slot=2)
    before = {s: g.layer("groundpatch", slot=s) for s in range(B)}
    cfgs = {s: bytes(g.get_config(slot=s)) for s in range(B)}
    L = g._l
    sl = np.arange(B, dtype=np.int32)
    cases = [
        ("null slots", lambda: L.gg_set_slot_configs_from_device(g._h, B, None, capi.C.byref(capi.DeviceConfigs(ct.data_ptr(), None)), None), ARG),
        ("null configs", lambda: L.gg_set_slot_configs_from_device(g._h, B, capi._ptr(sl), None, None), ARG),
        ("null cfg", lambda: g.set_configs_from_device_ptrs(sl, None, m.data_ptr(), None), ARG),
        ("count > n_slots", lambda: g.set_configs_from_device_ptrs(np.arange(B + 1, dtype=np.int32) % B, ct.data_ptr(), None, None), ARG),
        ("slot out of range", lambda: g.set_configs_from_device_ptrs([0, B], ct.data_ptr(), None, None), ARG),
        ("negative slot", lambda: g.set_configs_from_device_ptrs([-1], ct.data_ptr(), None, None), ARG),
        ("repeated slot", lambda: g.set_configs_from_device_ptrs([3, 1, 3], ct.data_ptr(), None, None), ARG),
        ("cfg misaligned", lambda: g.set_configs_from_device_ptrs([0], ct.data_ptr() + 4, None, None), ARG),
        ("mask misaligned", lambda: g.set_configs_from_device_ptrs([0], ct.data_ptr(), m.data_ptr() + 2, None), ARG),
        ("cfg on the layers", lambda: g.set_configs_from_device_ptrs([0, 1], layer, None, None), ARG),
        ("mask on the layers", lambda: g.set_configs_from_device_ptrs([0, 1], ct.data_ptr(), layer + 64, None), ARG),
    ]
    assert L.gg_set_slot_configs_from_device(None, 1, capi._ptr(sl), capi.C.byref(capi.DeviceConfigs(ct.data_ptr(), None)), None) == ARG
    g.set_configs_from_device_ptrs([], None, None, None)   # count == 0: nothing to do
    torch.cuda.synchronize()
    n0 = g.kernel_launches
    for what, call, code in cases:
        if what.startswith("null") and what != "null cfg":
            assert call() == code, what
            continue
        with pytest.raises(capi.GroundGridError) as e:
            call()
        assert e.value.code == code, what
    assert g.kernel_launches == n0
    # a plan recorded while the slots were host-configured carries their configurations by value
    inp = Inputs(torch, [1, 6], "records")
    plan = make_plan(g, inp, "all")
    with pytest.raises(capi.GroundGridError) as e:
        g.set_configs_from_device([6, 2], ct[:2])
    assert e.value.code == STATE
    assert g.kernel_launches == n0
    plan.close()
    # rejected plans: a recorded call that fails (a bad read-out name), and configs without cfg
    inp = Inputs(torch, [0, 5, 3], "records")
    with pytest.raises(capi.GroundGridError):
        make_plan(g, inp, "all", configs=ct[:3], layers=("no_such_layer",))
    d = capi.StepDesc()
    d.count = 3
    out = capi.C.c_void_p()
    assert L.gg_step_plan_create_with_configs(g._h, capi.C.byref(d), None, None, capi.C.byref(capi.DeviceConfigs(None, None)), None,
                                              capi.C.byref(out)) == ARG
    assert g.kernel_launches == n0
    # no slot was left bound or device-configured: a plan records them, and then refuses a device call as for any slot
    # that was host-configured at its creation
    plan = make_plan(g, inp, "all")
    with pytest.raises(capi.GroundGridError) as e:
        g.set_configs_from_device([0], ct[:1])
    assert e.value.code == STATE
    plan.close()
    for s in range(B):
        assert np.array_equal(g.layer("groundpatch", slot=s), before[s]), f"slot {s}: layers changed"
        assert bytes(g.get_config(slot=s)) == cfgs[s], f"slot {s}: configuration changed"
    # inputs may share memory: a mask inside cfg is accepted (its nonzero words reconfigure the slots)
    n1 = g.kernel_launches
    g.set_configs_from_device_ptrs([0, 1], ct.data_ptr(), ct.data_ptr() + 8, None)
    assert g.kernel_launches > n1
    assert bytes(g.get_config(slot=1)) == cfg_bytes(CFGS[1])

"""Step plan read-outs (gg_step_plan_create_with_readouts): layers, layer images, terrain images, terrain lookups, point
info and tallies written by every replay of a step plan.  Every case runs against a twin handle that makes the literal
call sequence -- the plan's step, then gg_get_layers_to_device, gg_layer_images_to_device, gg_terrain_images_to_device,
gg_sample_layers_to_device, gg_point_info_to_device and gg_eval_counts_to_device -- on the same tensors, and must be
bit-identical to it at every step.  Records past each scan's count are poison (test_gpu_device_counts)."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi
from test_gpu_device_counts import MAX_POINTS, point_info
from test_gpu_device_outputs import DEAD, LIVE, make_pair, torch_mod
from test_gpu_device_poses import pose_steps
from test_gpu_map_resets import plan_masks, reset_poses, twin_resets
from test_gpu_sample_layers import as_records, check, edge_xy, expected
from test_gpu_step_plans import CAPS, PLAN_SLOTS, Inputs, check_step, step_xy

pytestmark = pytest.mark.gpu

ARG, STATE, LAYER = -1, -3, -4
B, GROUPS = 8, 3
LAYER_NAMES = LIVE + DEAD                                 # every layer a full-layers handle keeps, "points" included
TERRAIN = slice(LAYER_NAMES.index("ground"), LAYER_NAMES.index("groundpatch") + 1)
IMAGE_NAMES = ("ground", "points", "pointsRaw", "variance")
SAMPLE_NAMES = ("ground", "groundpatch", "points")
EDGE_ROWS = 1500                                          # edge_xy(m=EDGE_ROWS) gives EDGE_ROWS + 10 positions


def handles(monkeypatch):
    monkeypatch.setenv("GG_STREAMS", str(GROUPS))
    g, twin = make_pair(99.0, 0.33, B, full_layers=True, max_points=MAX_POINTS)
    assert g.n_streams == GROUPS == twin.n_streams
    for h in (g, twin):
        h.res = 0.33   # what the lookup restatement needs
    return g, twin


def init_maps(g, twin, steps):
    for h in (g, twin):
        for s in range(B):
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)


def position_tensors(torch, slots):
    """Fixed position tensors of one plan: float2 sets for even positions in the batch, 32-byte records for odd ones."""
    n = EDGE_ROWS + 10
    return [torch.zeros((n, 8) if k % 2 else (n, 2), dtype=torch.float32, device="cuda") for k in range(len(slots))]


def write_positions(torch, g, slots, pos, rng):
    """New lookup positions around each slot's current map position (cell edges, outside the map, NaN, +-inf)."""
    xys = []
    for k, s in enumerate(slots):
        xy = edge_xy(g, int(s), rng, m=EDGE_ROWS)
        xys.append(xy)
        pos[k].copy_(torch.from_numpy(as_records(xy) if k % 2 else xy))
    return xys


def readout_kw(torch, slots, pos, mode):
    return dict(layers=LAYER_NAMES, layer_images=IMAGE_NAMES, terrain_images=True, samples=pos, sample_names=SAMPLE_NAMES,
                sample_mode=mode, sample_cells=True, point_info=("codes", "height"),
                tallies=torch.zeros((len(slots), 1024, 2), dtype=torch.int64, device="cuda"))


class Twin:
    """The six standalone calls on the twin, with capacity-sized point-info buffers and running tallies."""

    def __init__(self, torch, slots, mode):
        self.slots, self.mode = slots, mode
        self.tallies = torch.zeros((len(slots), 1024, 2), dtype=torch.int64, device="cuda")

    def readouts(self, torch, twin, pos):
        sl = self.slots
        r = {"layers": twin.get_layers_to_device(sl, LAYER_NAMES)}
        r["images"], r["ranges"] = twin.layer_images_to_device(sl, IMAGE_NAMES)
        r["terrain"] = twin.terrain_images_to_device(sl)
        r["samples"], r["cells"] = twin.sample_layers_to_device(sl, pos, SAMPLE_NAMES, mode=self.mode, cells=True)
        r["codes"], r["height"] = point_info(twin, sl, [CAPS[s] for s in sl], torch)
        twin.eval_counts_to_device(sl, out=self.tallies)
        r["tallies"] = self.tallies
        return r


def i32(t):
    return t.view(torch_mod().int32)


def assert_readouts(ro, want, us, ctx):
    """Every read-out of the plan against the twin's, bit for bit; codes and heights over the first u entries."""
    torch = torch_mod()
    torch.cuda.synchronize()
    assert torch.equal(i32(ro.layers), i32(want["layers"])), f"{ctx}: layers"
    assert torch.equal(ro.images, want["images"]) and torch.equal(i32(ro.ranges), i32(want["ranges"])), f"{ctx}: images"
    assert torch.equal(i32(ro.terrain), i32(want["terrain"])), f"{ctx}: terrain images"
    for k in range(len(us)):
        assert torch.equal(i32(ro.samples[k]), i32(want["samples"][k])), f"{ctx} set {k}: lookups"
        assert torch.equal(ro.cells[k], want["cells"][k]), f"{ctx} set {k}: cells"
        u = us[k]
        assert torch.equal(ro.codes[k][:u], want["codes"][k][:u]), f"{ctx} scan {k}: codes"
        assert torch.equal(i32(ro.height[k][:u]), i32(want["height"][k][:u])), f"{ctx} scan {k}: heights"
    assert torch.equal(ro.tallies, want["tallies"]), f"{ctx}: tallies"


@pytest.mark.parametrize("route", ["records", "msgs18"])
def test_rolling_sequence_matches_the_call_sequence(monkeypatch, route):
    """8 steps, two plans over the three stream groups (nearest and linear lookups), device counts with poison past each
    count, lookup positions rewritten every step; every read-out every step equals the twin's, the lookups also equal
    the restatement on the twin's planes, and each plan launches as many kernels as the twin's calls."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    STEPS = 8
    steps = pose_steps(B, STEPS, jump=30.0, seed=8100)
    rng = np.random.default_rng(81 + (route == "msgs18"))
    init_maps(g, twin, steps)
    modes = ("nearest", "linear")
    inputs = [Inputs(torch, list(sl), route) for sl in PLAN_SLOTS]
    pos = [position_tensors(torch, inp.slots) for inp in inputs]
    plans, twins = [], []
    for inp, p, mode, sel in zip(inputs, pos, modes, ("all", "nonground")):
        kw = dict(counts=inp.counts, xy=inp.xy, T_base_from_map=inp.T, pose_origins=inp.origins, pose_base_z=inp.base_z, moved=True,
                  labels=True, select=sel, index=True, **readout_kw(torch, inp.slots, p, mode))
        if route == "records":
            plans.append(g.step_plan(inp.slots, clouds=inp.buf, **kw))
        else:
            plans.append(g.step_plan(inp.slots, payloads=inp.buf, point_step=inp.step, field_offsets=inp.offs, T=list(inp.Tmap), **kw))
        twins.append(Twin(torch, inp.slots, mode))
    prev = {s: np.array(steps[0][s][2], np.float64) for s in range(B)}
    for k, row in enumerate(steps):
        xy, _ = step_xy(row, k, prev)
        written = [inp.write(torch, row, xy, rng, [(s + k) % 4 for s in inp.slots]) for inp in inputs]
        xys = [write_positions(torch, g, inp.slots, p, rng) for inp, p in zip(inputs, pos)]
        for plan in plans:
            plan.launch()
        for plan, inp, tw, p, sel, (us, _), xy_sets in zip(plans, inputs, twins, pos, ("all", "nonground"), written, xys):
            ctx = f"{route} step {k} plan {tw.mode}"
            t0 = twin.kernel_launches
            out_t, moved_t = inp.twin_step(twin, sel)
            want = tw.readouts(torch, twin, p)
            extra = len({s * GROUPS // B for s in inp.slots}) if route == "msgs18" else 0   # k_stage_transforms per branch
            assert plan.kernels == twin.kernel_launches - t0 + extra, ctx
            check_step(plan, out_t, moved_t, us, ctx)
            assert_readouts(plan.readouts, want, us, ctx)
            check(plan.readouts.samples, plan.readouts.cells, expected(twin, inp.slots, xy_sets, SAMPLE_NAMES, tw.mode), ctx)
        prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
    for plan in plans:
        plan.close()


def test_readouts_consumed_inside_a_torch_graph(monkeypatch):
    """plan.launch() and torch ops that read plan.readouts captured in one torch.cuda.graph, then 10 replays with new
    inputs: what the torch ops copied equals the twin's read-outs."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 11, jump=0.0, seed=8200)
    rng = np.random.default_rng(82)
    init_maps(g, twin, steps)
    inp = Inputs(torch, list(range(B))[::-1], "records")
    pos = position_tensors(torch, inp.slots)
    kw = dict(counts=inp.counts, xy=inp.xy, T_base_from_map=inp.T, pose_origins=inp.origins, pose_base_z=inp.base_z, moved=True, labels=True,
              select="all", index=True, **readout_kw(torch, inp.slots, pos, "linear"))
    plan = g.step_plan(inp.slots, clouds=inp.buf, **kw)
    ro = plan.readouts
    tw = Twin(torch, inp.slots, "linear")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan.launch()
        # the caller's own kernels on the read-outs, in the same capture: terrain planes and point heights
        planes = ro.layers[:, TERRAIN].contiguous()
        heights = torch.cat(ro.height)
        looked_up = torch.cat([s.reshape(-1) for s in ro.samples])
        tallies = ro.tallies.clone()
    prev = {s: np.array(steps[0][s][2], np.float64) for s in range(B)}
    offs = np.concatenate([[0], np.cumsum([CAPS[s] for s in inp.slots])])
    for k in range(1, 11):
        row = steps[k]
        xy, _ = step_xy(row, k, prev)
        us, _ = inp.write(torch, row, xy, rng, [(s + k) % 4 for s in inp.slots])
        write_positions(torch, g, inp.slots, pos, rng)
        graph.replay()
        out_t, moved_t = inp.twin_step(twin, "all")
        want = tw.readouts(torch, twin, pos)
        ctx = f"replay {k}"
        check_step(plan, out_t, moved_t, us, ctx)
        torch.cuda.synchronize()
        assert torch.equal(i32(planes), i32(want["layers"][:, TERRAIN].contiguous())), f"{ctx}: planes"
        for j, u in enumerate(us):
            assert torch.equal(i32(heights[offs[j]:offs[j] + u]), i32(want["height"][j][:u])), f"{ctx} scan {j}: heights"
        assert torch.equal(i32(looked_up), i32(torch.cat([s.reshape(-1) for s in want["samples"]]))), f"{ctx}: lookups"
        assert torch.equal(tallies, want["tallies"]), f"{ctx}: tallies"
        assert_readouts(ro, want, us, ctx)
        prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
    del graph
    plan.close()


def test_readouts_with_resets(monkeypatch):
    """A plan with resets and read-outs, the mask changing every step: point info and tallies are valid every step
    because the scan follows the reset, and everything equals the twin's host resets + call sequence."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    STEPS = 6
    steps = pose_steps(B, STEPS + 1, jump=0.0, seed=8300)
    rng = np.random.default_rng(83)
    init_maps(g, twin, steps)
    inp = Inputs(torch, [5, 2, 7, 0, 3, 6, 1, 4], "records")
    pos = position_tensors(torch, inp.slots)
    rx = torch.zeros((B, 3), dtype=torch.float64, device="cuda")
    rm = torch.zeros(B, dtype=torch.int32, device="cuda")
    base = dict(counts=inp.counts, xy=inp.xy, T_base_from_map=inp.T, pose_origins=inp.origins, pose_base_z=inp.base_z, moved=True,
                labels=True, select="all", index=True, reset_xyz=rx, reset_mask=rm)
    plain = g.step_plan(inp.slots, clouds=inp.buf, **base)
    k_plain = plain.kernels
    plain.close()
    plan = g.step_plan(inp.slots, clouds=inp.buf, **base, **readout_kw(torch, inp.slots, pos, "nearest"))
    tw = Twin(torch, inp.slots, "nearest")
    masks = plan_masks(STEPS)
    prev = {s: np.array(steps[0][s][2], np.float64) for s in range(B)}
    for k in range(STEPS):
        row = steps[k + 1]
        ctx = f"resets step {k}"
        xy, _ = step_xy(row, k + 1, prev)
        us, _ = inp.write(torch, row, xy, rng, [(s + k) % 4 for s in inp.slots])
        xyz = reset_poses(rng, [row[s][2] for s in inp.slots])
        rx.copy_(torch.tensor(xyz))
        rm.copy_(torch.tensor(masks[k]))
        write_positions(torch, g, inp.slots, pos, rng)
        plan.launch()
        torch.cuda.synchronize()
        twin_resets(twin, inp.slots, xyz, masks[k])
        out_t, moved_t = inp.twin_step(twin, "all")
        t0 = twin.kernel_launches
        want = tw.readouts(torch, twin, pos)
        assert plan.kernels == k_plain + twin.kernel_launches - t0, f"{ctx}: the read-outs' kernels"
        check_step(plan, out_t, moved_t, us, ctx)
        assert_readouts(plan.readouts, want, us, ctx)
        prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
    plan.close()


class Lib:
    """The library with gg_step_plan_create_with_scan_masks's read-outs replaced by `readouts`, or edited by `edit` first.
    `calls` counts the calls it intercepted."""

    def __init__(self, L, readouts=None, edit=None):
        self._L, self._r, self._edit = L, readouts, edit
        self.calls = 0

    def __getattr__(self, name):
        return getattr(self._L, name)

    def gg_step_plan_create_with_scan_masks(self, h, d, sp, r, cc, snap, ro, mask, p):
        self.calls += 1
        if self._edit is None:
            ro = self._r
        else:
            self._edit(ro._obj)
        return self._L.gg_step_plan_create_with_scan_masks(h, d, sp, r, cc, snap, ro, mask, p)


@pytest.mark.parametrize("resets", [False, True])
def test_plans_without_readouts_are_unchanged(monkeypatch, resets):
    """readouts NULL and a gg_step_readouts with nothing set give the plan gg_step_plan_create[_with_resets] gives: the
    same kernel count and the same outputs, step by step."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 4, jump=0.0, seed=8400)
    rng = np.random.default_rng(84)
    init_maps(g, twin, steps)
    for variant in (None, C.byref(capi.StepReadouts())):
        inp = Inputs(torch, list(range(B)), "records")
        extra = {}
        if resets:
            extra = dict(reset_xyz=torch.zeros((B, 3), dtype=torch.float64, device="cuda"), reset_mask=torch.zeros(B, dtype=torch.int32, device="cuda"))
        L = g._l
        g._l = shim = Lib(L, variant)
        try:
            plan = inp.plan(g, "all") if not resets else g.step_plan(inp.slots, clouds=inp.buf, counts=inp.counts, xy=inp.xy, T_base_from_map=inp.T,
                                                                     pose_origins=inp.origins, pose_base_z=inp.base_z, moved=True, labels=True,
                                                                     select="all", index=True, **extra)
        finally:
            g._l = L
        assert shim.calls == 1, f"variant {variant}: the plan was not created through the shim"
        ref = inp.plan(twin, "all") if not resets else twin.step_plan(inp.slots, clouds=inp.buf, counts=inp.counts, xy=inp.xy, T_base_from_map=inp.T,
                                                                      pose_origins=inp.origins, pose_base_z=inp.base_z, moved=True, labels=True,
                                                                      select="all", index=True, **extra)
        assert plan.kernels == ref.kernels, f"variant {variant}: kernels"
        prev = {s: np.array(steps[0][s][2], np.float64) for s in range(B)}
        for k in range(1, 4):
            xy, _ = step_xy(steps[k], k, prev)
            us, _ = inp.write(torch, steps[k], xy, rng, [(s + k) % 4 for s in inp.slots])
            plan.launch()
            ref.launch()
            check_step(plan, ref.outputs, ref.moved, us, f"variant {variant} step {k}")
            prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
        plan.close()
        ref.close()


def test_stream_contract(monkeypatch):
    """On a side stream with a sleep ahead of the launch and no host wait: work enqueued on the stream after launch sees
    the read-outs, and read-out destinations refilled on the stream before the next launch are overwritten."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 4, jump=0.0, seed=8500)
    rng = np.random.default_rng(85)
    init_maps(g, twin, steps)
    inp = Inputs(torch, list(range(B)), "records")
    pos = position_tensors(torch, inp.slots)
    kw = dict(counts=inp.counts, xy=inp.xy, T_base_from_map=inp.T, pose_origins=inp.origins, pose_base_z=inp.base_z, moved=True, labels=True,
              select="nonground", index=True, **readout_kw(torch, inp.slots, pos, "nearest"))
    plan = g.step_plan(inp.slots, clouds=inp.buf, **kw)
    ro = plan.readouts
    tw = Twin(torch, inp.slots, "nearest")
    side = torch.cuda.Stream()
    prev = {s: np.array(steps[0][s][2], np.float64) for s in range(B)}
    for k in range(4):
        row = steps[k]
        xy, _ = step_xy(row, k, prev)
        us, _ = inp.write(torch, row, xy, rng, [(s + k) % 4 for s in inp.slots])
        write_positions(torch, g, inp.slots, pos, rng)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(100_000_000)
            # destinations refilled on the stream right before the launch
            ro.layers.fill_(-5.0)
            ro.images.fill_(3)
            ro.terrain.fill_(1.5)
            for t in ro.samples + ro.codes:
                t.fill_(9)
        plan.launch(side)
        assert not side.query(), "gg_step_plan_launch waited for the stream"
        with torch.cuda.stream(side):   # consumed right after
            got = {"layers": ro.layers.clone(), "images": ro.images.clone(), "terrain": ro.terrain.clone(),
                   "samples": [t.clone() for t in ro.samples], "codes": [t.clone() for t in ro.codes],
                   "height": [t.clone() for t in ro.height], "tallies": ro.tallies.clone()}
        side.synchronize()
        out_t, _ = inp.twin_step(twin, "nonground")
        want = tw.readouts(torch, twin, pos)
        torch.cuda.synchronize()
        ctx = f"side stream step {k}"
        assert torch.equal(i32(got["layers"]), i32(want["layers"])), f"{ctx}: layers"
        assert torch.equal(got["images"], want["images"]) and torch.equal(i32(got["terrain"]), i32(want["terrain"])), f"{ctx}: images"
        assert torch.equal(got["tallies"], want["tallies"]), f"{ctx}: tallies"
        for j, u in enumerate(us):
            assert torch.equal(i32(got["samples"][j]), i32(want["samples"][j])), f"{ctx} set {j}: lookups"
            assert torch.equal(got["codes"][j][:u], want["codes"][j][:u]), f"{ctx} scan {j}: codes"
            assert torch.equal(i32(got["height"][j][:u]), i32(want["height"][j][:u])), f"{ctx} scan {j}: heights"
        prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
    plan.close()


def test_rejections(monkeypatch):
    """Each rejection of a read-out call rejects the plan with the standalone call's code, leaves no bound slot (a plain
    plan on the same slots then succeeds), gg_kernel_launches unchanged and the slots' state unchanged."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    steps = pose_steps(B, 2, jump=0.0, seed=8600)
    init_maps(g, twin, steps)
    slim = capi.GroundGridB200(99.0, 0.33, n_slots=B, max_points=MAX_POINTS)   # no full layers
    for s in range(B):
        slim.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    inp = Inputs(torch, [0, 3, 6], "records")
    rng = np.random.default_rng(86)
    inp.write(torch, steps[1], {s: np.array(steps[1][s][2]) for s in range(B)}, rng, [0, 1, 3])
    pos = position_tensors(torch, inp.slots)
    arena = g.layer_device_ptr("ground", slot=0)

    def plan(h, **kw):
        return h.step_plan(inp.slots, clouds=inp.buf, counts=inp.counts, xy=inp.xy, T_base_from_map=inp.T, pose_origins=inp.origins,
                           pose_base_z=inp.base_z, moved=True, labels=True, select="all", index=True, **kw)

    def sets(r):
        return (capi.Positions * 3).from_address(r.samples)

    def infos(r):
        return ((C.c_uint64 * 2) * 3).from_address(r.point_info)

    def shift(field, by):
        return lambda r: setattr(r, field, getattr(r, field) + by)

    def set_dst(r):
        sets(r)[1].dst = sets(r)[0].dst

    def point_into_positions(r):
        sets(r)[2].cell = sets(r)[0].data

    def share_codes(r):
        infos(r)[2][0] = infos(r)[0][0]

    def codes_on_heights(r):
        infos(r)[1][1] = infos(r)[1][0] + 8

    tallies = torch.zeros((3, 1024, 2), dtype=torch.int64, device="cuda")
    heights = dict(point_info=("codes", "height"))
    cases = {
        "unknown layer name": (g, dict(layers=("ground", "nope")), None, LAYER),
        "unknown image name": (g, dict(layer_images=("nope",)), None, LAYER),
        "unknown lookup name": (g, dict(samples=pos, sample_names=("nope",)), None, LAYER),
        "full-layers name without the flag": (slim, dict(layers=("pointsRaw",)), None, LAYER),
        "full-layers image without the flag": (slim, dict(layer_images=("m2",)), None, LAYER),
        "terrain images without the flag": (slim, dict(terrain_images=True), None, LAYER),
        "repeated name": (g, dict(layers=("ground", "variance", "ground")), None, ARG),
        "repeated lookup name": (g, dict(samples=pos, sample_names=("points", "points")), None, ARG),
        "13 names": (g, dict(layers=LAYER_NAMES + ("count", "obstacles")), None, ARG),
        "misaligned layers": (g, dict(layers=("ground",)), shift("layers", 2), ARG),
        "layers inside the arena": (g, dict(layers=("ground",)), lambda r: setattr(r, "layers", arena), ARG),
        "images inside the arena": (g, dict(layer_images=("ground",)), lambda r: setattr(r, "images", arena), ARG),
        "misaligned image ranges": (g, dict(layer_images=("ground",)), shift("image_ranges", 1), ARG),
        "misaligned terrain images": (g, dict(terrain_images=True), shift("terrain_images", 2), ARG),
        "lookups of two sets overlap": (g, dict(samples=pos), set_dst, ARG),
        "lookup cells on positions": (g, dict(samples=pos, sample_cells=True), point_into_positions, ARG),
        "unknown sample mode": (g, dict(samples=pos), lambda r: setattr(r, "sample_mode", 7), ARG),
        "codes of two slots overlap": (g, heights, share_codes, ARG),
        "codes overlap heights": (g, heights, codes_on_heights, ARG),
        "misaligned heights": (g, heights, lambda r: infos(r)[0].__setitem__(1, infos(r)[0][1] + 2), ARG),
        "heights inside the arena": (g, heights, lambda r: infos(r)[1].__setitem__(1, arena), ARG),
        "misaligned tallies": (g, dict(tallies=tallies), shift("eval_counts", 4), ARG),
    }
    for h in (g, slim):
        h.synchronize()
    for name, (h, kw, edit, want) in cases.items():
        before = h.kernel_launches
        pos_before = [h.position(slot=s).tobytes() for s in inp.slots]
        counts_before = [h.last_scan_points(slot=s) for s in inp.slots]
        L = h._l
        shim = None
        if edit is not None:
            h._l = shim = Lib(L, edit=edit)
        try:
            with pytest.raises(capi.GroundGridError) as e:
                plan(h, **kw)
        finally:
            h._l = L
        assert shim is None or shim.calls == 1, f"{name}: the edited read-outs did not reach the C call"
        assert e.value.code == want, f"{name}: {e.value}"
        assert h.kernel_launches == before, f"{name}: launches"
        assert [h.position(slot=s).tobytes() for s in inp.slots] == pos_before, f"{name}: positions"
        assert [h.last_scan_points(slot=s) for s in inp.slots] == counts_before, f"{name}: last scan points"
        # no slot is left bound: a plain plan on the same slots is accepted
        plain = plan(h)
        assert h.kernel_launches == before, f"{name}: the plain plan ran"
        plain.close()

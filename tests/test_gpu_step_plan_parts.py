"""Step plans whose step is a merged scan (gg_step_plan_create_with_parts): a multi-LiDAR rig's resets, part counts,
poses, per-part transforms, merged scans and read-outs recorded once as a CUDA graph and replayed from caller GPU memory.
Every replay is compared with a twin handle that runs the literal call sequence -- gg_init_maps_from_device,
gg_set_part_counts_from_device, gg_update_poses_from_device, gg_run_merged_cloud_msgs_to_device (host transforms of the
same values), gg_get_layers_to_device, gg_point_info_to_device, gg_eval_counts_to_device -- on the same tensors, and
must be bit-identical to it.  Records past each part's count are poison (test_gpu_merged_part_counts)."""
import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from test_gpu_cloud_msgs import map_from_sensor, payload
from test_gpu_device_outputs import make_pair, make_steps, torch_mod
from test_gpu_merged_part_counts import part_layout, sentinel, used

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
MAX_POINTS = 65536
PARTS = 4
LAYOUT = [(18, (0, 4, 8, 12, 16)), (32, (0, 4, 8, 16, 20)), (18, (0, 4, 8, 12, 16)), (22, (4, 8, 12, -1, 20))]
STEPS = 8


def caps_of(b):
    return [9000 + 1000 * b, 14000, 0 if b % 3 == 2 else 6000, 11000]   # fixed per scan: the buffers are the plan's


class RigInputs:
    """The fixed CUDA tensors of one rig plan.  host_T: parts with a fixed host transform (the others take a device
    transform rewritten every step, except part 3 of odd scans, in the map frame)."""

    def __init__(self, torch, B, counts, host_T=()):
        self.B, self.counts_on, self.host_T = B, counts, set(host_T)
        self.buf = [[torch.zeros(c * LAYOUT[p][0], dtype=torch.uint8, device="cuda") for p, c in enumerate(caps_of(b))] for b in range(B)]
        self.Tdev = torch.zeros((B, PARTS, 12), dtype=torch.float64, device="cuda")
        self.Thost = [[None] * PARTS for _ in range(B)]            # the transform of each part, as the twin passes it
        self.Tfix = [[map_from_sensor((0.0, 0.0), 0.5 * b - 0.3 * p) for p in range(PARTS)] for b in range(B)]
        self.part_counts = torch.zeros((B, PARTS), dtype=torch.int32, device="cuda")
        self.xy = torch.zeros((B, 2), dtype=torch.float64, device="cuda")
        self.T = torch.zeros((B, 12), dtype=torch.float64, device="cuda")
        self.origins = torch.zeros((B, 3), dtype=torch.float32, device="cuda")
        self.base_z = torch.zeros(B, dtype=torch.float64, device="cuda")
        self.reset_xyz = torch.zeros((B, 3), dtype=torch.float64, device="cuda")
        self.mask = torch.zeros(B, dtype=torch.int32, device="cuda")

    def frame(self, b, p):
        if p == 3 and b % 2:
            return None
        return "host" if p in self.host_T else "device"

    def plan_T(self):
        return [[self.Tdev[b, p] if self.frame(b, p) == "device" else (self.Tfix[b][p] if self.frame(b, p) == "host" else None)
                 for p in range(PARTS)] for b in range(self.B)]

    def plan(self, g, slots, tallies, select="all"):
        return g.step_plan(slots, parts=self.buf, point_step=[[s for s, _ in LAYOUT]] * self.B, field_offsets=[[o for _, o in LAYOUT]] * self.B,
                           T=self.plan_T(), origins="device", part_counts=self.part_counts if self.counts_on else None, xy=self.xy,
                           T_base_from_map=self.T, pose_origins=self.origins, pose_base_z=self.base_z, moved=True, labels=True, select=select,
                           index=True, reset_xyz=self.reset_xyz, reset_mask=self.mask, layers=("ground", "groundpatch"),
                           point_info=("codes", "height"), tallies=tallies)

    def write(self, torch, row, k, rng):
        """The next step's inputs, written into the tensors on the current stream.  Returns U per scan."""
        us, vs = [], np.zeros((self.B, PARTS), np.int32)
        Tdev = np.zeros((self.B, PARTS, 12))
        for b in range(self.B):
            pts = row[b][0]
            bounds = np.linspace(0, len(pts), PARTS + 1).astype(int)
            U = 0
            for p, c in enumerate(caps_of(b)):
                real = pts[bounds[p]:bounds[p + 1]][:c]
                if self.counts_on:
                    v, _ = part_layout(len(real), (b + 3 * p + k) % 9)
                    u = min(used(v, c), len(real))
                    v = v if used(v, c) == u else u
                else:
                    v = u = c                                  # the capacity is the count: poison included
                cloud = np.zeros(c, synth.POINT_DTYPE)
                cloud[:min(u, len(real))] = real[:u]
                cloud[min(u, len(real)):] = sentinel(pts, c - min(u, len(real)), rng)
                f = self.frame(b, p)
                if f == "device":
                    T = map_from_sensor(row[b][2], 0.2 * b + 0.6 * p + 0.05 * k)
                    Tdev[b, p] = T.reshape(12)
                else:
                    T = self.Tfix[b][p] if f == "host" else None
                self.Thost[b][p] = T
                raw = payload(cloud, LAYOUT[p][0], LAYOUT[p][1], T, rng)
                self.buf[b][p].copy_(torch.from_numpy(np.ascontiguousarray(raw).reshape(-1)))
                vs[b, p] = v
                U += u
            us.append(U)
        self.Tdev.copy_(torch.from_numpy(Tdev))
        self.part_counts.copy_(torch.from_numpy(vs))
        self.xy.copy_(torch.tensor(np.array([r[2] for r in row], np.float64)))
        self.T.copy_(torch.tensor(np.stack([r[3].reshape(12) for r in row])))
        self.origins.copy_(torch.tensor(np.array([r[1] for r in row], np.float32)))
        self.base_z.fill_(0.01 * k)
        self.reset_xyz.copy_(torch.tensor([[r[2][0], r[2][1], 0.05 * k] for r in row], dtype=torch.float64))
        self.mask.copy_(torch.from_numpy((rng.random(self.B) < 0.25).astype(np.int32)))
        return us

    def twin_step(self, twin, slots, tallies, select="all", stream=None):
        twin.init_maps_from_device(slots, self.reset_xyz, self.mask, stream=stream)
        if self.counts_on:
            twin.set_part_counts_from_device(slots, self.part_counts, stream=stream)
        moved = twin.update_poses_from_device(slots, self.xy, self.T, self.origins, self.base_z, moved=True, stream=stream)
        out = twin.run_merged_cloud_msgs_to_device(self.buf, [[s for s, _ in LAYOUT]] * self.B, [[o for _, o in LAYOUT]] * self.B, self.Thost,
                                                   slots, "device", None, labels=True, select=select, index=True, stream=stream,
                                                   device_counts=self.counts_on)
        layers = twin.get_layers_to_device(slots, ("ground", "groundpatch"), stream=stream)
        caps = [sum(caps_of(b)) for b in range(self.B)]
        codes = [torch_mod().full((c,), -7, dtype=torch_mod().int32, device="cuda") for c in caps]
        height = [torch_mod().full((c,), -7.0, dtype=torch_mod().float32, device="cuda") for c in caps]
        twin.point_info_to_device_ptrs(slots, [t.data_ptr() for t in codes], [t.data_ptr() for t in height],
                                       (stream or torch_mod().cuda.current_stream()).cuda_stream or None)
        twin.eval_counts_to_device(slots, out=tallies, stream=stream)
        return out, moved, layers, codes, height


def check_replay(plan, twin_out, us, ctx):
    torch = torch_mod()
    out_t, moved_t, layers_t, codes_t, height_t = twin_out
    torch.cuda.synchronize()
    out_g, ro = plan.outputs, plan.readouts
    assert torch.equal(plan.moved, moved_t), f"{ctx}: dev_moved"
    assert torch.equal(out_g.counts, out_t.counts), f"{ctx}: dev_counts"
    gc, gi = out_g.trimmed()
    tc, ti = out_t.trimmed()
    for k, u in enumerate(us):
        assert torch.equal(out_g.labels[k][:u], out_t.labels[k][:u]), f"{ctx} scan {k}: labels"
        assert torch.equal(gi[k], ti[k]) and torch.equal(gc[k].view(torch.int32), tc[k].view(torch.int32)), f"{ctx} scan {k}: index / cloud"
        assert torch.equal(ro.codes[k][:u], codes_t[k][:u]), f"{ctx} scan {k}: codes"
        assert torch.equal(ro.height[k][:u].view(torch.int32), height_t[k][:u].view(torch.int32)), f"{ctx} scan {k}: heights"
    assert torch.equal(ro.layers.contiguous().view(torch.int32), layers_t.contiguous().view(torch.int32)), f"{ctx}: layers"


@pytest.mark.parametrize("B,variant", [(4, "device"), (10, "device"), (4, "fixed"), (10, "mixed"), (4, "graph"), (10, "graph")])
def test_rig_plan_matches_the_call_sequence(monkeypatch, B, variant):
    """8 replays: per-part device transforms and part counts rewritten every step, device poses, resets with a seeded
    Bernoulli mask, layers, point info and tallies; batches over three stream groups."""
    torch = torch_mod()
    monkeypatch.setenv("GG_STREAMS", "3")
    g, twin = make_pair(99.0, 0.33, B, max_points=MAX_POINTS)
    slots = list(np.arange(B)[::-1])
    steps = make_steps(B, STEPS, seed=9100 + B)
    for h in (g, twin):
        for b, r in enumerate(steps[0]):
            h.init_map(r[2][0], r[2][1], 0.0, slot=b)
    inp = RigInputs(torch, B, counts=variant != "fixed", host_T=(1,) if variant == "mixed" else ())
    rng = np.random.default_rng(9100 + B)
    tallies_g = torch.zeros((B, 1024, 2), dtype=torch.int64, device="cuda")
    tallies_t = torch.zeros_like(tallies_g)
    torch.cuda.synchronize()
    plan = inp.plan(g, slots, tallies_g)
    graph = None
    if variant == "graph":
        side = torch.cuda.Stream()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            plan.launch()
    for k, row in enumerate(steps):
        us = inp.write(torch, row, k, rng)
        torch.cuda.synchronize()
        l0 = g.kernel_launches
        if graph is not None:
            graph.replay()
        else:
            plan.launch()
            assert g.kernel_launches - l0 == plan.kernels, "kernels per replay"
        want = inp.twin_step(twin, slots, tallies_t)
        check_replay(plan, want, us, f"{variant} step {k}")
        assert torch.equal(tallies_g, tallies_t), f"{variant} step {k}: tallies"
    for s in slots:
        assert g.last_scan_points(slot=int(s)) == twin.last_scan_points(slot=int(s))
        assert g.position(slot=int(s)).tobytes() == twin.position(slot=int(s)).tobytes()
    plan.close()
    g.close()
    twin.close()


def test_rejected_plans_bind_nothing_and_launch_nothing(monkeypatch):
    torch = torch_mod()
    monkeypatch.setenv("GG_STREAMS", "3")
    B = 4
    g, twin = make_pair(99.0, 0.33, B + 1, max_points=MAX_POINTS)    # slot B is never initialised
    twin.close()
    row = make_steps(B, 1, seed=9200)[0]
    for b, r in enumerate(row):
        g.init_map(r[2][0], r[2][1], 0.0, slot=b)
    slots = list(range(B))
    inp = RigInputs(torch, B, counts=True)
    inp.write(torch, row, 0, np.random.default_rng(9200))
    tallies = torch.zeros((B, 1024, 2), dtype=torch.int64, device="cuda")
    other = torch.zeros(B, dtype=torch.int32, device="cuda")
    base = torch.zeros(64, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()

    def plan(**over):
        kw = dict(parts=inp.buf, point_step=[[s for s, _ in LAYOUT]] * B, field_offsets=[[o for _, o in LAYOUT]] * B, T=inp.plan_T(),
                  origins="device", part_counts=inp.part_counts, xy=inp.xy, T_base_from_map=inp.T, pose_origins=inp.origins,
                  pose_base_z=inp.base_z, labels=True, select="all", index=True, tallies=tallies)
        kw.update(over)
        return lambda: g.step_plan(slots, **kw)

    overlap_T = inp.plan_T()
    overlap_T[0][0], overlap_T[1][0] = base[0:12], base[6:18]
    too_many = [[s[0]] for s in inp.buf]
    too_many[2] = too_many[2] * (capi.MAX_CLOUD_PARTS + 1)
    cases = {
        "device counts with parts": (plan(counts=other), ARG),
        "parts_per_slot 17": (plan(part_counts=torch.zeros((B, 17), dtype=torch.int32, device="cuda")), ARG),
        "overlapping device transforms": (plan(T=overlap_T), ARG),
        "17 parts": (plan(parts=too_many, point_step=18, field_offsets=LAYOUT[0][1], T=None), ARG),
        "repeated slot": (lambda: g.step_plan([0, 1, 1, 3], parts=inp.buf, point_step=[[s for s, _ in LAYOUT]] * B,
                                              field_offsets=[[o for _, o in LAYOUT]] * B, part_counts=inp.part_counts,
                                              origins=[r[1] for r in row], base_z=0.0), ARG),
        "map not initialised": (lambda: g.step_plan([0, 1, 2, B], parts=inp.buf, point_step=[[s for s, _ in LAYOUT]] * B,
                                                    field_offsets=[[o for _, o in LAYOUT]] * B, part_counts=inp.part_counts,
                                                    origins=[r[1] for r in row], base_z=0.0), STATE),
    }
    for name, (fn, code) in cases.items():
        l0 = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            fn()
        assert e.value.code == code, f"{name}: code {e.value.code} ({e.value})"
        assert g.kernel_launches == l0, f"{name}: something was launched"
    # nothing is bound: a valid plan on the same slots records, and a second one on one of them is refused
    p = plan()()
    l0 = g.kernel_launches
    with pytest.raises(capi.GroundGridError) as e:
        g.step_plan([3], parts=inp.buf[3:], point_step=[[s for s, _ in LAYOUT]], field_offsets=[[o for _, o in LAYOUT]], origins="device")
    assert e.value.code == STATE and g.kernel_launches == l0
    p.close()
    g.close()

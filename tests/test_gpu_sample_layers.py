"""Terrain lookups (gg_sample_layers_to_device): layer values of many slots at map-frame positions, written into
caller-owned CUDA memory and ordered on the caller's stream.  Every check is bit-exact (uint32 views) against
tests/sample_ref.py fed with gg_get_layer and gg_get_map_position of the same handle, or against the scan's own cells."""
import numpy as np
import pytest

import sample_ref
from groundgrid_b200 import capi
from test_gpu_device_outputs import DEAD, LIVE, advance, make_steps, to_device, torch_mod

pytestmark = pytest.mark.gpu

LIVE_ALL = LIVE + ("count", "obstacles")


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def make(dim, res, B, full_layers=False, max_points=65536):
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=max_points, full_layers=full_layers)
    g.res = res   # the map resolution the restatement needs
    return g


def edge_xy(g, slot, rng, m=4000):
    """float32 [m + ..., 2]: positions on both sides of cell edges near and at the map's borders, random positions over
    and beyond the map, and non-finite ones."""
    N, res = g.n, float(np.float32(g.res))
    px, py = g.position(slot)
    half = 0.5 * N * res
    i = rng.integers(-2, N + 2, m)
    edge = (px + (half - 0.5 * res) - res * i) + 0.5 * res                # the +x edge of cell i
    k = rng.integers(-2, 3, m)
    x = np.array([np.float32(e) for e in edge], np.float32)
    for _ in range(2):
        x = np.where(k > 0, np.nextafter(x, np.float32(np.inf)), np.where(k < 0, np.nextafter(x, np.float32(-np.inf)), x))
        k = k - np.sign(k)
    y = (py + rng.uniform(-half - 2, half + 2, m)).astype(np.float32)
    swap = rng.random(m) < 0.5
    x, y = np.where(swap, y - py + px, x), np.where(swap, x - px + py, y)
    special = np.array([[np.nan, py], [px, np.nan], [np.inf, py], [-np.inf, py], [px, np.inf], [px + 1e6, py],
                        [px + half, py], [px - half, py], [px, py + half], [px, py - half]], np.float32)
    return np.concatenate([np.stack([x, y], 1).astype(np.float32), special])


def as_records(xy):
    """The float32 [n, 8] view of 32-byte records with x, y in the first two columns (the rest is filler)."""
    rec = np.full((len(xy), 8), 7.25, np.float32)
    rec[:, :2] = xy
    return rec


def expected(g, slots, xys, names, mode):
    g.synchronize()
    out = []
    for s, xy in zip(slots, xys):
        planes = [g.layer(n, slot=int(s)) for n in names]
        px, py = g.position(int(s))
        out.append(sample_ref.sample_layers(planes, g.n, g.res, px, py, xy[:, 0], xy[:, 1], mode))
    return out


def check(got, cells, want, ctx):
    torch_mod().cuda.synchronize()
    for k, (v, c) in enumerate(want):
        gv = got[k].cpu().numpy()
        assert gv.shape == v.shape, f"{ctx} set {k}: shape"
        bad = np.nonzero(bits(gv) != bits(v))
        assert len(bad[0]) == 0, f"{ctx} set {k}: {len(bad[0])} values differ, first at {tuple(b[0] for b in bad)}"
        if cells is not None:
            assert np.array_equal(cells[k].cpu().numpy(), c), f"{ctx} set {k}: cells"


def positions(g, slots, row, rng, big=None):
    """One set per slot: the slot's next cloud with edge positions; float2 sets for even positions in the batch,
    32-byte records for odd ones.  Returns (host xy per set, device tensors)."""
    torch = torch_mod()
    xys, dev = [], []
    for k, s in enumerate(slots):
        pts = row[k][0]
        xy = np.concatenate([np.stack([pts["x"], pts["y"]], 1), edge_xy(g, int(s), rng)]).astype(np.float32)
        if big is not None and k == big:
            xy = np.concatenate([xy] * 2)   # more positions than the handle's max_points
        xys.append(xy)
        dev.append(torch.from_numpy(as_records(xy) if k % 2 else xy.copy()).cuda())
    return xys, dev


@pytest.mark.parametrize("dim,res,B,full_layers", [
    (99.0, 0.33, 4, True),       # N = 300, one slot per stream group
    (99.0, 0.33, 10, False),     # ten slots over eight stream groups
    (33.33, 0.33, 10, True),     # N = 101
    (33.33, 0.33, 4, False),
])
def test_matches_the_restatement_over_a_rolling_stream(dim, res, B, full_layers):
    g = make(dim, res, B, full_layers)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(8100 + B)
    name_sets = (LIVE_ALL, DEAD) if full_layers else (LIVE_ALL,)
    steps = make_steps(B, 4, seed=8100 + B)
    for k in range(3):
        row = steps[k]
        advance((g,), k, row, slots)
        order = rng.permutation(B).astype(np.int32)
        # right after the roll (the prior), then after the scan; the positions are those of the slot's next cloud
        for when in ("prior", "scan"):
            if when == "scan":
                g.run_scans_to_device([to_device(r[0]) for r in row], slots, [r[1] for r in row], 0.01 * k, labels=True, select=None)
            xys, dev = positions(g, order, [steps[k + 1][int(np.nonzero(slots == s)[0][0])] for s in order], rng,
                                 big=1 if k == 0 else None)
            for names in name_sets:
                for mode in ("nearest", "linear"):
                    got, cells = g.sample_layers_to_device(order, dev, names, mode=mode, cells=True)
                    check(got, cells, expected(g, order, xys, names, mode), f"step {k} {when} {mode} {names[0]}")
    g.close()


def test_scan_points_land_in_their_own_cells():
    """Sampling a scan's own cloud right after the scan: the cell of every rasterised point is the one the scan used,
    -1 for absent points, and the nearest ground is the layer at that cell."""
    dim, res, B = 99.0, 0.33, 4
    g = make(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    steps = make_steps(B, 2, seed=8200)
    for k, row in enumerate(steps):
        advance((g,), k, row, slots)
        dev = [to_device(r[0]) for r in row]
        g.run_scans_to_device(dev, slots, [r[1] for r in row], 0.0, labels=True, select=None)
        got, cells = g.sample_layers_to_device(slots, dev, ("ground",), cells=True)
        torch_mod().cuda.synchronize()
        for b, s in enumerate(slots):
            n = len(row[b][0])
            codes = g.point_classes(n, slot=int(s))
            c = cells[b].cpu().numpy()
            cls = codes >> 24
            assert np.array_equal(c[cls != 0], (codes[cls != 0] & 0xFFFFFF).astype(np.int32)), f"step {k} slot {s}: cells"
            assert (c[cls == 0] == -1).all(), f"step {k} slot {s}: absent points"
            ground = g.layer("ground", slot=int(s)).reshape(-1, order="F")
            v = got[b].cpu().numpy()[0]
            inside = c >= 0
            assert np.array_equal(bits(v[inside]), bits(ground[c[inside]])), f"step {k} slot {s}: ground"
            assert (bits(v[~inside]) == 0x7FC00000).all()
    g.close()


def test_points_in_a_mixed_batch_and_non_finite_layers():
    """"points" per slot in a batch that mixes scans stopped after rasterising with complete ones; layers holding NaN,
    +-inf and -0 (set through gg_set_layers_from_device); an empty set with null data."""
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 4
    g = make(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    row = make_steps(B, 1, seed=8300)[0]
    advance((g,), 0, row, slots)
    dev = [to_device(r[0]) for r in row]
    for part, stop in ((slice(0, 2), 1), (slice(2, B), 0)):
        idx = list(range(B))[part]
        descs = g.make_descs([int(slots[i]) for i in idx], [len(row[i][0]) for i in idx], [row[i][1] for i in idx], [0.0] * len(idx))
        g.run_scans_device(descs, [dev[i].data_ptr() for i in idx], stop_after=stop)
    rng = np.random.default_rng(8300)
    special = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1e38, -1e38, 1e-45], np.float32)
    names = ("ground", "groundpatch")
    imp = torch.from_numpy(rng.choice(special, (B, 2, g.n, g.n)).astype(np.float32)).cuda()
    g.set_layers_from_device(slots, names, imp)
    order = np.array([3, 0, 2, 1], np.int32)
    xys, dev_xy = positions(g, order, [row[int(s)] for s in order], rng)
    xys[2], dev_xy[2] = np.zeros((0, 2), np.float32), torch.empty((0, 2), device="cuda")
    for mode in ("nearest", "linear"):
        for nm in (("points", "ground", "groundpatch"), ("variance", "points")):
            got, cells = g.sample_layers_to_device(order, dev_xy, nm, mode=mode, cells=True)
            check(got, cells, expected(g, order, xys, nm, mode), f"{mode} {nm}")
    g.synchronize()
    assert np.array_equal(bits(g.layer("points", slot=0)), bits(g.layer("count", slot=0)))
    g.close()


@pytest.mark.parametrize("which", ["current", "side"])
def test_stream_order_without_host_waits(which):
    """(a) the call returns while the stream is busy, (b) positions produced by a torch op right before the call and
    freed and refilled right after it give the results of the original positions, (c) a clone enqueued right after
    the call sees them, (d) the slot's next scan enqueued right after the call does not change them."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 4
    g = make(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    steps = make_steps(B, 3, seed=8400)
    stream = torch.cuda.current_stream() if which == "current" else torch.cuda.Stream()
    names = ("ground", "groundpatch", "variance")
    rng = np.random.default_rng(8400)
    for k in range(2):
        advance((g,), k, steps[k], slots)
        g.run_scans_to_device([to_device(r[0]) for r in steps[k]], slots, [r[1] for r in steps[k]], 0.0, select=None)
    xys, _ = positions(g, slots, steps[2], rng)
    base = [xy - np.float32(0.5) for xy in xys]
    want = expected(g, slots, [b + np.float32(0.5) for b in base], names, "linear")   # the float32 sums the stream computes
    base = [torch.from_numpy(b).cuda() for b in base]
    nxt = [to_device(r[0]) for r in steps[2]]
    with torch.cuda.stream(stream):               # warm-up of every kernel below (module loads, allocator pools)
        pos = [b + 0.5 for b in base]
        got, _ = g.sample_layers_to_device(slots, pos, names, mode="linear", cells=True, stream=stream)
        clone = [t.clone() for t in got]
        refill = [torch.full((p.numel(),), float("nan"), device="cuda") for p in pos]
        del pos, got, clone, refill
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(400_000_000)
        before = torch.cuda.Event()
        before.record(stream)
        pos = [b + 0.5 for b in base]                 # produced on the stream right before the call
        got, cells = g.sample_layers_to_device(slots, pos, names, mode="linear", cells=True, stream=stream)
        assert not before.query(), "the call waited on the host for the stream"
        clone = [t.clone() for t in got]
        sizes = [p.numel() for p in pos]
        del pos
        refill = [torch.full((n,), float("nan"), device="cuda") for n in sizes]
        g.run_scans_to_device(nxt, slots, [r[1] for r in steps[2]], 0.0, select=None, stream=stream)
    pending = not before.query()
    torch.cuda.synchronize()
    assert pending, "the sleep did not cover the calls"
    check(got, cells, want, f"{which}: results")
    check(clone, None, want, f"{which}: clone")
    del refill
    g.close()


def test_launch_plan_one_launch_per_stream_group():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 10
    g = make(dim, res, B)
    for s in range(B):
        g.init_map(0.1 * s, 0.0, 0.0, slot=s)
    groups = sorted({s * g.n_streams // B for s in range(B)})
    xy = torch.zeros((100, 2), device="cuda")
    g.profile_enable(True)
    g.profile_read(reset=True)
    for sel, want in ((list(range(B)), len(groups)), ([0], 1), ([1, 2], 2)):
        l0 = g.kernel_launches
        g.sample_layers_to_device(sel, [xy] * len(sel), ("ground",))
        torch.cuda.synchronize()
        counts = {k: c for k, (_, c) in g.profile_read(reset=True).items() if c}
        assert counts == {"k_sample_layers": want}, f"{sel}: {counts}"
        assert g.kernel_launches - l0 == want
    # a group whose sets are all empty launches nothing; a call with only empty sets enqueues nothing
    empty = torch.zeros((0, 2), device="cuda")
    l0 = g.kernel_launches
    g.sample_layers_to_device([0, B - 1], [empty, xy], ("ground",))
    torch.cuda.synchronize()
    assert g.kernel_launches - l0 == 1
    l0 = g.kernel_launches
    g.sample_layers_to_device([0, B - 1], [empty, empty], ("ground",))
    assert g.kernel_launches == l0
    g.profile_enable(False)
    g.close()


def test_rejected_calls_enqueue_nothing():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 4
    g = make(dim, res, B)
    for s in range(3):
        g.init_map(0.0, 0.0, 0.0, slot=s)            # slot 3 has no map
    n = 64
    pos = torch.zeros((n, 8), device="cuda")
    out = torch.zeros((4, n), device="cuda")
    cell = torch.zeros(n, dtype=torch.int32, device="cuda")
    arena = g.layer_device_ptr("ground", slot=1)

    def q(**kw):
        a = np.zeros(1, capi.POSITIONS_DTYPE)
        a[0] = (pos.data_ptr(), n, 32, 0, 4, out.data_ptr(), cell.data_ptr())
        for k, v in kw.items():
            a[k][0] = v
        return a

    two = np.concatenate([q(), q(dst=out.data_ptr() + 4 * 2 * n, cell=0)])
    cases = [
        ("slot without a map", [3], q(), ("ground",), 0, -3),
        ("slot out of range", [9], q(), ("ground",), 0, -1),
        ("repeated slot", [1, 1], two, ("ground",), 0, -1),
        ("unknown name", [0], q(), ("nope",), 0, -4),
        ("expectedPoints", [0], q(), ("expectedPoints",), 0, -4),
        ("dead layer without full layers", [0], q(), ("m2",), 0, -4),
        ("repeated name", [0], q(), ("ground", "ground"), 0, -1),
        ("13 names", [0], q(), ("ground",) * 13, 0, -1),
        ("null queries", [0], None, ("ground",), 0, -1),
        ("bad mode", [0], q(), ("ground",), 2, -1),
        ("null data", [0], q(data=0), ("ground",), 0, -1),
        ("null dst", [0], q(dst=0), ("ground",), 0, -1),
        ("n > INT32_MAX", [0], q(n=2**31), ("ground",), 0, -1),
        ("point_step 4", [0], q(point_step=4), ("ground",), 0, -1),
        ("point_step 10", [0], q(point_step=10), ("ground",), 0, -1),
        ("off_x 2", [0], q(off_x=2), ("ground",), 0, -1),
        ("off_y -4", [0], q(off_y=-4), ("ground",), 0, -1),
        ("off_y outside", [0], q(off_y=32), ("ground",), 0, -1),
        ("misaligned data", [0], q(data=pos.data_ptr() + 2), ("ground",), 0, -1),
        ("misaligned dst", [0], q(dst=out.data_ptr() + 2), ("ground",), 0, -1),
        ("misaligned cell", [0], q(cell=cell.data_ptr() + 1), ("ground",), 0, -1),
        ("dst in the layers", [0], q(dst=arena), ("ground",), 0, -1),
        ("cell in the layers", [0], q(cell=arena + 400), ("ground",), 0, -1),
        ("dst over the positions", [0], q(dst=pos.data_ptr() + 64), ("ground",), 0, -1),
        ("cell over dst", [0], q(cell=out.data_ptr() + 4 * 3), ("ground",), 0, -1),
        ("dst over another set's positions", [0, 1], np.concatenate([q(), q(dst=pos.data_ptr(), cell=0)]), ("ground",), 0, -1),
        ("dst over another set's dst", [0, 1], np.concatenate([q(cell=0), q(dst=out.data_ptr() + 4 * (n - 1), cell=0)]), ("ground",), 0, -1),
    ]
    for name, sl, qs, names, mode, code in cases:
        l0 = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            g.sample_layers_to_device_ptrs(sl, qs, names, mode, None)
        assert e.value.code == code, f"{name}: code {e.value.code}: {e.value}"
        torch.cuda.synchronize()
        assert g.kernel_launches == l0, f"{name}: something was launched"
    # valid calls that do nothing
    l0 = g.kernel_launches
    g.sample_layers_to_device_ptrs([], None, ("ground",), 0, None)
    g.sample_layers_to_device_ptrs([0], q(), (), 0, None)
    g.sample_layers_to_device_ptrs([0], q(n=0, data=0, dst=0, cell=0), ("ground",), 0, None)
    # two sets may share their positions
    g.sample_layers_to_device_ptrs([0, 1], two, ("ground", "groundpatch"), 1, None)
    torch.cuda.synchronize()
    assert g.kernel_launches == l0 + 2   # slots 0 and 1 are in two stream groups
    g.close()

"""Batched layer transfer (gg_get_layers_to_device / gg_set_layers_from_device): the layers of many slots copied into /
out of one caller-owned CUDA buffer, ordered on the caller's stream.  Every check is bit-exact (uint32 views) against a
twin handle driven through the existing calls and read with gg_get_layer."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi
from test_gpu_device_outputs import LIVE, DEAD, advance, assert_state_equal, make_pair, make_steps, to_device, torch_mod

pytestmark = pytest.mark.gpu

LIVE_ALL = LIVE + ("count", "obstacles")     # every name of a live layer ("points" aliases "obstacles" after a scan)
IMPORTABLE = LIVE + ("count",)                # no name twice for one layer: an import writes each layer once
CONFIG_FIELDS = [f for f, _ in capi.Config._fields_]


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def run_both(g, twin, slots, row, base_z=0.0):
    """One scan per slot: the handle under test through gg_run_scans_to_device (labels), the twin through
    gg_run_scans_device.  Neither waits on the host."""
    dev = [to_device(r[0]) for r in row]
    g.run_scans_to_device(dev, slots, [r[1] for r in row], base_z, labels=True, select=None)
    descs = twin.make_descs(list(slots), [len(r[0]) for r in row], [r[1] for r in row], [base_z] * len(row))
    twin.run_scans_device(descs, [t.data_ptr() for t in dev])
    return dev


def check_export(exp, twin, slots, names, ctx):
    """exp: what get_layers_to_device returned, [k, l, i, j]; every plane equals the twin's gg_get_layer."""
    torch = torch_mod()
    torch.cuda.synchronize()
    got = exp.cpu().numpy()
    assert got.shape == (len(slots), len(names), twin.n, twin.n)
    for k, s in enumerate(slots):
        for l, name in enumerate(names):
            want = twin.layer(name, slot=int(s))
            assert np.array_equal(bits(got[k, l]), bits(want)), f"{ctx}: slot {s} layer {name}"


def copy_config(src, s, dst, d):
    cfg = src.get_config(slot=s)
    dst.set_config(slot=d, **{f: getattr(cfg, f) for f in CONFIG_FIELDS})


@pytest.mark.parametrize("dim,res,B,full_layers", [
    (99.0, 0.33, 4, True),       # N = 300, one slot per stream group
    (99.0, 0.33, 10, False),     # ten slots over eight stream groups
    (33.33, 0.33, 10, True),     # N = 101: N * N is odd
    (33.33, 0.33, 4, False),
])
def test_export_matches_get_layer_over_a_rolling_stream(dim, res, B, full_layers):
    g, twin = make_pair(dim, res, B, full_layers)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(6100 + B)
    batches = (LIVE_ALL, DEAD) if full_layers else (LIVE_ALL,)   # 7 + 6 names: two calls of at most 12
    steps = make_steps(B, 4, seed=6100 + B)
    for k, row in enumerate(steps[:3]):
        advance((g, twin), k, row, slots)
        run_both(g, twin, slots, row, base_z=0.02 * k)
        order = rng.permutation(B).astype(np.int32)
        exports = [g.get_layers_to_device(order, names) for names in batches]
        for names, exp in zip(batches, exports):
            check_export(exp, twin, order, names, f"step {k}")
    # the rolled prior: a roll with no scan after it
    advance((g, twin), 3, steps[3], slots)
    order = rng.permutation(B).astype(np.int32)
    check_export(g.get_layers_to_device(order), twin, order, ("ground", "groundpatch"), "rolled prior")
    # a subset of the slots, names in another order, into a caller-provided tensor
    torch = torch_mod()
    sub = order[: max(1, B // 3)]
    sub_names = ("groundpatch", "minGroundHeight", "ground")
    out = torch.full((len(sub), len(sub_names), g.n, g.n), -5.0, device="cuda").transpose(-1, -2)
    assert g.get_layers_to_device(sub, sub_names, out=out) is out
    check_export(out, twin, sub, sub_names, "subset")
    g.close()
    twin.close()


def test_points_names_the_kept_count_after_a_partial_scan():
    """"points" is resolved per slot as gg_get_layer resolves it: the kept-point count after a scan stopped after
    rasterising, the non-ground count after a complete one.  One batch mixes both."""
    dim, res, B = 33.33, 0.33, 4
    g, twin = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    row = make_steps(B, 1, seed=6150)[0]
    advance((g, twin), 0, row, slots)
    dev = [to_device(r[0]) for r in row]
    for h in (g, twin):
        for part, stop in ((slice(0, 2), 1), (slice(2, B), 0)):
            idx = list(range(B))[part]
            descs = h.make_descs([int(slots[i]) for i in idx], [len(row[i][0]) for i in idx], [row[i][1] for i in idx], [0.0] * len(idx))
            h.run_scans_device(descs, [dev[i].data_ptr() for i in idx], stop_after=stop)
    names = ("points", "count", "obstacles")
    check_export(g.get_layers_to_device(slots, names), twin, slots, names, "points alias")
    g.synchronize()
    assert np.array_equal(bits(g.layer("points", slot=0)), bits(g.layer("count", slot=0)))
    assert np.array_equal(bits(g.layer("points", slot=3)), bits(g.layer("obstacles", slot=3)))
    g.close()
    twin.close()


def test_round_trip_restores_every_layer_and_the_next_scan():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 6
    g, twin = make_pair(dim, res, B, full_layers=True)
    slots = np.arange(B, dtype=np.int32)
    names = IMPORTABLE + DEAD
    steps = make_steps(B, 3, seed=6200)
    for k, row in enumerate(steps[:2]):
        advance((g, twin), k, row, slots)
        run_both(g, twin, slots, row)
    order = slots[::-1].copy()
    exp = g.get_layers_to_device(order, names)
    sentinel = torch.full((B, len(names), g.n, g.n), 1234.5, device="cuda")
    g.set_layers_from_device(order, names, sentinel)
    g.synchronize()
    for s in (0, B - 1):
        for name in ("ground", "groundpatch", "pointsRaw"):
            assert (g.layer(name, slot=s) == 1234.5).all(), f"sentinel import: slot {s} layer {name}"
    g.set_layers_from_device(order, names, exp)
    check_export(exp, twin, order, names, "export")
    for s in slots:
        for name in names:
            assert np.array_equal(bits(g.layer(name, slot=int(s))), bits(twin.layer(name, slot=int(s)))), f"restored: slot {s} {name}"
    row = steps[2]
    advance((g, twin), 2, row, slots)
    run_both(g, twin, slots, row)
    torch.cuda.synchronize()
    assert_state_equal(g, twin, slots, row, LIVE + DEAD, "next scan after the round trip")
    g.close()
    twin.close()


def migrate_and_compare(a, c, moved, dest, steps, first, device, ctx):
    """Moves slots `moved` of `a` to slots `dest` of `c` (init_map at the position, the slot's configuration, then
    ground + groundpatch), then runs the remaining steps on both and compares every output."""
    torch = torch_mod()
    for s, d in zip(moved, dest):
        copy_config(a, int(s), c, int(d))
        x, y = a.position(int(s))
        c.init_map(x, y, 0.0, slot=int(d))
    exp = a.get_layers_to_device(moved)
    if device != a.device:
        exp = exp.to(device)
    with torch.cuda.device(device):
        c.set_layers_from_device(dest, ("ground", "groundpatch"), exp)
    B = a.n_slots
    a_slots = np.arange(B, dtype=np.int32)
    for k, row in enumerate(steps[first:], start=first):
        advance((a,), k, row, a_slots)
        mrow = [row[int(s)] for s in moved]
        c.update_pose_batch(dest, np.array([r[2] for r in mrow]), np.stack([r[3].reshape(12) for r in mrow]))
        dev_a = [to_device(r[0]) for r in row]
        out_a = a.run_scans_to_device(dev_a, a_slots, [r[1] for r in row], 0.0, labels=True, select="all", index=True)
        with torch.cuda.device(device):
            dev_c = [to_device(r[0]).to(device) for r in mrow]
            out_c = c.run_scans_to_device(dev_c, dest, [r[1] for r in mrow], 0.0, labels=True, select="all", index=True)
            torch.cuda.synchronize(device)
        torch.cuda.synchronize()
        for j, s in enumerate(moved):
            s, d = int(s), int(dest[j])
            tag = f"{ctx} step {k} slot {s} -> {d}"
            assert np.array_equal(out_a.labels[s].cpu().numpy(), out_c.labels[j].cpu().numpy()), f"{tag}: labels"
            ia, ca = a.get_output(slot=s, want_cloud=True)
            ic, cc = c.get_output(slot=d, want_cloud=True)
            assert np.array_equal(ia, ic) and ca.tobytes() == cc.tobytes(), f"{tag}: get_output"
            for name in LIVE_ALL:
                assert np.array_equal(bits(a.layer(name, slot=s)), bits(c.layer(name, slot=d))), f"{tag}: layer {name}"
            assert np.array_equal(a.position(s), c.position(d)), f"{tag}: position"


def test_migration_to_other_slots_of_another_handle_continues_bit_identically():
    dim, res, B = 99.0, 0.33, 6
    a, _ = make_pair(dim, res, B)                       # slots 1 and 5 run their own configurations
    c = capi.GroundGridB200(dim, res, n_slots=9, max_points=65536)
    steps = make_steps(B, 6, seed=6300)
    slots = np.arange(B, dtype=np.int32)
    for k, row in enumerate(steps[:3]):
        advance((a,), k, row, slots)
        dev = [to_device(r[0]) for r in row]
        a.run_scans_to_device(dev, slots, [r[1] for r in row], 0.0, labels=True, select=None)
    moved = np.array([5, 1, 2, 0], np.int32)
    dest = np.array([0, 7, 3, 8], np.int32)          # other slot numbers, other stream groups
    migrate_and_compare(a, c, moved, dest, steps, 3, 0, "same GPU")
    a.close()
    c.close()


def test_migration_across_gpus():
    torch = torch_mod()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    dim, res, B = 99.0, 0.33, 4
    a, _ = make_pair(dim, res, B)
    c = capi.GroundGridB200(dim, res, device=1, n_slots=5, max_points=65536)
    steps = make_steps(B, 5, seed=6400)
    slots = np.arange(B, dtype=np.int32)
    for k, row in enumerate(steps[:2]):
        advance((a,), k, row, slots)
        dev = [to_device(r[0]) for r in row]
        a.run_scans_to_device(dev, slots, [r[1] for r in row], 0.0, labels=True, select=None)
    migrate_and_compare(a, c, np.array([3, 1], np.int32), np.array([4, 0], np.int32), steps, 2, 1, "cuda:1")
    a.close()
    c.close()


@pytest.mark.parametrize("which", ["current", "side"])
def test_stream_order_without_host_waits(which):
    """(a) the calls return while the stream is still busy, (b) an export enqueued after a scan sees that scan's
    layers, (c) a source freed right after an import and its memory refilled on the stream does not change what was
    imported.  `current` runs on torch's current (legacy default) stream, `side` on a torch.cuda.Stream passed
    explicitly."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 4
    g, twin = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    steps = make_steps(B, 3, seed=6500)
    stream = torch.cuda.current_stream() if which == "current" else torch.cuda.Stream()
    if which == "current":
        assert stream.cuda_stream == 0
    names = LIVE_ALL
    imported = ("variance", "minGroundHeight")
    # warm-up step: module loads, allocator pools
    advance((g, twin), 0, steps[0], slots)
    run_both(g, twin, slots, steps[0])
    g.get_layers_to_device(slots, names, stream=stream)
    torch.cuda.synchronize()
    g.synchronize()
    row = steps[1]
    advance((g, twin), 1, row, slots)
    dev = [to_device(r[0]) for r in row]
    twin_descs = twin.make_descs(list(slots), [len(r[0]) for r in row], [r[1] for r in row], [0.0] * B)
    twin.run_scans_device(twin_descs, [t.data_ptr() for t in dev])
    torch.cuda.synchronize()
    shape = (B, len(imported), g.n, g.n)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(400_000_000)               # ~200 ms of device time ahead of everything below
        before = torch.cuda.Event()
        before.record(stream)
        g.run_scans_to_device(dev, slots, [r[1] for r in row], 0.0, labels=True, select=None, stream=stream)
        exp = g.get_layers_to_device(slots, names, stream=stream)
        assert not before.query(), "the export waited on the host for the stream"
        exp_clone = exp.clone()
        src = torch.full(shape, 3.5, device="cuda").transpose(-1, -2)
        g.set_layers_from_device(slots, imported, src, stream=stream)
        assert not before.query(), "the import waited on the host for the stream"
        numel = src.numel()
        del src
        refill = torch.full((numel,), float("nan"), device="cuda")
    pending = not before.query()
    torch.cuda.synchronize()
    assert pending, "the sleep did not cover the calls"
    check_export(exp, twin, slots, names, f"{which}: export after the scan")
    check_export(exp_clone, twin, slots, names, f"{which}: clone enqueued after the export")
    g.synchronize()
    for s in slots:
        for name in imported:
            assert (g.layer(name, slot=int(s)) == 3.5).all(), f"{which}: slot {s} layer {name} after the import"
            twin.set_layer(name, np.full((g.n, g.n), 3.5, np.float32), slot=int(s))
    del refill
    row = steps[2]
    advance((g, twin), 2, row, slots)
    run_both(g, twin, slots, row)
    torch.cuda.synchronize()
    assert_state_equal(g, twin, slots, row, LIVE, f"{which}: next scan")
    g.close()
    twin.close()


def test_rejected_calls_enqueue_nothing():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 4
    g, twin = make_pair(dim, res, B + 1)                  # slot B is never initialised
    slots = np.arange(B, dtype=np.int32)
    steps = make_steps(B, 2, seed=6600)
    advance((g, twin), 0, steps[0], slots)
    run_both(g, twin, slots, steps[0])
    N2 = g.n * g.n
    names = ("ground", "groundpatch")
    dst = torch.full((B + 2, 13, N2), -9.0, device="cuda")
    src = torch.full((B + 2, 13, N2), 77.0, device="cuda")
    arena = g.layer_device_ptr("ground", slot=0)
    torch.cuda.synchronize()
    g.synchronize()

    def raw(fn, count, slots_ptr, n_names, names_ptr, buf):
        rc = fn(g._h, count, slots_ptr, n_names, names_ptr, buf, None)
        if rc != 0:
            raise capi.GroundGridError(rc, g._l.gg_last_error().decode())

    two = (C.c_char_p * 2)(b"ground", b"groundpatch")
    sl = np.ascontiguousarray(slots)
    ARG, STATE, LAYER = -1, -3, -4
    cases = {
        "null slots": (ARG, lambda f, buf: raw(f, B, None, 2, two, buf)),
        "null names": (ARG, lambda f, buf: raw(f, B, sl.ctypes.data, 2, None, buf)),
        "null buffer": (ARG, lambda f, buf: raw(f, B, sl.ctypes.data, 2, two, None)),
        "count exceeds slots": (ARG, dict(slots_=list(range(B + 1)) + [0])),
        "slot out of range": (ARG, dict(slots_=[0, 1, B + 1])),
        "negative slot": (ARG, dict(slots_=[0, -1])),
        "repeated slot": (ARG, dict(slots_=[0, 2, 2])),
        "repeated name": (ARG, dict(names_=("ground", "variance", "ground"))),
        "13 names": (ARG, dict(names_=IMPORTABLE + ("m2",) * 7)),
        "misaligned buffer": (ARG, dict(offset=2)),
        "buffer in the arena": (ARG, dict(ptr=arena)),
        "buffer ends in the arena": (ARG, dict(ptr=arena - 4 * N2 * 2 + 4)),
        "unknown name": (LAYER, dict(names_=("ground", "nonsense"))),
        "dead layer": (LAYER, dict(names_=("ground", "m2"))),
        "expectedPoints": (LAYER, dict(names_=("expectedPoints",))),
        "map not initialised": (STATE, dict(slots_=[0, B])),
    }
    import_only = {"points and the layer it names": (ARG, dict(names_=("points", "obstacles")))}
    for direction, fn, buf, extra in (("get", g._l.gg_get_layers_to_device, dst, {}),
                                      ("set", g._l.gg_set_layers_from_device, src, import_only)):
        method = g.get_layers_to_device_ptrs if direction == "get" else g.set_layers_from_device_ptrs
        for name, (code, how) in {**cases, **extra}.items():
            l0 = g.kernel_launches
            with pytest.raises(capi.GroundGridError) as e:
                if callable(how):
                    how(fn, buf.data_ptr())
                else:
                    p = how.get("ptr", buf.data_ptr() + how.get("offset", 0))
                    method(how.get("slots_", [0, 1]), how.get("names_", names), p, None)
            assert e.value.code == code, f"{direction} {name}: code {e.value.code}"
            assert g.kernel_launches == l0, f"{direction} {name}: something was launched"
        # empty batches are accepted and enqueue nothing
        l0 = g.kernel_launches
        method([], names, buf.data_ptr(), None)
        method([0, 1], (), buf.data_ptr(), None)
        assert g.kernel_launches == l0, f"{direction}: an empty batch launched something"
    torch.cuda.synchronize()
    assert (dst == -9.0).all(), "a rejected export wrote into dst"
    # nothing was imported: the handle still matches its twin, before and after the next scan
    for s in slots:
        for name in LIVE_ALL:
            assert np.array_equal(bits(g.layer(name, slot=int(s))), bits(twin.layer(name, slot=int(s)))), f"slot {s} {name}"
    row = steps[1]
    advance((g, twin), 1, row, slots)
    run_both(g, twin, slots, row)
    torch.cuda.synchronize()
    assert_state_equal(g, twin, slots, row, LIVE, "after the rejected calls")
    g.close()
    twin.close()

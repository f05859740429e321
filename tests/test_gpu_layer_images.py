"""Batched layer images (gg_layer_images_to_device / gg_terrain_images_to_device): the 8-bit layer images and the terrain
image of many slots written into caller-owned CUDA memory, ordered on the caller's stream.  Every image and range is
checked bit-exact against the same handle's per-slot gg_layer_image_u8 / gg_terrain_image, and for one slot per step
against oracle/nextrows.py on the oracle's layers."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi
from oracle import Oracle, nextrows
from test_gpu_device_outputs import LIVE, DEAD, advance, make_pair, make_steps, to_device, torch_mod

pytestmark = pytest.mark.gpu

LIVE_ALL = LIVE + ("count", "obstacles")
ARG, STATE, LAYER = -1, -3, -4


def fbits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def check_images(g, slots, names, imgs, ranges, ctx):
    """imgs [k, l, i, j] / ranges [k, l, 2] equal gg_layer_image_u8 of every slot and name."""
    torch = torch_mod()
    torch.cuda.synchronize()
    got, rng = imgs.cpu().numpy(), ranges.cpu().numpy()
    assert got.shape == (len(slots), len(names), g.n, g.n) and rng.shape == (len(slots), len(names), 2)
    for k, s in enumerate(slots):
        for l, name in enumerate(names):
            want, lo, hi = g.layer_image_u8(name, slot=int(s))
            assert np.array_equal(got[k, l], want), f"{ctx}: slot {s} {name}: {int((got[k, l] != want).sum())} pixels differ"
            assert np.array_equal(fbits(rng[k, l]), fbits([lo, hi])), f"{ctx}: slot {s} {name}: range {rng[k, l]} != {(lo, hi)}"


def check_terrain(g, slots, imgs, ctx):
    torch = torch_mod()
    torch.cuda.synchronize()
    got = imgs.cpu().numpy()
    assert got.shape == (len(slots), g.n, g.n, 3)
    for k, s in enumerate(slots):
        assert np.array_equal(fbits(got[k]), fbits(g.terrain_image(slot=int(s)))), f"{ctx}: terrain of slot {s}"


def check_oracle(imgs, ranges, terrain, k, o, names, ctx, after_scan):
    """Scan k of a batch against nextrows on the oracle's layers (where the 8-bit image is defined: a finite cell).
    Between a roll and the next scan only the rolled prior is defined (INTEGRATION.md): the per-scan layers hold NaN
    strips whose contents the handle does not promise to share with the reference."""
    got, rng = imgs.cpu().numpy()[k], ranges.cpu().numpy()[k]
    for l, name in enumerate(names):
        if name in ("count", "obstacles"):   # the C-ABI's names of the two meanings of "points", not layers of the reference
            continue
        if not after_scan and name not in ("ground", "groundpatch"):
            continue
        layer = o.layer(name)
        if not np.isfinite(layer).any():
            continue
        want, lo, hi = nextrows.layer_image_u8(layer)
        assert np.array_equal(got[l], want), f"{ctx}: oracle {name}"
        assert (float(rng[l, 0]), float(rng[l, 1])) == (lo, hi), f"{ctx}: oracle range of {name}"
    if terrain is not None and after_scan:
        want = nextrows.terrain_image(o.layer("ground"), o.layer("pointsRaw"))
        assert np.array_equal(fbits(terrain.cpu().numpy()[k]), fbits(want)), f"{ctx}: oracle terrain"


@pytest.mark.parametrize("dim,res,B,full_layers", [
    (99.0, 0.33, 4, True),       # N = 300 (TMA patch detection), one slot per stream group
    (99.0, 0.33, 10, False),     # ten slots over eight stream groups
    (33.33, 0.33, 10, True),     # N = 101: N * N is odd, plain-load patch detection
    (33.33, 0.33, 4, False),
])
def test_parity_over_a_rolling_stream(dim, res, B, full_layers):
    """Every step: the images right after the roll (NaN strips, no scan in between) and after the scan, for every live
    name (and every dead one with the full layers), slots permuted.  Slots 1 and B - 1 run their own configurations;
    slot 0 runs the default one and is followed by the oracle."""
    torch = torch_mod()
    g, _ = make_pair(dim, res, B, full_layers)
    o = Oracle(dim, res)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(7100 + B)
    batches = (LIVE_ALL, DEAD) if full_layers else (LIVE_ALL,)   # at most 12 names per call
    for k, row in enumerate(make_steps(B, 3, seed=7100 + B)):
        advance((g,), k, row, slots)
        if k == 0:
            o.init_map(row[0][2][0], row[0][2][1], 0.0)
        else:
            o.update(row[0][2][0], row[0][2][1], row[0][3])
        for phase in ("after the roll", "after the scan"):
            if phase == "after the scan":
                dev = [to_device(r[0]) for r in row]
                g.run_scans_to_device(dev, slots, [r[1] for r in row], 0.02 * k, labels=True, select=None)
                o.filter_cloud(row[0][0], row[0][1], 0.02 * k, threads=1)
            order = rng.permutation(B).astype(np.int32)
            ctx = f"step {k} {phase}"
            images = [g.layer_images_to_device(order, names) for names in batches]
            terrain = g.terrain_images_to_device(order) if full_layers else None
            k0 = int(np.flatnonzero(order == 0)[0])
            for names, (imgs, ranges) in zip(batches, images):
                check_images(g, order, names, imgs, ranges, ctx)
                check_oracle(imgs, ranges, terrain if names is batches[0] else None, k0, o, names, ctx, phase == "after the scan")
            if full_layers:
                check_terrain(g, order, terrain, ctx)
    if not full_layers:
        with pytest.raises(capi.GroundGridError) as e:
            g.terrain_images_to_device(slots)
        assert e.value.code == LAYER
    # a subset into caller-provided tensors
    sub = slots[::-1][: max(1, B // 3)].copy()
    names = ("groundpatch", "minGroundHeight")
    out = torch.full((len(sub), len(names), g.n, g.n), 7, dtype=torch.uint8, device="cuda")
    ranges = torch.full((len(sub), len(names), 2), -1.0, device="cuda")
    imgs, r = g.layer_images_to_device(sub, names, out=out, ranges=ranges)
    assert imgs is out and r is ranges
    check_images(g, sub, names, out, ranges, "subset")
    g.close()


def test_points_in_a_batch_of_partial_and_complete_scans():
    dim, res, B = 33.33, 0.33, 4
    g, _ = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    row = make_steps(B, 1, seed=7150)[0]
    advance((g,), 0, row, slots)
    dev = [to_device(r[0]) for r in row]
    for part, stop in ((slice(0, 2), 1), (slice(2, B), 0)):
        idx = list(range(B))[part]
        descs = g.make_descs([int(slots[i]) for i in idx], [len(row[i][0]) for i in idx], [row[i][1] for i in idx], [0.0] * len(idx))
        g.run_scans_device(descs, [dev[i].data_ptr() for i in idx], stop_after=stop)
    names = ("points", "count", "obstacles")
    order = np.array([3, 0, 2, 1], np.int32)
    imgs, ranges = g.layer_images_to_device(order, names)
    check_images(g, order, names, imgs, ranges, "points alias")
    got = imgs.cpu().numpy()
    assert np.array_equal(got[1, 0], got[1, 1]) and np.array_equal(got[0, 0], got[0, 2])   # slot 0: count, slot 3: obstacles
    g.close()


def edge_planes(n):
    rng = np.random.default_rng(7200)
    base = rng.uniform(-2.0, 3.0, (n, n)).astype(np.float32)
    special = base.copy()
    special.flat[::7] = np.nan
    special.flat[3::11] = np.inf
    special.flat[5::13] = -np.inf
    single = np.full((n, n), np.nan, np.float32)
    single[n // 2, n // 3] = 0.625
    none = np.where(rng.random((n, n)) < 0.5, np.nan, np.inf).astype(np.float32)
    none.flat[1::2] = -np.inf
    negzero = rng.uniform(0.0, 1.0, (n, n)).astype(np.float32)
    negzero.flat[10] = -0.0
    negzero.flat[20] = 0.0
    poszero = np.abs(negzero)
    poszero.flat[30] = 0.0
    # lower 0, upper 255: pixel = trunc(x), so integers land exactly and their predecessors just below
    steps = np.zeros(n * n, np.float32)
    ints = np.arange(256, dtype=np.float32)
    below = np.nextafter(ints[1:], np.float32(0.0))
    vals = np.concatenate([ints, below, np.float32(255.0) * rng.random(n * n).astype(np.float32)])[: n * n]
    steps[:] = vals
    steps = steps.reshape(n, n, order="F")
    unit = (np.arange(n * n, dtype=np.float32) / np.float32(n * n - 1)).reshape(n, n)   # upper hits 255 exactly
    return {
        "special": special, "constant": np.full((n, n), 1.5, np.float32), "no finite cell": none, "single finite": single,
        "-0 minimum": negzero, "+0 minimum": poszero, "quantisation": steps, "unit ramp": unit,
    }


def test_edge_planes():
    dim, res = 33.33, 0.33
    g = capi.GroundGridB200(dim, res, n_slots=3, max_points=16384, full_layers=True)
    for s in range(3):
        g.init_map(0.0, 0.0, 0.0, slot=s)
    planes = edge_planes(g.n)
    names = ("ground", "groundpatch", "variance", "minGroundHeight", "m2", "meanVariance", "pointsRaw", "planeDist")
    assign = {}
    for q, (what, plane) in enumerate(planes.items()):
        slot, name = (0, 2)[q % 2], names[q]
        g.set_layer(name, plane, slot=slot)
        assign[(slot, name)] = what
    rng = np.random.default_rng(7201)
    g.set_layer("pointsRaw", rng.integers(0, 7, (g.n, g.n)).astype(np.float32), slot=1)
    g.set_layer("ground", planes["special"], slot=1)
    order = np.array([2, 0, 1], np.int32)
    imgs, ranges = g.layer_images_to_device(order, names)
    check_images(g, order, names, imgs, ranges, "edge planes")
    got, rg = imgs.cpu().numpy(), ranges.cpu().numpy()
    for k, s in enumerate(order):
        for l, name in enumerate(names):
            what = assign.get((int(s), name))
            if what is None:
                continue
            plane = planes[what]
            if what == "no finite cell":
                assert (got[k, l] == 0).all() and (rg[k, l] == [np.inf, -np.inf]).all(), what
                continue
            if what == "-0 minimum":
                assert fbits(rg[k, l])[0] == 0x80000000, "-0 sorts below +0"
            if what == "constant":
                assert (got[k, l] == 0).all(), "0 / 0 gives 0"
            if what == "quantisation":
                assert got[k, l].max() == 255
            want, lo, hi = nextrows.layer_image_u8(plane)
            if not what.endswith("minimum"):   # nextrows does not define the sign of a zero minimum
                assert (float(rg[k, l, 0]), float(rg[k, l, 1])) == (lo, hi), what
            assert np.array_equal(got[k, l], want), f"{what}: {int((got[k, l] != want).sum())} pixels differ from nextrows"
    terrain = g.terrain_images_to_device(order)
    check_terrain(g, order, terrain, "edge planes")
    t = terrain.cpu().numpy()
    want = nextrows.terrain_image(g.layer("ground", slot=1), g.layer("pointsRaw", slot=1))
    assert np.array_equal(fbits(t[2]), fbits(want)) and t[2][:, :, 1].sum() > 0
    g.close()


@pytest.mark.parametrize("which", ["current", "side"])
def test_stream_order_without_host_waits(which):
    """(a) the calls return while the stream is still busy, (b) images enqueued right after a scan see that scan,
    (c) a clone enqueued right after the call sees the images, (d) a dst freed right after the call and its memory
    refilled on the stream keeps the refill."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 4
    g, _ = make_pair(dim, res, B, full_layers=True)
    slots = np.arange(B, dtype=np.int32)
    steps = make_steps(B, 2, seed=7300)
    stream = torch.cuda.current_stream() if which == "current" else torch.cuda.Stream()
    if which == "current":
        assert stream.cuda_stream == 0
    names = LIVE_ALL

    def enqueue(row, before):
        """The scan, the images, their clones, and a second set of images freed and refilled right away."""
        def busy(what):
            assert before is None or not before.query(), f"{what} waited on the host for the stream"

        dev = [to_device(r[0]) for r in row]
        with torch.cuda.stream(stream):
            if before is not None:
                torch.cuda._sleep(400_000_000)               # ~200 ms of device time ahead of everything below
                before.record(stream)
            g.run_scans_to_device(dev, slots, [r[1] for r in row], 0.0, labels=True, select=None, stream=stream)
            imgs, ranges = g.layer_images_to_device(slots, names, stream=stream)
            busy("gg_layer_images_to_device")
            terrain = g.terrain_images_to_device(slots, stream=stream)
            busy("gg_terrain_images_to_device")
            clones = imgs.clone(), ranges.clone(), terrain.clone()
            freed, freed_r = g.layer_images_to_device(slots, names, stream=stream)
            freed_t = g.terrain_images_to_device(slots, stream=stream)
            busy("the second images")
            sizes = (freed.numel(), freed_t.numel())
            del freed, freed_r, freed_t
            refill = torch.full((sizes[0],), 0xAB, dtype=torch.uint8, device="cuda")
            refill_t = torch.full((sizes[1],), -3.25, device="cuda")
            busy("the refill")
        return imgs, ranges, terrain, clones, refill, refill_t

    # warm-up with the same sequence: module loads, allocator pools, the range scratch
    advance((g,), 0, steps[0], slots)
    enqueue(steps[0], None)
    torch.cuda.synchronize()
    g.synchronize()
    advance((g,), 1, steps[1], slots)
    torch.cuda.synchronize()
    before = torch.cuda.Event()
    imgs, ranges, terrain, clones, refill, refill_t = enqueue(steps[1], before)
    pending = not before.query()
    torch.cuda.synchronize()
    assert pending, "the sleep did not cover the calls"
    check_images(g, slots, names, imgs, ranges, f"{which}: images after the scan")
    check_terrain(g, slots, terrain, f"{which}: terrain after the scan")
    check_images(g, slots, names, clones[0], clones[1], f"{which}: clone")
    check_terrain(g, slots, clones[2], f"{which}: terrain clone")
    assert (refill == 0xAB).all() and (refill_t == -3.25).all(), f"{which}: a freed dst was written after the refill"
    g.close()


def test_rejected_calls_enqueue_nothing():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 4
    g, twin = make_pair(dim, res, B + 1, full_layers=True)   # slot B is never initialised
    slots = np.arange(B, dtype=np.int32)
    row = make_steps(B, 1, seed=7400)[0]
    for h in (g, twin):
        advance((h,), 0, row, slots)
        dev = [to_device(r[0]) for r in row]
        h.run_scans_to_device(dev, slots, [r[1] for r in row], 0.0, labels=True, select=None)
    N2 = g.n * g.n
    names = ("ground", "groundpatch")
    dst = torch.full((B + 2, 13, N2), 0x5A, dtype=torch.uint8, device="cuda")
    rng_buf = torch.full((B + 2, 13, 2), -9.0, device="cuda")
    tdst = torch.full((B + 2, N2 * 3), -9.0, device="cuda")
    arena = g.layer_device_ptr("ground", slot=0)
    torch.cuda.synchronize()
    g.synchronize()
    two = (C.c_char_p * 2)(b"ground", b"groundpatch")
    sl = np.ascontiguousarray(slots)
    D, R = dst.data_ptr(), rng_buf.data_ptr()

    def images(slots_=(0, 1), names_=names, d=D, r=R):
        g.layer_images_to_device_ptrs(list(slots_), names_, d, r, None)

    def raw_images(count, slots_ptr, n_names, names_ptr, d, r):
        rc = g._l.gg_layer_images_to_device(g._h, count, slots_ptr, n_names, names_ptr, d, r, None)
        if rc != 0:
            raise capi.GroundGridError(rc, g._l.gg_last_error().decode())

    def terrain(slots_=(0, 1), d=tdst.data_ptr()):
        g.terrain_images_to_device_ptrs(list(slots_), d, None)

    cases = {
        "null slots": (ARG, lambda: raw_images(B, None, 2, two, D, R)),
        "null names": (ARG, lambda: raw_images(B, sl.ctypes.data, 2, None, D, R)),
        "null dst": (ARG, lambda: raw_images(B, sl.ctypes.data, 2, two, None, R)),
        "count exceeds slots": (ARG, lambda: images(list(range(B + 1)) + [0])),
        "slot out of range": (ARG, lambda: images([0, 1, B + 1])),
        "negative slot": (ARG, lambda: images([0, -1])),
        "repeated slot": (ARG, lambda: images([0, 2, 2])),
        "repeated name": (ARG, lambda: images(names_=("ground", "variance", "ground"))),
        "13 names": (ARG, lambda: images(names_=LIVE_ALL + DEAD)),
        "misaligned dev_range": (ARG, lambda: images(r=R + 2)),
        "dst in the arena": (ARG, lambda: images(d=arena)),
        "dst ends in the arena": (ARG, lambda: images(d=arena - 2 * N2 * 2 + 1)),
        "dev_range in the arena": (ARG, lambda: images(r=arena + 64)),
        "dst overlaps dev_range": (ARG, lambda: images(r=D + 4 * N2 - 8)),
        "dev_range overlaps dst": (ARG, lambda: images(d=R - 2 * N2 + 1)),
        "unknown name": (LAYER, lambda: images(names_=("ground", "nonsense"))),
        "expectedPoints": (LAYER, lambda: images(names_=("expectedPoints",))),
        "map not initialised": (STATE, lambda: images([0, B])),
        "terrain: null dst": (ARG, lambda: terrain(d=None)),
        "terrain: misaligned dst": (ARG, lambda: terrain(d=tdst.data_ptr() + 2)),
        "terrain: dst in the arena": (ARG, lambda: terrain(d=arena)),
        "terrain: repeated slot": (ARG, lambda: terrain([1, 1])),
        "terrain: slot out of range": (ARG, lambda: terrain([0, B + 1])),
        "terrain: map not initialised": (STATE, lambda: terrain([B])),
    }
    for name, (code, call) in cases.items():
        l0 = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            call()
        assert e.value.code == code, f"{name}: code {e.value.code}"
        assert g.kernel_launches == l0, f"{name}: something was launched"
    # a dead layer and the terrain image need the full layers
    lean = capi.GroundGridB200(dim, res, n_slots=2, max_points=16384)
    lean.init_map(0.0, 0.0, 0.0, slot=0)
    for name, call in (("dead layer", lambda: lean.layer_images_to_device_ptrs([0], ("ground", "m2"), D, R, None)),
                       ("terrain", lambda: lean.terrain_images_to_device_ptrs([0], tdst.data_ptr(), None))):
        l0 = lean.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            call()
        assert e.value.code == LAYER, f"lean {name}: code {e.value.code}"
        assert lean.kernel_launches == l0, f"lean {name}: something was launched"
    lean.close()
    # empty batches are accepted and enqueue nothing; dev_range may be null
    l0 = g.kernel_launches
    images([])
    images(names_=())
    terrain([])
    assert g.kernel_launches == l0, "an empty batch launched something"
    torch.cuda.synchronize()
    assert (dst == 0x5A).all() and (rng_buf == -9.0).all() and (tdst == -9.0).all(), "a rejected call wrote into a buffer"
    images(r=None)
    torch.cuda.synchronize()
    assert (rng_buf == -9.0).all()
    want = [g.layer_image_u8(n_, slot=s)[0] for s in (0, 1) for n_ in names]
    got = dst.cpu().numpy()[0, :4].reshape(4, -1)[:, :N2]
    assert all(np.array_equal(got[q].reshape(g.n, g.n), want[q]) for q in range(4)), "dev_range = NULL"
    # the layers are the twin's
    g.synchronize()
    for s in slots:
        for n_ in LIVE_ALL + DEAD:
            assert np.array_equal(fbits(g.layer(n_, slot=int(s))), fbits(twin.layer(n_, slot=int(s)))), f"slot {s} {n_}"
    g.close()
    twin.close()

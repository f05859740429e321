"""Map snapshots in caller GPU memory (gg_save_maps_to_device, gg_restore_maps_from_device, and their stages in
gg_step_plan_create_with_snapshots).  A stream saved after k steps and restored elsewhere -- other slots, another
handle, another GPU, a round trip through a file -- must continue bit-identically to the uninterrupted stream; a restore
must equal host gg_init_map + gg_set_layer("ground") + gg_set_layer("groundpatch") on a twin; slots whose index is out
of range or whose record is rejected must come out bit-unchanged."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi
from test_gpu_device_counts import MAX_POINTS, assert_twin
from test_gpu_device_outputs import DEAD, LIVE, make_pair, to_device, torch_mod
from test_gpu_device_poses import pose_steps
from test_gpu_map_resets import assert_layers, assert_positions, bits
from test_gpu_step_plans import CAPS, Inputs, check_step, step_xy

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
B, GROUPS = 8, 3


def handles(monkeypatch, dim=99.0, res=0.33, full_layers=False):
    monkeypatch.setenv("GG_STREAMS", str(GROUPS))
    g, twin = make_pair(dim, res, B, full_layers=full_layers, max_points=MAX_POINTS)
    assert g.n_streams == GROUPS == twin.n_streams
    return g, twin


def scan_step(h, slots, row, mode, rows_of=None):
    """One roll + scan of `slots`, each following the stream rows_of[k] of `row` (default: its own slot): host poses
    (update_pose + host origins) or device poses (update_poses_from_device + GG_SCAN_DEVICE_POSE).  Returns the labels."""
    torch = torch_mod()
    src = list(slots) if rows_of is None else list(rows_of)
    if mode == "host":
        for s, r in zip(slots, src):
            h.update_pose(row[r][2][0], row[r][2][1], row[r][3], slot=int(s))
        origins, base_z = [row[r][1] for r in src], [row[r][4] for r in src]
    else:
        h.update_poses_from_device(list(slots), torch.tensor(np.array([row[r][2] for r in src], np.float64), device=f"cuda:{h.device}"),
                                   torch.tensor(np.stack([row[r][3].reshape(12) for r in src]), device=f"cuda:{h.device}"),
                                   torch.tensor(np.array([row[r][1] for r in src], np.float32), device=f"cuda:{h.device}"),
                                   torch.tensor(np.array([row[r][4] for r in src], np.float64), device=f"cuda:{h.device}"))
        origins, base_z = "device", None
    clouds = [to_device(row[r][0]).to(f"cuda:{h.device}") for r in src]
    out = h.run_scans_to_device(clouds, list(slots), origins, base_z, labels=True, select="all", index=True)
    torch.cuda.synchronize(h.device)
    return [out.labels[k].cpu().numpy() for k in range(len(src))]


def state_of(h, slots, names):
    return {(int(s), n): bits(h.layer(n, slot=int(s))) for s in slots for n in names}, {int(s): bits(h.position(slot=int(s))) for s in slots}


@pytest.mark.parametrize("target", ["other_slots", "second_handle", "cuda1", "file"])
@pytest.mark.parametrize("mode", ["host", "device"])
def test_continuation(monkeypatch, tmp_path, mode, target):
    """Slots 0-3 run k steps, are saved, and run m more steps; the saved records restored into slots 4-7 of the same
    handle, into a second handle (on cuda:1 for "cuda1"), or through host memory and a file, then run the same m steps:
    labels, every layer and the positions are bit-identical to the uninterrupted run."""
    torch = torch_mod()
    if target == "cuda1" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    monkeypatch.setenv("GG_STREAMS", str(GROUPS))
    g = capi.GroundGridB200(99.0, 0.33, n_slots=B, max_points=MAX_POINTS, full_layers=True)
    K, M = 4, 3
    steps = pose_steps(4, K + M, jump=0.0, seed=7600)
    src = [0, 1, 2, 3]
    for s in src:
        g.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    for k in range(1, K):
        scan_step(g, src, steps[k], mode)
    snap = g.save_maps_to_device(src)
    if target == "other_slots":
        h, dst = g, [6, 4, 7, 5]
    else:
        h = capi.GroundGridB200(99.0, 0.33, device=1 if target == "cuda1" else 0, n_slots=5, max_points=MAX_POINTS, full_layers=True)
        dst = [4, 0, 3, 1]
    if target == "file":
        path = tmp_path / "maps.npy"
        np.save(path, snap.cpu().numpy())
        pool = torch.from_numpy(np.load(path)).to(f"cuda:{h.device}")
    else:
        pool = snap.to(f"cuda:{h.device}")
    for s in dst:
        h.init_map(-50.0, 20.0, 3.0, slot=s)        # any map: the restore replaces it
    status = h.restore_maps_from_device(dst, pool, status=True)
    assert status.tolist() == [1] * 4
    names = LIVE + DEAD
    for k in range(K, K + M):
        want = scan_step(g, src, steps[k], mode)
        got = scan_step(h, dst, steps[k], mode, rows_of=src)
        for j in range(4):
            assert np.array_equal(got[j], want[j]), f"{mode} {target} step {k} slot {dst[j]}: labels"
    for s, d in zip(src, dst):
        for n in names:
            assert np.array_equal(bits(h.layer(n, slot=d)), bits(g.layer(n, slot=s))), f"{mode} {target} slot {d}: {n}"
        assert bits(h.position(slot=d)).tolist() == bits(g.position(slot=s)).tolist(), f"{mode} {target} slot {d}: position"
    # a second save of the continued streams gives byte-identical records
    assert torch.equal(h.save_maps_to_device(dst).cpu(), g.save_maps_to_device(src).cpu()), f"{mode} {target}: records"


def crafted_planes(rng, n):
    """ground / groundpatch with NaN payloads, +-inf, -0, denormals and ordinary values (column-major N x N)."""
    out = []
    for _ in range(2):
        a = rng.uniform(-5.0, 5.0, n * n).astype(np.float32)
        w = a.view(np.uint32)
        w[::7] = 0x7FC01234                 # quiet NaN with a payload
        w[3::11] = 0xFF812345               # negative signalling NaN with a payload
        w[1::13] = 0x7F800000               # +inf
        w[2::17] = 0xFF800000               # -inf
        w[5::19] = 0x80000000               # -0
        w[6::23] = 0x00000003               # denormal
        out.append(a.reshape(n, n, order="F"))
    return out


def expected_record(n, res, px, py, G, Cp):
    """The record the header describes, built on the host."""
    n2 = n * n
    n2p = (n2 + 3) // 4 * 4
    rec = np.zeros(capi.snapshot_bytes(n), np.uint8)
    hdr = capi.MapSnapshot(capi.SNAPSHOT_MAGIC, capi.SNAPSHOT_VERSION, n, res)
    hdr.position[0], hdr.position[1] = px, py
    rec[:64] = np.frombuffer(bytes(hdr), np.uint8)
    planes = rec[64:].view(np.uint32)
    planes[:n2] = G.reshape(-1, order="F").view(np.uint32)
    planes[n2p:n2p + n2] = Cp.reshape(-1, order="F").view(np.uint32)
    return rec


GEOMETRIES = {"n300": (99.0, 0.33), "odd_n55": (18.15, 0.33)}


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
@pytest.mark.parametrize("full_layers", [False, True])
def test_host_twin(monkeypatch, geometry, full_layers):
    """Records saved from crafted states (far-from-origin positions; host-owned, device-rolled and device-reset
    positions; non-finite and signed-zero planes) are the host-built records byte for byte, padding 0 included; restored
    into other slots they equal host gg_init_map + gg_set_layer x 2 on the twin: every layer and the position."""
    torch = torch_mod()
    dim, res = GEOMETRIES[geometry]
    g, twin = handles(monkeypatch, dim, res, full_layers)
    n = g.n
    assert (n * n % 4 != 0) == (geometry == "odd_n55")
    names = LIVE + DEAD if full_layers else LIVE
    rng = np.random.default_rng(77)
    src = [0, 3, 6]
    pos = {0: (1.0e7 + 0.123456789, -3.5e6 - 0.987654321), 3: (-0.33, 12.5), 6: (123456.789, -98765.4321)}
    planes = {s: crafted_planes(rng, n) for s in src}
    for s in src:
        g.init_map(pos[s][0], pos[s][1], 0.25, slot=s)
        g.set_layer("ground", planes[s][0], slot=s)
        g.set_layer("groundpatch", planes[s][1], slot=s)
    # slot 3: device-owned by a roll to where it is (no cell shift); slot 6: device-owned by a reset at its position
    T = np.eye(4)[:3].reshape(12)
    assert g.update_poses_from_device([3], torch.tensor([pos[3]], dtype=torch.float64, device="cuda"),
                                      torch.tensor(T[None], device="cuda"), moved=True).tolist() == [0]
    g.init_maps_from_device([6], torch.tensor([[pos[6][0], pos[6][1], 0.25]], dtype=torch.float64, device="cuda"))
    g.set_layers_from_device([6], ["ground", "groundpatch"],
                             torch.tensor(np.stack(planes[6])[None], device="cuda"))
    snap = g.save_maps_to_device(src).cpu().numpy()
    for k, s in enumerate(src):
        want = expected_record(n, res, pos[s][0], pos[s][1], planes[s][0], planes[s][1])
        assert np.array_equal(snap[k], want), f"slot {s}: record bytes"
    dst = [7, 1, 4]
    for h in (g, twin):
        for s in dst:
            h.init_map(5.0, -5.0, 1.0, slot=s)
    g.restore_maps_from_device(dst, torch.tensor(snap, device="cuda"))
    for s, d in zip(src, dst):
        twin.init_map(pos[s][0], pos[s][1], -7.5, slot=d)
        twin.set_layer("ground", planes[s][0], slot=d)
        twin.set_layer("groundpatch", planes[s][1], slot=d)
    assert_layers(g, twin, dst, names, f"{geometry} full={full_layers}")
    assert_positions(g, twin, dst, f"{geometry} full={full_layers}")


def test_index_status_and_masks(monkeypatch):
    """Out-of-range and negative indices leave the slot bit-unchanged (status 0); one record restored into many slots;
    a corrupted magic or version, and a record of another N or resolution, give status -1 and leave the slot unchanged;
    masked-off save records stay untouched."""
    torch = torch_mod()
    g, twin = handles(monkeypatch, full_layers=False)
    rng = np.random.default_rng(78)
    n = g.n
    for s in range(B):
        g.init_map(2.0 * s, -1.0 * s, 0.1 * s, slot=s)
        G, Cp = crafted_planes(rng, n)
        g.set_layer("ground", G, slot=s)
        g.set_layer("groundpatch", Cp, slot=s)
    pool = g.save_maps_to_device([1, 5, 2])          # records 0, 1, 2
    bad = pool[:1].clone().repeat(4, 1)              # records 3-6: rejected copies of record 0
    bad[0, 0] ^= 1                                   # magic
    bad[1, 4] = 2                                    # version
    bad[2, 8:12] = torch.tensor(np.array([n + 1], np.int32).view(np.uint8), device="cuda")   # cells_per_side
    other = capi.GroundGridB200(49.5, 0.165, n_slots=1, max_points=1000)   # same N, another resolution
    assert other.n == n and other.snapshot_bytes == g.snapshot_bytes
    other.init_map(0.0, 0.0, 0.0)
    bad[3] = other.save_maps_to_device([0])[0]
    pool = torch.cat([pool, bad]).contiguous()
    slots = [0, 1, 2, 3, 4, 5, 6, 7]
    index = [-1, 7, 2, 2, 3, 4, 5, 6]                # 7 == n_pool: out of range; 2 twice: a broadcast
    index[0] = -(2 ** 31)
    before = state_of(g, range(B), LIVE)
    status = g.restore_maps_from_device(slots, pool, torch.tensor(index, dtype=torch.int32, device="cuda"), status=True)
    assert status.tolist() == [0, 0, 1, 1, -1, -1, -1, -1]
    after = state_of(g, range(B), LIVE)
    for k, s in enumerate(slots):
        if status[k] != 1:
            for nm in LIVE:
                assert np.array_equal(after[0][(s, nm)], before[0][(s, nm)]), f"slot {s}: {nm} changed"
            assert after[1][s].tolist() == before[1][s].tolist(), f"slot {s}: position changed"
        else:
            for nm in ("ground", "groundpatch"):
                assert np.array_equal(after[0][(s, nm)], before[0][([1, 5, 2][index[k]], nm)]), f"slot {s}: {nm}"
    # the save mask: masked-off records keep their bytes
    out = torch.full((B, g.snapshot_bytes), 0xAB, dtype=torch.uint8, device="cuda")
    mask = torch.tensor([1, 0, 0, 1, 0, 1, 1, 0], dtype=torch.int32, device="cuda")
    g.save_maps_to_device(slots, mask=mask, out=out)
    full = g.save_maps_to_device(slots)
    for k in range(B):
        if mask[k]:
            assert torch.equal(out[k], full[k]), f"record {k}"
        else:
            assert bool((out[k] == 0xAB).all()), f"record {k} touched"


def test_odd_padding_and_empty_pool(monkeypatch):
    """On an odd N the padding floats of both planes are 0; an empty pool restores nothing (status 0)."""
    torch = torch_mod()
    g, _ = handles(monkeypatch, 18.15, 0.33)
    n = g.n
    n2, n2p = n * n, (n * n + 3) // 4 * 4
    assert n2 != n2p
    for s in range(2):
        g.init_map(0.0, 0.0, 1.0, slot=s)
        g.set_layer("ground", np.full((n, n), np.nan, np.float32), slot=s)
        g.set_layer("groundpatch", np.full((n, n), -np.inf, np.float32), slot=s)
    out = torch.full((2, g.snapshot_bytes), 0xCD, dtype=torch.uint8, device="cuda")
    g.save_maps_to_device([0, 1], out=out)
    w = out.cpu().numpy()[:, 64:].view(np.uint32)
    assert (w[:, n2:n2p] == 0).all() and (w[:, n2p + n2:] == 0).all()
    before = state_of(g, [0], LIVE)
    st = g.restore_maps_from_device([0], torch.empty((0, g.snapshot_bytes), dtype=torch.uint8, device="cuda"), status=True)
    assert st.tolist() == [0]
    after = state_of(g, [0], LIVE)
    assert all(np.array_equal(after[0][k], before[0][k]) for k in before[0])


@pytest.mark.parametrize("capture", [False, True])
def test_plan_with_restore_and_save(monkeypatch, capture):
    """step_plan(..., restore_pool, restore_index, restore_status, save, save_mask) with the index and the mask rewritten
    before every replay and the pool refilled from the previous step's saves, plain or captured in torch.cuda.graph:
    each replay equals the literal call sequence restore -> counts -> poses -> scan -> save on the twin."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    STEPS = 6
    steps = pose_steps(B, STEPS + 1, jump=0.0, seed=7700)
    rng = np.random.default_rng(79)
    for h in (g, twin):
        for s in range(B):
            h.init_map(steps[0][s][2][0], steps[0][s][2][1], 0.0, slot=s)
    inp = Inputs(torch, [5, 2, 7, 0, 3, 6], "records")
    n = len(inp.slots)
    pool = g.save_maps_to_device(inp.slots)
    assert torch.equal(pool, twin.save_maps_to_device(inp.slots))
    idx = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    sm = torch.zeros(n, dtype=torch.int32, device="cuda")
    plain = inp.plan(g, "all")
    k_plain = plain.kernels
    plain.close()
    kw = dict(counts=inp.counts, xy=inp.xy, T_base_from_map=inp.T, pose_origins=inp.origins, pose_base_z=inp.base_z, moved=True,
              labels=True, select="all", index=True)
    plan = g.step_plan(inp.slots, clouds=inp.buf, restore_pool=pool, restore_index=idx, restore_status=True, save=True, save_mask=sm, **kw)
    assert plan.kernels == k_plain + 2 * GROUPS
    twin_saved = torch.zeros_like(plan.saved)
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
        index = rng.integers(-2, n + 2, n).astype(np.int32)
        index[k % n] = (k + 1) % n                     # at least one slot restores every step
        mask = (rng.random(n) < 0.5).astype(np.int32)
        idx.copy_(torch.tensor(index))
        sm.copy_(torch.tensor(mask))
        g0 = g.kernel_launches
        if capture:
            graph.replay()
        else:
            plan.launch()
            assert g.kernel_launches - g0 == plan.kernels, ctx
        torch.cuda.synchronize()
        st = twin.restore_maps_from_device(inp.slots, pool, idx, status=True)
        out_t, moved_t = inp.twin_step(twin, "all")
        twin.save_maps_to_device(inp.slots, mask=sm, out=twin_saved)
        torch.cuda.synchronize()
        check_step(plan, out_t, moved_t, us, ctx)
        assert torch.equal(plan.restore_status, st), f"{ctx}: status"
        assert torch.equal(plan.saved, twin_saved), f"{ctx}: saved records"
        pool.copy_(torch.where(sm[:, None] != 0, plan.saved, pool))   # the next step restores from this step's saves
        prev = {s: (xy[s] if np.all(np.isfinite(xy[s])) else prev[s]) for s in range(B)}
    assert_twin(g, twin, inp.slots, us, [CAPS[s] for s in inp.slots], f"capture={capture} end")
    assert_positions(g, twin, range(B), f"capture={capture} end")
    # standalone calls on bound slots are accepted
    sel = inp.slots[:3]
    st_g = g.restore_maps_from_device(sel, pool, torch.tensor([2, 0, 1], dtype=torch.int32, device="cuda"), status=True)
    st_t = twin.restore_maps_from_device(sel, pool, torch.tensor([2, 0, 1], dtype=torch.int32, device="cuda"), status=True)
    assert torch.equal(st_g, st_t) and st_g.tolist() == [1, 1, 1]
    assert torch.equal(g.save_maps_to_device(inp.slots), twin.save_maps_to_device(inp.slots))
    assert_layers(g, twin, inp.slots, LIVE, "bound slots")
    del graph
    plan.close()


def test_stream_contract(monkeypatch):
    """Pool and index produced on a side stream behind a sleep, the calls on that stream returning before it gets there,
    and both overwritten on the stream right after the restore: the restore uses the values of the call, and a save
    enqueued after it sees the restored maps."""
    torch = torch_mod()
    g, twin = handles(monkeypatch)
    for h in (g, twin):
        for s in range(B):
            h.init_map(1.5 * s, -0.5 * s, 0.3 * s, slot=s)
    src = g.save_maps_to_device([6, 7])
    pool = torch.zeros_like(src)
    idx = torch.zeros(4, dtype=torch.int32, device="cuda")
    want_idx = torch.tensor([1, 0, 1, 5], dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        pool.copy_(src)
        idx.copy_(want_idx)
    g.restore_maps_from_device([0, 1, 2, 3], pool, idx, stream=side)
    saved = g.save_maps_to_device([0, 1, 2, 3], stream=side)
    assert not side.query(), "the snapshot calls waited for the stream"
    with torch.cuda.stream(side):
        pool.fill_(0x55)
        idx.fill_(0)
    side.synchronize()
    twin.restore_maps_from_device([0, 1, 2, 3], src, want_idx)
    assert_layers(g, twin, range(B), LIVE, "stream contract")
    assert_positions(g, twin, range(B), "stream contract")
    assert torch.equal(saved, twin.save_maps_to_device([0, 1, 2, 3]))


def test_rejections_enqueue_nothing(monkeypatch):
    """Every GG_E_ARG / GG_E_STATE of both calls and of a plan whose snapshot stage is rejected leaves
    gg_kernel_launches unchanged; count 0 succeeds and enqueues nothing."""
    torch = torch_mod()
    g, _ = handles(monkeypatch)
    L = g._l
    for s in range(B - 1):                 # slot B - 1 stays uninitialised
        g.init_map(0.0, 0.0, 0.0, slot=s)
    rb = g.snapshot_bytes
    buf = torch.zeros((B + 2) * rb + 64, dtype=torch.uint8, device="cuda")
    at = buf.data_ptr()
    ints = torch.zeros(2 * B + 2, dtype=torch.int32, device="cuda")
    ip = ints.data_ptr()
    ground = g.layer_device_ptr("ground", slot=2)
    g.synchronize()
    before = g.kernel_launches

    def save(slots=(0, 3, 5), dst=at, mask=None, h=g._h, null_slots=False, count=None):
        sl = np.ascontiguousarray(slots, np.int32)
        return L.gg_save_maps_to_device(h, len(sl) if count is None else count, None if null_slots else capi._ptr(sl), dst, mask, None)

    def restore(slots=(0, 3, 5), pool=at, n_pool=2, index=None, status=None, h=g._h, r=True, null_slots=False, count=None):
        sl = np.ascontiguousarray(slots, np.int32)
        rr = capi.MapRestore(pool, n_pool, index, status)
        return L.gg_restore_maps_from_device(h, len(sl) if count is None else count, None if null_slots else capi._ptr(sl),
                                             C.byref(rr) if r else None, None)

    cases = {
        "save: null handle": (lambda: save(h=None), ARG),
        "save: null slots": (lambda: save(null_slots=True), ARG),
        "save: null dst": (lambda: save(dst=None), ARG),
        "save: count > n_slots": (lambda: save(slots=list(range(B + 1))), ARG),
        "save: slot out of range": (lambda: save(slots=(0, B)), ARG),
        "save: repeated slot": (lambda: save(slots=(3, 3)), ARG),
        "save: dst not 16-byte aligned": (lambda: save(dst=at + 8), ARG),
        "save: mask not 4-byte aligned": (lambda: save(mask=ip + 2), ARG),
        "save: dst overlapping the layers": (lambda: save(dst=ground), ARG),
        "save: dst overlapping the mask": (lambda: save(mask=at + 64), ARG),
        "save: map not initialised": (lambda: save(slots=(0, B - 1)), STATE),
        "restore: null handle": (lambda: restore(h=None), ARG),
        "restore: null slots": (lambda: restore(null_slots=True), ARG),
        "restore: null r": (lambda: restore(r=False), ARG),
        "restore: null pool": (lambda: restore(pool=None), ARG),
        "restore: negative n_pool": (lambda: restore(n_pool=-1), ARG),
        "restore: count > n_slots": (lambda: restore(slots=list(range(B + 1))), ARG),
        "restore: slot out of range": (lambda: restore(slots=(0, -1)), ARG),
        "restore: repeated slot": (lambda: restore(slots=(5, 5)), ARG),
        "restore: pool not 16-byte aligned": (lambda: restore(pool=at + 4), ARG),
        "restore: index not 4-byte aligned": (lambda: restore(index=ip + 1), ARG),
        "restore: status not 4-byte aligned": (lambda: restore(status=ip + 2), ARG),
        "restore: pool overlapping the layers": (lambda: restore(pool=ground), ARG),
        "restore: status overlapping the pool": (lambda: restore(status=at + rb), ARG),
        "restore: status overlapping the index": (lambda: restore(index=ip, status=ip + 4), ARG),
        "restore: status overlapping the layers": (lambda: restore(status=ground), ARG),
        "restore: map not initialised": (lambda: restore(slots=(0, B - 1)), STATE),
    }
    for name, (fn, want) in cases.items():
        assert fn() == want, name
        assert g.kernel_launches == before, name
    assert save(count=0) == 0 and save(count=0, null_slots=True, dst=None) == 0
    assert restore(count=0) == 0 and restore(count=0, r=False, null_slots=True) == 0
    assert g.kernel_launches == before, "count 0"
    # a plan whose save stage is rejected (a misaligned dst) leaves no plan and no bound slot
    p = C.c_void_p()
    snaps = capi.StepSnapshots()
    snaps.save = at + 8
    scans = np.zeros(1, capi.SCAN_DESC_DTYPE)
    clouds = np.array([at], np.uint64)
    d = capi.StepDesc()
    d.count, d.scans, d.dev_points = 1, scans.ctypes.data, clouds.ctypes.data
    rc = L.gg_step_plan_create_with_snapshots(g._h, C.byref(d), None, None, None, C.byref(snaps), None, C.byref(p))
    assert rc == ARG and not p.value
    assert g.kernel_launches == before
    assert save(slots=(0,)) == 0, "slot 0 is not bound"
    g.synchronize()
    before = g.kernel_launches
    # valid calls launch one kernel per stream group with slots in the call
    assert save() == 0
    assert g.kernel_launches == before + len({s * GROUPS // B for s in (0, 3, 5)})
    g.synchronize()

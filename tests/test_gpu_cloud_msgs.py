"""Sensor-frame clouds from caller GPU memory (gg_run_cloud_msgs_to_device): PointCloud2 payloads in CUDA memory are
unpacked and transformed to the map frame on the device, then run like gg_run_scans_to_device, ordered on the caller's
stream.  Every check is bit-exact against a twin handle fed the same payload bytes from host memory through
gg_upload_cloud_msg + gg_run_scans + gg_download_labels + gg_get_output (and, for one slot per step, against the oracle
on oracle.nextrows.unpack_transform of the payload)."""
import math

import numpy as np
import pytest

from groundgrid_b200 import capi
from oracle import Oracle, nextrows
from test_gpu_device_outputs import DEAD, LIVE, SELECTS, advance, assert_layers_equal, assert_state_equal, check_outputs, make_pair, \
    make_steps, records, selected, to_device, torch_mod

pytestmark = pytest.mark.gpu

# (point_step, field offsets of x, y, z, intensity, ring): 32-byte PointXYZIR, the KITTI player's 18 bytes, 22 bytes
# without intensity, float32 [n, 4] without ring
LAYOUTS = [(32, (0, 4, 8, 16, 20)), (18, (0, 4, 8, 12, 16)), (22, (4, 8, 12, -1, 20)), (16, (0, 4, 8, 12, -1))]


def map_from_sensor(ego, yaw, pitch=0.03, height=1.7):
    """Row-major 3x4 of lookupTransform("map", sensor frame) for a sensor at (ego, height) with yaw and pitch."""
    cy, sy, cp, sp = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch)
    R = np.array([[cy, -sy, 0.0], [sy, cy, 0.0], [0.0, 0.0, 1.0]]) @ np.array([[cp, 0.0, sp], [0.0, 1.0, 0.0], [-sp, 0.0, cp]])
    return np.concatenate([R, np.array([[ego[0]], [ego[1]], [height]])], axis=1)


def payload(pts, step, offsets, T, rng):
    """PointCloud2 bytes uint8 [n, step] of map-frame points: in the sensor frame of T (inverse transform, float32) when T
    is given.  Bytes no field covers are random: the unpack must ignore them."""
    n = len(pts)
    fields = {name: np.ascontiguousarray(pts[name]) for name in ("x", "y", "z", "intensity", "ring")}
    if T is not None:
        p = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(np.float64) - T[:, 3]
        q = (p @ T[:, :3]).astype(np.float32)          # R^T (p - t)
        fields["x"], fields["y"], fields["z"] = (np.ascontiguousarray(q[:, c]) for c in range(3))
    raw = rng.integers(0, 256, (n, step), dtype=np.uint8)
    for name, off, width in zip(("x", "y", "z", "intensity", "ring"), offsets, (4, 4, 4, 4, 2)):
        if off >= 0:
            raw[:, off:off + width] = fields[name].view(np.uint8).reshape(n, width)
    return raw


def make_msgs(row, k, rng):
    """[(raw, step, offsets, T)] per scan: layouts and frames mixed within the batch and across steps."""
    msgs = []
    for b, r in enumerate(row):
        step, offsets = LAYOUTS[(b + k) % len(LAYOUTS)]
        T = map_from_sensor(r[2], 0.3 * b + 0.1 * k) if b % 3 != k % 3 else None
        msgs.append((payload(r[0], step, offsets, T, rng), step, offsets, T))
    return msgs


def cuda_bytes(raw):
    torch = torch_mod()
    return torch.from_numpy(np.ascontiguousarray(raw).reshape(-1).copy()).cuda()


def twin_run_msgs(twin, slots, row, msgs, base_z):
    """Labels, output index and output cloud of every scan through gg_upload_cloud_msg (host payload) + gg_run_scans."""
    keep = [twin.upload_cloud_msg(m[0], len(m[0]), m[1], m[2], m[3], slot=int(s)) for s, m in zip(slots, msgs)]
    twin.run_scans(twin.make_descs(list(slots), [len(m[0]) for m in msgs], [r[1] for r in row], [base_z] * len(row)))
    labels = [twin.download_labels(len(m[0]), slot=int(s)) for s, m in zip(slots, msgs)]
    twin.synchronize()
    del keep
    outs = [twin.get_output(slot=int(s), want_cloud=True) for s in slots]
    return labels, [o[0] for o in outs], [o[1] for o in outs]


def run_msgs(g, slots, row, msgs, base_z, **kw):
    return g.run_cloud_msgs_to_device([cuda_bytes(m[0]) for m in msgs], [m[1] for m in msgs], [m[2] for m in msgs],
                                      [m[3] for m in msgs], slots, [r[1] for r in row], base_z, **kw)


@pytest.mark.parametrize("dim,res,B,full_layers", [
    (99.0, 0.33, 4, True),       # N = 300: one slot per stream group
    (99.0, 0.33, 10, False),     # ten slots over eight stream groups
    (33.33, 0.33, 10, True),     # N = 101
    (33.33, 0.33, 4, False),
])
def test_parity_with_the_twin_over_a_rolling_stream(dim, res, B, full_layers):
    g, twin = make_pair(dim, res, B, full_layers)
    o = Oracle(dim, res)                                 # slot 0 runs the default configuration
    slots = np.arange(B, dtype=np.int32)[::-1].copy()   # batch order differs from slot order; slot 0 is last
    names = LIVE + (DEAD if full_layers else ())
    rng = np.random.default_rng(6100 + B)
    for k, row in enumerate(make_steps(B, 4, seed=6100 + B)):
        advance((g, twin), k, row, slots)
        if k == 0:
            o.init_map(row[-1][2][0], row[-1][2][1], 0.0)
        else:
            o.update(row[-1][2][0], row[-1][2][1], row[-1][3])
        msgs = make_msgs(row, k, rng)
        assert any(m[3] is None for m in msgs) and any(m[3] is not None for m in msgs)
        select = (SELECTS + (None,))[k % 4]             # the last step asks for labels only
        base_z = 0.02 * k
        out = run_msgs(g, slots, row, msgs, base_z, labels=True, select=select, index=select is not None)
        want_labels, want_index, want_cloud = twin_run_msgs(twin, slots, row, msgs, base_z)
        ctx = f"step {k} select {select}"
        if select is None:
            torch_mod().cuda.synchronize()
            assert out.cloud is None and out.index is None and out.counts is None
            for b in range(B):
                assert np.array_equal(out.labels[b].cpu().numpy(), want_labels[b]), f"{ctx} scan {b}: labels"
        else:
            check_outputs(out, select, want_labels, want_index, want_cloud, ctx)
        raw, step, offsets, T = msgs[-1]
        ol, oi, _ = o.filter_cloud(nextrows.unpack_transform(raw, len(raw), step, offsets, T), row[-1][1], base_z, threads=1)
        assert np.array_equal(out.labels[-1].cpu().numpy(), ol) and np.array_equal(want_index[-1], oi), f"{ctx}: oracle"
        assert_state_equal(g, twin, slots, [(m[0],) for m in msgs], names, ctx)
    g.close()
    twin.close()


def test_same_outputs_as_run_scans_to_device_on_host_unpacked_records():
    dim, res, B = 99.0, 0.33, 6
    g, h2 = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(6200)
    for k, row in enumerate(make_steps(B, 3, seed=6200)):
        advance((g, h2), k, row, slots)
        msgs = make_msgs(row, k, rng)
        recs = [to_device(nextrows.unpack_transform(m[0], len(m[0]), m[1], m[2], m[3])) for m in msgs]
        a = run_msgs(g, slots, row, msgs, 0.0, labels=True, select="all", index=True)
        b = h2.run_scans_to_device(recs, slots, [r[1] for r in row], 0.0, labels=True, select="all", index=True)
        torch_mod().cuda.synchronize()
        assert np.array_equal(a.counts.cpu().numpy(), b.counts.cpu().numpy()), f"step {k}: counts"
        (ac, ai), (bc, bi) = a.trimmed(), b.trimmed()
        for s in range(B):
            assert np.array_equal(a.labels[s].cpu().numpy(), b.labels[s].cpu().numpy()), f"step {k} scan {s}: labels"
            assert np.array_equal(ai[s].cpu().numpy(), bi[s].cpu().numpy()), f"step {k} scan {s}: index"
            assert records(ac[s]).tobytes() == records(bc[s]).tobytes(), f"step {k} scan {s}: cloud"
        assert_layers_equal(g, h2, slots, LIVE, f"step {k}")
    g.close()
    h2.close()


def test_edge_cases_empty_full_and_outputs_over_the_payload():
    """An empty cloud with data == NULL, a cloud of exactly max_points, labels written over the scan's own 18-byte
    payload and the output cloud written over the scan's own 32-byte payload."""
    torch = torch_mod()
    dim, res = 99.0, 0.33
    steps = make_steps(4, 1, seed=6300)[0]
    cap = max(len(r[0]) for r in steps)
    full = next(r for r in steps if len(r[0]) == cap)
    row = [(steps[0][0][:0], steps[0][1], steps[0][2], None), full, steps[2], steps[3]]
    B = len(row)
    g, twin = make_pair(dim, res, B, max_points=cap)
    slots = np.arange(B, dtype=np.int32)
    advance((g, twin), 0, row, slots)
    rng = np.random.default_rng(6300)
    msgs = [(payload(r[0], step, offsets, T, rng), step, offsets, T)
            for r, (step, offsets), T in zip(row, (LAYOUTS[0], LAYOUTS[0], LAYOUTS[1], LAYOUTS[0]),
                                             (None, map_from_sensor(full[2], 0.4), None, map_from_sensor(steps[3][2], -0.2)))]
    n = [len(m[0]) for m in msgs]
    assert n[0] == 0 and n[1] == cap
    data = [None] + [cuda_bytes(m[0]) for m in msgs[1:]]
    lab = [torch.full((m + 16,), 0xAB, dtype=torch.uint8, device="cuda") for m in n]
    idx = [torch.full((m + 16,), -7, dtype=torch.int32, device="cuda") for m in n]
    cld = [torch.full((m + 1, 8), -3.0, dtype=torch.float32, device="cuda") for m in n]
    counts = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    ptrs = np.array([[a.data_ptr(), b.data_ptr(), c.data_ptr()] for a, b, c in zip(lab, idx, cld)], np.uint64)
    ptrs[2, 0] = data[2].data_ptr()                     # labels of scan 2 over its own payload
    ptrs[3, 2] = data[3].data_ptr()                     # output cloud of scan 3 over its own payload
    descs = g.make_descs(list(slots), n, [r[1] for r in row], [0.0] * B)
    torch.cuda.synchronize()
    g.run_cloud_msgs_to_device_ptrs(descs, [0] + [d.data_ptr() for d in data[1:]], [m[1] for m in msgs], [m[2] for m in msgs],
                                    [m[3] for m in msgs], ptrs, 3, counts.data_ptr(), None)
    want_labels, want_index, want_cloud = twin_run_msgs(twin, slots, row, msgs, 0.0)
    torch.cuda.synchronize()
    got_counts = counts.cpu().numpy()
    for b in range(B):
        wi, wc = selected(want_labels[b], want_index[b], want_cloud[b], "all")
        c = int(got_counts[b])
        assert c == len(wi), f"scan {b}: count"
        L = data[2].cpu().numpy()[:n[2]] if b == 2 else lab[b].cpu().numpy()
        assert np.array_equal(L[:n[b]], want_labels[b]), f"scan {b}: labels"
        assert np.array_equal(idx[b][:c].cpu().numpy().view(np.uint32), wi) and (idx[b][c:].cpu().numpy() == -7).all(), f"scan {b}: index"
        Cl = data[3].cpu().numpy()[:32 * c].tobytes() if b == 3 else cld[b][:c].cpu().numpy().tobytes()
        assert Cl == wc.tobytes(), f"scan {b}: cloud"
    assert got_counts[0] == 0 and (lab[0].cpu().numpy() == 0xAB).all() and (cld[0].cpu().numpy() == -3.0).all()
    assert_state_equal(g, twin, slots, [(m[0],) for m in msgs], LIVE, "edge cases")
    g.close()
    twin.close()


@pytest.mark.parametrize("which", ["current", "side"])
def test_stream_order_without_host_waits(which):
    """(a) payloads produced on the stream right before the call are waited for on the device, (b) work enqueued after
    the call sees the outputs, (c) payloads freed right after the call and their memory refilled on the stream do not race
    with the unpack, and gg_get_output still works afterwards."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 4
    g, twin = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    steps = make_steps(B, 2, seed=6400)
    rng = np.random.default_rng(6400)
    stream = torch.cuda.current_stream() if which == "current" else torch.cuda.Stream()
    if which == "current":
        assert stream.cuda_stream == 0     # NULL is the legacy default stream, not "unordered"
    row = steps[0]                         # warm-up step: module loads, allocator pools
    advance((g, twin), 0, row, slots)
    msgs = make_msgs(row, 0, rng)
    run_msgs(g, slots, row, msgs, 0.0, select="all", stream=stream)
    twin_run_msgs(twin, slots, row, msgs, 0.0)
    torch.cuda.synchronize()
    row = steps[1]
    advance((g, twin), 1, row, slots)
    msgs = make_msgs(row, 1, rng)
    src = [cuda_bytes(m[0]) for m in msgs]
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        payloads = [torch.zeros_like(s) for s in src]
        torch.cuda._sleep(400_000_000)               # ~200 ms of device time ahead of the writes below
        for t, s in zip(payloads, src):
            t.copy_(s)
        before = torch.cuda.Event()
        before.record(stream)
        out = g.run_cloud_msgs_to_device(payloads, [m[1] for m in msgs], [m[2] for m in msgs], [m[3] for m in msgs], slots,
                                         [r[1] for r in row], 0.0, labels=True, select="all", index=True, stream=stream)
        assert not before.query(), "the call waited on the host for the stream"
        clones = ([t.clone() for t in out.labels], [t.clone() for t in out.cloud], [t.clone() for t in out.index], out.counts.clone())
        sizes = [t.numel() for t in payloads]
        del payloads
        refill = [torch.full((m,), 0xFF, dtype=torch.uint8, device="cuda") for m in sizes]
    pending = not before.query()
    want_labels, want_index, want_cloud = twin_run_msgs(twin, slots, row, msgs, 0.0)
    torch.cuda.synchronize()
    assert pending, "the sleep did not cover the call"
    check_outputs(out, "all", want_labels, want_index, want_cloud, f"{which}: outputs")
    labels_c, cloud_c, index_c, counts_c = clones
    cnt = counts_c.cpu().numpy()
    for k in range(B):
        assert np.array_equal(labels_c[k].cpu().numpy(), want_labels[k]), f"{which} scan {k}: cloned labels"
        assert cnt[k] == len(want_index[k]), f"{which} scan {k}: cloned count"
        assert np.array_equal(index_c[k][:cnt[k]].cpu().numpy().view(np.uint32), want_index[k]), f"{which} scan {k}: cloned index"
        assert records(cloud_c[k][:cnt[k]]).tobytes() == np.ascontiguousarray(want_cloud[k]).tobytes(), f"{which} scan {k}: cloned cloud"
    assert_state_equal(g, twin, slots, [(m[0],) for m in msgs], LIVE, which)   # gg_get_output with the payloads gone
    del refill
    g.close()
    twin.close()


def test_rejected_calls_enqueue_nothing_and_leave_the_handle_usable():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 4
    cap = 65536
    g, twin = make_pair(dim, res, B + 1, max_points=cap)       # slot B is never initialised
    slots = np.arange(B, dtype=np.int32)
    row = make_steps(B, 1, seed=6500)[0]
    advance((g, twin), 0, row, slots)
    msgs = make_msgs(row, 0, np.random.default_rng(6500))
    data = [cuda_bytes(m[0]) for m in msgs]
    n = [len(m[0]) for m in msgs]
    origins = [r[1] for r in row]
    big = torch.zeros(32 * (cap + 1), dtype=torch.uint8, device="cuda")
    lab = [torch.zeros(m, dtype=torch.uint8, device="cuda") for m in n]
    idx = [torch.zeros(m + 4, dtype=torch.int32, device="cuda") for m in n]
    cld = [torch.zeros((m + 1, 8), dtype=torch.float32, device="cuda") for m in n]
    counts = torch.zeros(B + 1, dtype=torch.int32, device="cuda")
    good_ptrs = np.array([[a.data_ptr(), b.data_ptr(), c.data_ptr()] for a, b, c in zip(lab, idx, cld)], np.uint64)
    good_in = [t.data_ptr() for t in data]
    steps_ = [m[1] for m in msgs]
    offs_ = [m[2] for m in msgs]
    Ts = [m[3] for m in msgs]

    def call(slots_=slots, n_=n, ins=good_in, st=steps_, of=offs_, ptrs=good_ptrs, select=3, cnt=counts.data_ptr()):
        descs = g.make_descs(list(slots_), list(n_), origins, [0.0] * len(slots_))
        g.run_cloud_msgs_to_device_ptrs(descs, ins, st, of, Ts, ptrs, select, cnt, None)

    def with_ptr(col, scan, value):
        p = good_ptrs.copy()
        p[scan, col] = value
        return p

    def replaced(seq, k, value):
        s = list(seq)
        s[k] = value
        return s

    def null_msgs():
        descs = g.make_descs(list(slots), n, origins, [0.0] * B)
        capi._check(g._l.gg_run_cloud_msgs_to_device(g._h, B, descs, None, capi._ptr(good_ptrs), 3, counts.data_ptr(), None))

    cases = {
        "repeated slot": lambda: call(slots_=[0, 1, 1, 3]),
        "capacity exceeded": lambda: call(n_=replaced(n, 1, cap + 1), ins=replaced(good_in, 1, big.data_ptr()), st=replaced(steps_, 1, 32),
                                          of=replaced(offs_, 1, LAYOUTS[0][1])),
        "null msgs": null_msgs,
        "null data": lambda: call(ins=replaced(good_in, 2, 0)),
        "point_step below 12": lambda: call(st=replaced(steps_, 0, 11), of=replaced(offs_, 0, (0, 4, 7, -1, -1))),
        "x absent": lambda: call(of=replaced(offs_, 1, (-1, 4, 8, 12, -1))),
        "z absent": lambda: call(of=replaced(offs_, 3, (0, 4, -1, 12, -1))),
        "field outside point_step": lambda: call(st=replaced(steps_, 2, 18), of=replaced(offs_, 2, (0, 4, 8, 12, 17))),
        "index with select 0": lambda: call(ptrs=np.array([[0, p[1], 0] for p in good_ptrs], np.uint64), select=0),
        "cloud with select 0": lambda: call(ptrs=np.array([[0, 0, p[2]] for p in good_ptrs], np.uint64), select=0),
        "unknown select bits": lambda: call(select=7),
        "no dev_counts": lambda: call(cnt=None),
        "misaligned dev_counts": lambda: call(cnt=counts.data_ptr() + 2),
        "misaligned index": lambda: call(ptrs=with_ptr(1, 2, int(good_ptrs[2, 1]) + 2)),
        "misaligned cloud": lambda: call(ptrs=with_ptr(2, 1, int(good_ptrs[1, 2]) + 8)),
    }
    torch.cuda.synchronize()
    for name, fn in cases.items():
        l0 = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            fn()
        assert e.value.code == -1, f"{name}: code {e.value.code}"
        assert g.kernel_launches == l0, f"{name}: something was launched"
    l0 = g.kernel_launches
    with pytest.raises(capi.GroundGridError) as e:
        call(slots_=[0, 1, 2, B])
    assert e.value.code == -3 and g.kernel_launches == l0, "map not initialised"
    g.run_cloud_msgs_to_device_ptrs(g.make_descs([], [], [], []), [], 32, LAYOUTS[0][1], None, None, 0, None, None)
    assert g.kernel_launches == l0, "count 0 launched something"
    torch.cuda.synchronize()
    # nothing was enqueued: the handle still holds the initial maps, and a correct call matches the twin
    call()
    want_labels, want_index, want_cloud = twin_run_msgs(twin, slots, row, msgs, 0.0)
    torch.cuda.synchronize()
    got_counts = counts.cpu().numpy()
    for k in range(B):
        assert np.array_equal(lab[k].cpu().numpy(), want_labels[k])
        c = int(got_counts[k])
        assert c == len(want_index[k])
        assert np.array_equal(idx[k][:c].cpu().numpy().view(np.uint32), want_index[k])
        assert records(cld[k][:c]).tobytes() == np.ascontiguousarray(want_cloud[k]).tobytes()
    assert_state_equal(g, twin, slots, [(m[0],) for m in msgs], LIVE, "after the rejected calls")
    g.close()
    twin.close()

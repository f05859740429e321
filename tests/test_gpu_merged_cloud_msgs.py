"""Multi-sensor scans from caller GPU memory (gg_run_merged_cloud_msgs_to_device): several PointCloud2 payloads per scan,
each in its own frame, unpacked and transformed into the slot's buffer one after the other, then run like
gg_run_cloud_msgs_to_device.  Every check is bit-exact against a twin handle fed the same payload bytes from host memory
through gg_upload_cloud_msgs + gg_run_scans (and, for one slot per step, against the oracle on the concatenation of
oracle.nextrows.unpack_transform of each part)."""
import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from oracle import Oracle, nextrows
from test_gpu_cloud_msgs import LAYOUTS, cuda_bytes, make_msgs, map_from_sensor, payload, run_msgs
from test_gpu_device_outputs import DEAD, LIVE, SELECTS, advance, assert_layers_equal, assert_state_equal, check_outputs, make_pair, \
    make_steps, records, selected, torch_mod

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3


def make_scans(row, k, rng, max_parts=4):
    """[scan][part] -> (raw, step, offsets, T): each scan cut into 1..max_parts parts at seeded points, the second of
    three or more parts empty; layouts and frames mixed within a scan."""
    scans = []
    for b, r in enumerate(row):
        pts = r[0]
        m = 1 + (b + k) % max_parts
        cuts = np.sort(rng.integers(0, len(pts) + 1, m - 1))
        if m >= 3:
            cuts[1] = cuts[0]
        bounds = np.r_[0, cuts, len(pts)]
        parts = []
        for p in range(m):
            step, offsets = LAYOUTS[(b + p + k) % len(LAYOUTS)]
            T = map_from_sensor(r[2], 0.3 * b + 0.7 * p + 0.1 * k) if (b + 2 * p + k) % 3 else None
            parts.append((payload(pts[bounds[p]:bounds[p + 1]], step, offsets, T, rng), step, offsets, T))
        scans.append(parts)
    return scans


def n_of(parts):
    return sum(len(p[0]) for p in parts)


def concat(parts):
    """The map-frame records of a merged scan as the reference's upstream merge builds them."""
    recs = [nextrows.unpack_transform(p[0], len(p[0]), p[1], p[2], p[3]) for p in parts]
    out = np.zeros(sum(len(r) for r in recs), synth.POINT_DTYPE)
    at = 0
    for r in recs:
        for f in ("x", "y", "z", "intensity", "ring"):
            out[f][at:at + len(r)] = r[f]
        at += len(r)
    return out


def nested(scans, i):
    return [[p[i] for p in parts] for parts in scans]


def run_merged(g, slots, origins, scans, base_z, **kw):
    return g.run_merged_cloud_msgs_to_device([[cuda_bytes(p[0]) for p in parts] for parts in scans], nested(scans, 1), nested(scans, 2),
                                             nested(scans, 3), slots, origins, base_z, **kw)


def twin_run_merged(twin, slots, origins, scans, base_z):
    """Labels, output index and output cloud of every scan through gg_upload_cloud_msgs (host payloads) + gg_run_scans."""
    keep = [twin.upload_cloud_msgs(parts, slot=int(s)) for s, parts in zip(slots, scans)]
    n = [n_of(parts) for parts in scans]
    twin.run_scans(twin.make_descs(list(slots), n, origins, [base_z] * len(scans)))
    labels = [twin.download_labels(m, slot=int(s)) for s, m in zip(slots, n)]
    twin.synchronize()
    del keep
    outs = [twin.get_output(slot=int(s), want_cloud=True) for s in slots]
    return labels, [o[0] for o in outs], [o[1] for o in outs]


def sized(scans):
    """Rows for assert_state_equal: only their point counts are read."""
    return [(np.zeros(n_of(parts)),) for parts in scans]


@pytest.mark.parametrize("dim,res,B,full_layers", [
    (99.0, 0.33, 4, True),       # N = 300: one slot per stream group
    (99.0, 0.33, 10, False),     # ten slots over eight stream groups
    (33.33, 0.33, 10, True),     # N = 101
])
def test_parity_with_the_twin_over_a_rolling_stream(dim, res, B, full_layers):
    g, twin = make_pair(dim, res, B, full_layers)
    o = Oracle(dim, res)                                 # slot 0 runs the default configuration
    slots = np.arange(B, dtype=np.int32)[::-1].copy()   # batch order differs from slot order; slot 0 is last
    names = LIVE + (DEAD if full_layers else ())
    rng = np.random.default_rng(7100 + B)
    for k, row in enumerate(make_steps(B, 4, seed=7100 + B)):
        advance((g, twin), k, row, slots)
        if k == 0:
            o.init_map(row[-1][2][0], row[-1][2][1], 0.0)
        else:
            o.update(row[-1][2][0], row[-1][2][1], row[-1][3])
        scans = make_scans(row, k, rng)
        parts = [p for s in scans for p in s]
        assert any(p[3] is None for p in parts) and any(p[3] is not None for p in parts) and any(len(p[0]) == 0 for p in parts)
        assert {len(s) for s in scans} == {1, 2, 3, 4}
        select = (SELECTS + (None,))[k % 4]             # the last step asks for labels only
        base_z = 0.02 * k
        origins = [r[1] for r in row]
        out = run_merged(g, slots, origins, scans, base_z, labels=True, select=select, index=select is not None)
        want_labels, want_index, want_cloud = twin_run_merged(twin, slots, origins, scans, base_z)
        ctx = f"step {k} select {select}"
        if select is None:
            torch_mod().cuda.synchronize()
            assert out.cloud is None and out.index is None and out.counts is None
            for b in range(B):
                assert np.array_equal(out.labels[b].cpu().numpy(), want_labels[b]), f"{ctx} scan {b}: labels"
        else:
            check_outputs(out, select, want_labels, want_index, want_cloud, ctx)
        ol, oi, _ = o.filter_cloud(concat(scans[-1]), row[-1][1], base_z, threads=1)
        assert np.array_equal(out.labels[-1].cpu().numpy(), ol) and np.array_equal(want_index[-1], oi), f"{ctx}: oracle"
        assert_state_equal(g, twin, slots, sized(scans), names, ctx)
    g.close()
    twin.close()


def test_one_part_per_scan_is_run_cloud_msgs_to_device():
    dim, res, B = 99.0, 0.33, 6
    g, h2 = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(7200)
    for k, row in enumerate(make_steps(B, 3, seed=7200)):
        advance((g, h2), k, row, slots)
        msgs = make_msgs(row, k, rng)
        a = run_merged(g, slots, [r[1] for r in row], [[m] for m in msgs], 0.01 * k, labels=True, select="all", index=True)
        b = run_msgs(h2, slots, row, msgs, 0.01 * k, labels=True, select="all", index=True)
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


def test_part_order_is_the_concatenation_order():
    dim, res = 99.0, 0.33
    g = capi.GroundGridB200(dim, res, n_slots=1, max_points=65536)
    row = make_steps(1, 1, seed=7300)[0]
    pts, org, ego, _ = row[0]
    rng = np.random.default_rng(7300)
    cut = len(pts) // 3
    a = (payload(pts[:cut], 18, LAYOUTS[1][1], map_from_sensor(ego, 0.5), rng), 18, LAYOUTS[1][1], map_from_sensor(ego, 0.5))
    b = (payload(pts[cut:], 32, LAYOUTS[0][1], map_from_sensor(ego, -1.1), rng), 32, LAYOUTS[0][1], map_from_sensor(ego, -1.1))
    labels = {}
    for order in ((a, b), (b, a)):
        g.init_map(ego[0], ego[1], 0.0)
        o = Oracle(dim, res)
        o.init_map(ego[0], ego[1], 0.0)
        out = run_merged(g, [0], [org], [list(order)], 0.0, labels=True, select="all", index=True)
        _, got_index = out.trimmed()
        want_labels, want_index, _ = o.filter_cloud(concat(order), org, 0.0, threads=1)
        key = "ab" if order[0] is a else "ba"
        labels[key] = out.labels[0].cpu().numpy()
        assert np.array_equal(labels[key], want_labels), f"{key}: labels"
        assert np.array_equal(got_index[0].cpu().numpy().view(np.uint32), want_index), f"{key}: index"
        assert np.array_equal(g.layer("ground"), o.layer("ground")), f"{key}: ground"
    assert not np.array_equal(labels["ab"], labels["ba"])
    g.close()


def test_eval_tallies_after_the_payloads_are_freed():
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 4
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(7400)
    stream = torch.cuda.Stream()
    tallies = torch.zeros((B, 1024, 2), dtype=torch.int64, device="cuda")
    want = np.zeros((B, 1024, 2), np.uint64)
    for k, row in enumerate(make_steps(B, 2, seed=7400)):
        advance((g,), k, row, slots)
        for r in row:                                 # ids spread over the tally
            r[0]["ring"] = rng.integers(0, 1100, len(r[0])).astype(np.uint16)
        scans = make_scans(row, k, rng)
        with torch.cuda.stream(stream):
            payloads = [[cuda_bytes(p[0]) for p in parts] for parts in scans]
            out = g.run_merged_cloud_msgs_to_device(payloads, nested(scans, 1), nested(scans, 2), nested(scans, 3), slots,
                                                    [r[1] for r in row], 0.0, labels=True, select=None)
            del payloads
            junk = [torch.full((n_of(parts) * 32,), 0xFF, dtype=torch.uint8, device="cuda") for parts in scans]
            g.eval_counts_to_device(slots, out=tallies, stream=stream)
        torch.cuda.synchronize()
        del junk
        for b, parts in enumerate(scans):
            want[b] += nextrows.eval_counts(out.labels[b].cpu().numpy(), concat(parts)["ring"])
        assert np.array_equal(tallies.cpu().numpy().view(np.uint64), want), f"step {k}"
        assert want.sum() > 0
    g.close()


@pytest.mark.parametrize("which", ["current", "side"])
def test_stream_order_without_host_waits(which):
    """(a) parts produced on the stream right before the call are waited for on the device, (b) work enqueued after the
    call sees the outputs, (c) parts freed right after the call and their memory refilled on the stream do not race with
    the unpack, and gg_get_output still works afterwards."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 4
    g, twin = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    steps = make_steps(B, 2, seed=7500)
    rng = np.random.default_rng(7500)
    stream = torch.cuda.current_stream() if which == "current" else torch.cuda.Stream()
    row = steps[0]                         # warm-up step: module loads, allocator pools
    advance((g, twin), 0, row, slots)
    scans = make_scans(row, 0, rng)
    origins = [r[1] for r in row]
    run_merged(g, slots, origins, scans, 0.0, select="all", stream=stream)
    twin_run_merged(twin, slots, origins, scans, 0.0)
    torch.cuda.synchronize()
    row = steps[1]
    advance((g, twin), 1, row, slots)
    scans = make_scans(row, 1, rng)
    origins = [r[1] for r in row]
    src = [[cuda_bytes(p[0]) for p in parts] for parts in scans]
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        payloads = [[torch.zeros_like(s) for s in parts] for parts in src]
        torch.cuda._sleep(400_000_000)               # ~200 ms of device time ahead of the writes below
        for tp, sp in zip(payloads, src):
            for t, s in zip(tp, sp):
                t.copy_(s)
        before = torch.cuda.Event()
        before.record(stream)
        out = g.run_merged_cloud_msgs_to_device(payloads, nested(scans, 1), nested(scans, 2), nested(scans, 3), slots, origins, 0.0,
                                                labels=True, select="all", index=True, stream=stream)
        assert not before.query(), "the call waited on the host for the stream"
        clones = ([t.clone() for t in out.labels], [t.clone() for t in out.cloud], [t.clone() for t in out.index], out.counts.clone())
        sizes = [t.numel() for tp in payloads for t in tp]
        del payloads, tp
        refill = [torch.full((m,), 0xFF, dtype=torch.uint8, device="cuda") for m in sizes]
    pending = not before.query()
    want_labels, want_index, want_cloud = twin_run_merged(twin, slots, origins, scans, 0.0)
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
    assert_state_equal(g, twin, slots, sized(scans), LIVE, which)   # gg_get_output with the payloads gone
    del refill
    g.close()
    twin.close()


def test_outputs_over_the_scans_own_parts():
    """Each scan's parts sit back to back in one buffer; labels of scan 0 and the output cloud of scan 1 are written over
    it, and the other outputs go to their own buffers."""
    torch = torch_mod()
    dim, res, B = 99.0, 0.33, 3
    g, twin = make_pair(dim, res, B)
    slots = np.arange(B, dtype=np.int32)
    row = make_steps(B, 1, seed=7600)[0]
    advance((g, twin), 0, row, slots)
    rng = np.random.default_rng(7600)
    scans = make_scans(row, 2, rng)
    scans[1] = [(payload(p, 32, LAYOUTS[0][1], T, rng), 32, LAYOUTS[0][1], T)     # 32-byte parts: room for the cloud
                for p, T in ((row[1][0][:5000], map_from_sensor(row[1][2], 0.2)), (row[1][0][5000:], None))]
    origins = [r[1] for r in row]
    bufs = [cuda_bytes(np.concatenate([p[0].reshape(-1) for p in parts])) for parts in scans]
    ptrs = []
    for buf, parts in zip(bufs, scans):
        at, ps = 0, []
        for p in parts:
            ps.append(buf.data_ptr() + at)
            at += p[0].size
        ptrs.append(ps)
    n = [n_of(parts) for parts in scans]
    assert bufs[0].numel() >= n[0]
    lab = [torch.full((m,), 0xAB, dtype=torch.uint8, device="cuda") for m in n]
    idx = [torch.full((m,), -7, dtype=torch.int32, device="cuda") for m in n]
    cld = [torch.full((m, 8), -3.0, dtype=torch.float32, device="cuda") for m in n]
    counts = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    out_ptrs = np.array([[a.data_ptr(), b.data_ptr(), c.data_ptr()] for a, b, c in zip(lab, idx, cld)], np.uint64)
    out_ptrs[0, 0] = bufs[0].data_ptr()
    out_ptrs[1, 2] = bufs[1].data_ptr()
    n_parts, parts, keep = capi.cloud_parts([[p[0].size for p in s] for s in scans], ptrs, nested(scans, 1), nested(scans, 2), nested(scans, 3))
    torch.cuda.synchronize()
    g.run_merged_cloud_msgs_to_device_ptrs(g.make_descs(list(slots), n, origins, [0.0] * B), n_parts, parts, out_ptrs, 3, counts.data_ptr(), None)
    want_labels, want_index, want_cloud = twin_run_merged(twin, slots, origins, scans, 0.0)
    torch.cuda.synchronize()
    got_counts = counts.cpu().numpy()
    for b in range(B):
        wi, wc = selected(want_labels[b], want_index[b], want_cloud[b], "all")
        c = int(got_counts[b])
        assert c == len(wi), f"scan {b}: count"
        L = bufs[0].cpu().numpy()[:n[0]] if b == 0 else lab[b].cpu().numpy()
        assert np.array_equal(L, want_labels[b]), f"scan {b}: labels"
        assert np.array_equal(idx[b][:c].cpu().numpy().view(np.uint32), wi), f"scan {b}: index"
        Cl = bufs[1].cpu().numpy()[:32 * c].tobytes() if b == 1 else cld[b][:c].cpu().numpy().tobytes()
        assert Cl == wc.tobytes(), f"scan {b}: cloud"
    assert (lab[0].cpu().numpy() == 0xAB).all() and (cld[1].cpu().numpy() == -3.0).all()
    assert_state_equal(g, twin, slots, sized(scans), LIVE, "outputs over the parts")
    del keep
    g.close()
    twin.close()


def test_rejected_calls_enqueue_nothing_and_leave_the_handle_usable():
    torch = torch_mod()
    dim, res, B = 33.33, 0.33, 4
    cap = 65536
    g, twin = make_pair(dim, res, B + 1, max_points=cap)       # slot B is never initialised
    slots = np.arange(B, dtype=np.int32)
    row = make_steps(B, 1, seed=7700)[0]
    advance((g, twin), 0, row, slots)
    scans = make_scans(row, 1, np.random.default_rng(7700))      # 2, 3, 4 and 1 parts
    assert [len(s) for s in scans] == [2, 3, 4, 1]
    data = [[cuda_bytes(p[0]) for p in parts] for parts in scans]
    origins = [r[1] for r in row]
    n = [n_of(parts) for parts in scans]
    big = torch.zeros(32 * (cap + 1), dtype=torch.uint8, device="cuda")
    lab = [torch.zeros(m, dtype=torch.uint8, device="cuda") for m in n]
    idx = [torch.zeros(m + 4, dtype=torch.int32, device="cuda") for m in n]
    cld = [torch.zeros((m + 1, 8), dtype=torch.float32, device="cuda") for m in n]
    counts = torch.zeros(B + 1, dtype=torch.int32, device="cuda")
    good_ptrs = np.array([[a.data_ptr(), b.data_ptr(), c.data_ptr()] for a, b, c in zip(lab, idx, cld)], np.uint64)
    good_np, good_parts, keep = capi.cloud_parts([[p[0].size for p in s] for s in scans], [[t.data_ptr() for t in s] for s in data],
                                                 nested(scans, 1), nested(scans, 2), nested(scans, 3))

    def call(slots_=slots, n_=n, n_parts=good_np, parts=good_parts, ptrs=good_ptrs, select=3, cnt=counts.data_ptr()):
        descs = g.make_descs(list(slots_), list(n_), origins[:len(slots_)], [0.0] * len(slots_))
        g.run_merged_cloud_msgs_to_device_ptrs(descs, n_parts, parts, ptrs, select, cnt, None)

    def part(p, **fields):
        """good_parts with part p (flat index) changed."""
        q = good_parts.copy()
        for k, v in fields.items():
            q[k][p] = v
        return q

    def raw(n_parts_ptr, parts_ptr):
        descs = g.make_descs(list(slots), n, origins, [0.0] * B)
        capi._check(g._l.gg_run_merged_cloud_msgs_to_device(g._h, B, descs, n_parts_ptr, parts_ptr, capi._ptr(good_ptrs), 3, counts.data_ptr(),
                                                             None))

    # flat index of scan 2's part 1 (scan 0 has 2 parts, scan 1 has 3)
    s2p1 = 2 + 3 + 1
    big_parts = part(0, data=big.data_ptr(), point_step=32, field_offsets=LAYOUTS[0][1], n_points=cap + 1 - int(good_parts["n_points"][1]))
    cases = {
        "repeated slot": (lambda: call(slots_=[0, 1, 1, 3]), None),
        "capacity exceeded": (lambda: call(n_=[cap + 1] + n[1:], parts=big_parts), None),
        "null n_parts": (lambda: raw(None, capi._ptr(good_parts)), "null argument"),
        "null parts": (lambda: raw(capi._ptr(good_np), None), "null argument"),
        "negative n_parts": (lambda: call(n_parts=[2, 3, -1, 1]), "scan 2"),
        "too many parts": (lambda: call(n_parts=[2, 3, capi.MAX_CLOUD_PARTS + 1, 1], parts=np.concatenate([good_parts] * 3)), "scan 2"),
        "parts hold fewer points": (lambda: call(n_=n[:1] + [n[1] + 1] + n[2:]), "scan 1"),
        "parts hold more points": (lambda: call(n_=n[:3] + [n[3] - 1]), "scan 3"),
        "null data": (lambda: call(parts=part(s2p1 + 1, data=0)), "scan 2 part 2"),
        "point_step below 12": (lambda: call(parts=part(s2p1, point_step=11, field_offsets=(0, 4, 7, -1, -1))), "scan 2 part 1"),
        "x absent": (lambda: call(parts=part(1, field_offsets=(-1, 4, 8, 12, -1))), "scan 0 part 1"),
        "field outside point_step": (lambda: call(parts=part(2, point_step=18, field_offsets=(0, 4, 8, 12, 17))), "scan 1 part 0"),
        "index with select 0": (lambda: call(ptrs=np.array([[0, p[1], 0] for p in good_ptrs], np.uint64), select=0), None),
        "unknown select bits": (lambda: call(select=7), None),
        "no dev_counts": (lambda: call(cnt=None), None),
        "misaligned dev_counts": (lambda: call(cnt=counts.data_ptr() + 2), None),
        "misaligned cloud": (lambda: call(ptrs=np.where(np.arange(3) == 2, good_ptrs + 8, good_ptrs).astype(np.uint64)), None),
    }
    assert good_parts["n_points"][s2p1 + 1] > 0
    torch.cuda.synchronize()
    for name, (fn, text) in cases.items():
        l0 = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            fn()
        assert e.value.code == ARG, f"{name}: code {e.value.code}"
        assert text is None or text in str(e.value), f"{name}: {e.value}"
        assert g.kernel_launches == l0, f"{name}: something was launched"
    l0 = g.kernel_launches
    with pytest.raises(capi.GroundGridError) as e:
        call(slots_=[0, 1, 2, B])
    assert e.value.code == STATE and g.kernel_launches == l0, "map not initialised"
    # the host form rejects the same part rules, naming the part
    for fn, text in ((lambda: g.upload_cloud_msgs([scans[0][0]] * (capi.MAX_CLOUD_PARTS + 1), slot=0), None),
                     (lambda: g.upload_cloud_msgs([scans[0][0], (np.zeros(22, np.uint8), 11, (0, 4, 7, -1, -1), None)], slot=0), "part 1")):
        with pytest.raises(capi.GroundGridError) as e:
            fn()
        assert e.value.code == ARG and (text is None or text in str(e.value)) and g.kernel_launches == l0
    g.run_merged_cloud_msgs_to_device_ptrs(g.make_descs([], [], [], []), np.zeros(0, np.int32), np.zeros(0, capi.CLOUD_PART_DTYPE), None, 0,
                                           None, None)
    assert g.kernel_launches == l0, "count 0 launched something"
    torch.cuda.synchronize()
    # nothing was enqueued: the handle still holds the initial maps, and a correct call matches the twin
    call()
    want_labels, want_index, want_cloud = twin_run_merged(twin, slots, origins, scans, 0.0)
    torch.cuda.synchronize()
    got_counts = counts.cpu().numpy()
    for k in range(B):
        assert np.array_equal(lab[k].cpu().numpy(), want_labels[k])
        c = int(got_counts[k])
        assert c == len(want_index[k])
        assert np.array_equal(idx[k][:c].cpu().numpy().view(np.uint32), want_index[k])
        assert records(cld[k][:c]).tobytes() == np.ascontiguousarray(want_cloud[k]).tobytes()
    assert_state_equal(g, twin, slots, sized(scans), LIVE, "after the rejected calls")
    del keep
    g.close()
    twin.close()

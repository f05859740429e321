"""Per-part point counts from caller GPU memory (gg_set_part_counts_from_device + GG_SCAN_DEVICE_PART_COUNTS on
gg_run_merged_cloud_msgs_to_device): multi-sensor scans whose per-sensor counts only the device knows.  Every case runs
against a twin handle that makes the host-count merged call on the same device payloads, with parts of n_points = u_p,
and must be bit-identical to it: labels, index, cloud, dev_counts, every live layer, gg_get_output, gg_last_scan_points,
point-info codes and heights, and tallies (and, for slot 0 every step, the oracle on the concatenation of each part's
first u_p records).  Every payload's records past u_p are poison: in-map points high above the terrain with counted
rings, and NaN / huge coordinates, so a read past a part's count shows."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from oracle import Oracle, nextrows
from test_gpu_cloud_msgs import LAYOUTS, map_from_sensor, payload
from test_gpu_device_counts import INT32_MAX, INT32_MIN, assert_twin, poison
from test_gpu_device_outputs import LIVE, advance, make_pair, make_steps, torch_mod

pytestmark = pytest.mark.gpu

ARG, STATE = -1, -3
MAX_POINTS = 65536
P = capi.MAX_CLOUD_PARTS


def part_layout(L, kind):
    """(stored v, capacity c) of a part with L real records: u = v, u = c, u = c - 1, v = c + 1, -1, INT32_MAX,
    INT32_MIN, a part of capacity 0, u < c."""
    return [(L, L), (L, L + 9), (max(L - 1, 0), L), (L + 1, L), (-1, L), (INT32_MAX, L), (INT32_MIN, L), (5, 0), (L // 2, L + 37)][kind]


def used(v, c):
    return v if 0 <= v <= c else 0


def sentinel(pts, n, rng):
    """n poison records: in-map points above the terrain with rings the tallies count, every third one NaN, huge or
    with a ring past max_ring."""
    out = poison(pts, n, rng)
    out["x"][0::3] = np.nan
    out["z"][1::3] = 3.0e38
    out["ring"][2::3] = 60000
    return out


class Rig:
    """One step of merged scans: per scan its parts as (device payload, step, offsets, T, v, c, u, real records)."""

    def __init__(self, torch, row, k, rng, n_parts, stored=None, flagged=None, fill_to=None):
        self.scans, self.flagged = [], flagged if flagged is not None else [True] * len(row)
        for b, r in enumerate(row):
            pts, m = r[0], n_parts[b]
            cuts = np.sort(rng.integers(0, len(pts) + 1, m - 1))
            bounds = np.r_[0, cuts, len(pts)]
            parts = []
            for p in range(m):
                real = pts[bounds[p]:bounds[p + 1]]
                L = len(real)
                if not self.flagged[b]:
                    v, c = L, L
                elif stored is not None:          # counts stored by an earlier step: capacities at L keep u <= L
                    v, c = int(stored[b][p]), L
                else:
                    v, c = part_layout(L, (3 * b + 5 * p + k) % 9)
                u = used(v, c)
                step, offs = LAYOUTS[(b + p + k) % len(LAYOUTS)]
                T = map_from_sensor(r[2], 0.3 * b + 0.7 * p + 0.1 * k) if (b + 2 * p + k) % 3 else None
                parts.append([real, step, offs, T, v, c, u])
            if fill_to is not None and b == fill_to and self.flagged[b]:   # capacities summing to exactly max_points
                q = parts[-1]
                q[5] += MAX_POINTS - sum(x[5] for x in parts)
                q[6] = used(q[4], q[5])
                if q[6] > len(q[0]):                      # a count the grown capacity would admit past the real records
                    q[4], q[6] = -1, 0
            for q in parts:
                real, step, offs, T, v, c, u = q
                cloud = np.zeros(c, synth.POINT_DTYPE)
                cloud[:u] = real[:u]
                cloud[u:] = sentinel(pts, c - u, rng)
                raw = payload(cloud, step, offs, T, rng)
                q.insert(0, torch.from_numpy(np.ascontiguousarray(raw).reshape(-1).copy()).cuda())
            self.scans.append(parts)
        self.us = [sum(q[7] for q in s) for s in self.scans]
        self.caps = [sum(q[6] for q in s) for s in self.scans]

    def counts(self, torch):
        v = np.zeros((len(self.scans), P), np.int64)
        for b, s in enumerate(self.scans):
            for p, q in enumerate(s):
                v[b, p] = q[5]
        return torch.tensor(v, dtype=torch.int32, device="cuda")

    def call(self, h, slots, origins, base_z, select, device, stream=None):
        """device: the flagged call at capacity; else the twin's host-count call on the first u_p records."""
        torch = torch_mod()
        nested = lambda i: [[q[i] for q in s] for s in self.scans]   # noqa: E731
        if device:
            data = [[q[0] for q in s] for s in self.scans]
        else:
            data = [[q[0][:q[7] * q[2]] for q in s] for s in self.scans]
        n_parts, parts, keep = capi.cloud_parts([[t.numel() for t in s] for s in data], [[t.data_ptr() for t in s] for s in data],
                                                nested(2), nested(3), nested(4))
        n = self.caps if device else self.us
        descs = h._device_descs(slots, n, origins, base_z)
        if device:
            descs["flags"] |= np.where(self.flagged, capi.SCAN_DEVICE_PART_COUNTS, 0).astype(np.int32)
        st = torch.cuda.current_stream() if stream is None else stream
        sel = capi.SELECT[select]
        out, ptrs = h._device_outputs(torch, torch.device("cuda"), st, n, True, sel, sel != 0, [])
        h.run_merged_cloud_msgs_to_device_ptrs(descs, n_parts, parts, ptrs, sel, out.counts.data_ptr() if out.counts is not None else None,
                                               st.cuda_stream or None)
        del keep
        return out

    def concat(self, b):
        recs = [nextrows.unpack_transform(payload_bytes(q), q[7], q[2], q[3], q[4]) for q in self.scans[b] if q[7]]
        out = np.zeros(sum(len(r) for r in recs), synth.POINT_DTYPE)
        at = 0
        for r in recs:
            for f in ("x", "y", "z", "intensity", "ring"):
                out[f][at:at + len(r)] = r[f]
            at += len(r)
        return out


def payload_bytes(q):
    return q[0][:q[7] * q[2]].cpu().numpy()


def check(out_g, out_t, us, ctx):
    torch = torch_mod()
    torch.cuda.synchronize()
    if out_t.counts is not None:
        assert torch.equal(out_g.counts, out_t.counts), f"{ctx}: dev_counts"
        gc, gi = out_g.trimmed()
        tc, ti = out_t.trimmed()
        for k in range(len(us)):
            assert torch.equal(gc[k].view(torch.int32), tc[k].view(torch.int32)), f"{ctx} scan {k}: cloud"
            if gi is not None:
                assert torch.equal(gi[k], ti[k]), f"{ctx} scan {k}: index"
    for k, u in enumerate(us):
        assert torch.equal(out_g.labels[k][:u], out_t.labels[k]), f"{ctx} scan {k}: labels"


def set_poses(hs, slots, row, base_z):
    torch = torch_mod()
    xy = torch.tensor(np.array([r[2] for r in row], np.float64), device="cuda")
    T = torch.tensor(np.stack([r[3].reshape(12) for r in row]), dtype=torch.float64, device="cuda")
    org = torch.tensor(np.array([r[1] for r in row], np.float32), device="cuda")
    bz = torch.full((len(row),), base_z, dtype=torch.float64, device="cuda")
    for h in hs:
        h.update_poses_from_device(slots, xy, T, org, bz)


@pytest.mark.parametrize("dim,res,B,streams,device_pose", [
    (99.0, 0.33, 4, 2, False),      # N = 300, two slots per stream group
    (99.0, 0.33, 10, 3, True),      # ten slots over three stream groups, device poses
    (33.33, 0.33, 10, None, False),  # N = 101, ten slots over the eight default groups
    (33.33, 0.33, 4, None, True),
])
def test_parity_with_the_twin_over_a_rolling_stream(monkeypatch, dim, res, B, streams, device_pose):
    """8 steps: 1 ... 16 parts per scan, every count kind, a step that reuses the stored counts, steps that mix flagged
    and unflagged scans, capacities summing to max_points; every selection and labels only."""
    torch = torch_mod()
    if streams:
        monkeypatch.setenv("GG_STREAMS", str(streams))
    g, twin = make_pair(dim, res, B, max_points=MAX_POINTS)
    o = Oracle(dim, res)                                  # slot 0 runs the default configuration; it is last in the batch
    slots = np.arange(B, dtype=np.int32)[::-1].copy()
    rng = np.random.default_rng(8100 + B)
    seen_parts, kinds_seen = set(), set()
    prev = None
    for k, row in enumerate(make_steps(B, 8, seed=8100 + B)):
        base_z = 0.02 * k
        if device_pose and k:
            set_poses((g, twin), slots, row, base_z)
        else:
            advance((g, twin), k, row, slots)
            if device_pose:
                set_poses((g, twin), slots, row, base_z)
        if k == 0:
            o.init_map(row[-1][2][0], row[-1][2][1], 0.0)
        else:
            o.update(row[-1][2][0], row[-1][2][1], row[-1][3])
        reuse = k == 3                                    # no store: the counts of step 2 again
        n_parts = prev[0] if reuse else [1 + (5 * b + 3 * k) % P for b in range(B)]
        flagged = [(b + k) % 4 != 1 for b in range(B)] if k in (2, 6) else None
        rig = Rig(torch, row, k, rng, n_parts, stored=prev[1] if reuse else None, flagged=flagged, fill_to=None if reuse else k % B)
        if not reuse:
            g.set_part_counts_from_device(slots, rig.counts(torch))
        seen_parts |= set(n_parts)
        kinds_seen |= {(q[7] == q[6], q[7] == 0, q[6] == 0) for s in rig.scans for q in s}
        select = ("all", "nonground", "ground", None)[k % 4]
        origins = "device" if device_pose else [r[1] for r in row]
        out = rig.call(g, slots, origins, base_z, select, True)
        want = rig.call(twin, slots, origins, base_z, select, False)
        ctx = f"step {k}"
        check(out, want, rig.us, ctx)
        ol, _, _ = o.filter_cloud(rig.concat(B - 1), row[-1][1], base_z, threads=1)
        assert np.array_equal(out.labels[-1][:rig.us[-1]].cpu().numpy(), ol), f"{ctx}: oracle"
        assert_twin(g, twin, slots, rig.us, rig.caps, ctx)
        prev = (n_parts, [[q[5] for q in s] + [0] * (P - len(s)) for s in rig.scans])
    assert seen_parts >= {1, P} and len(kinds_seen) >= 4
    g.close()
    twin.close()


@pytest.mark.parametrize("which", ["legacy", "side"])
def test_counts_written_behind_a_sleep_then_freed_and_refilled(which):
    """Counts (and payloads) produced on the stream behind ~200 ms of device work are waited for on the device, and
    freeing and refilling the counts right after the store does not race with the scans."""
    torch = torch_mod()
    B = 4
    g, twin = make_pair(99.0, 0.33, B, max_points=MAX_POINTS)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(8200)
    stream = torch.cuda.default_stream() if which == "legacy" else torch.cuda.Stream()
    steps = make_steps(B, 2, seed=8200)
    for k, row in enumerate(steps):
        advance((g, twin), k, row, slots)
        rig = Rig(torch, row, k + 4, rng, [4, 7, 2, 16])
        src = rig.counts(torch)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            counts = torch.zeros_like(src)
            torch.cuda._sleep(400_000_000)
            counts.copy_(src)
            before = torch.cuda.Event()
            before.record(stream)
            g.set_part_counts_from_device(slots, counts, stream=stream)
            del counts
            refill = torch.full((B, P), 3, dtype=torch.int32, device="cuda")   # takes the freed block
            out = rig.call(g, slots, [r[1] for r in row], 0.0, "all", True, stream=stream)
            assert k == 0 or not before.query(), "a call waited on the host for the stream"
        want = rig.call(twin, slots, [r[1] for r in row], 0.0, "all", False)
        check(out, want, rig.us, f"{which} step {k}")
        assert_twin(g, twin, slots, rig.us, rig.caps, f"{which} step {k}")
        del refill
    g.close()
    twin.close()


def test_init_map_forgets_the_part_counts_and_device_resets_keep_them():
    torch = torch_mod()
    B = 3
    g, twin = make_pair(99.0, 0.33, B, max_points=MAX_POINTS)
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(8300)
    row = make_steps(B, 1, seed=8300)[0]
    advance((g, twin), 0, row, slots)
    rig = Rig(torch, row, 0, rng, [3, 3, 3])
    g.set_part_counts_from_device(slots, rig.counts(torch))
    # gg_init_maps_from_device keeps them
    xyz = torch.tensor([[r[2][0], r[2][1], 0.0] for r in row], dtype=torch.float64, device="cuda")
    g.init_maps_from_device(slots, xyz)
    twin.init_maps_from_device(slots, xyz)
    again = Rig(torch, row, 1, rng, [3, 3, 3], stored=[[q[5] for q in s] for s in rig.scans])
    out = again.call(g, slots, [r[1] for r in row], 0.0, "all", True)
    want = again.call(twin, slots, [r[1] for r in row], 0.0, "all", False)
    check(out, want, again.us, "after device resets")
    assert_twin(g, twin, slots, again.us, again.caps, "after device resets")
    # gg_init_map forgets them: a flagged scan of that slot is GG_E_STATE and enqueues nothing
    g.init_map(row[1][2][0], row[1][2][1], 0.0, slot=1)
    l0 = g.kernel_launches
    with pytest.raises(capi.GroundGridError) as e:
        again.call(g, slots, [r[1] for r in row], 0.0, "all", True)
    assert e.value.code == STATE and "slot 1" in str(e.value) and g.kernel_launches == l0
    g.close()
    twin.close()


def test_rejections_enqueue_nothing():
    torch = torch_mod()
    B = 4
    g, _twin = make_pair(33.33, 0.33, B + 1, max_points=MAX_POINTS)    # slot B is never initialised
    _twin.close()
    slots = np.arange(B, dtype=np.int32)
    row = make_steps(B, 1, seed=8400)[0]
    advance((g,), 0, row, slots)
    rng = np.random.default_rng(8400)
    rig = Rig(torch, row, 0, rng, [2, 5, 3, 1])
    counts = rig.counts(torch)
    origins = [r[1] for r in row]
    torch.cuda.synchronize()

    def store(sl=slots, pps=P, ptr=None, stream=None):
        return lambda: g.set_part_counts_from_device_ptrs(sl, pps, counts.data_ptr() if ptr is None else ptr, stream)

    def flagged_call(flags=capi.SCAN_DEVICE_PART_COUNTS):
        def fn():
            data = [[q[0] for q in s] for s in rig.scans]
            n_parts, parts, keep = capi.cloud_parts([[t.numel() for t in s] for s in data], [[t.data_ptr() for t in s] for s in data],
                                                    [[q[2] for q in s] for s in rig.scans], [[q[3] for q in s] for s in rig.scans],
                                                    [[q[4] for q in s] for s in rig.scans])
            descs = g._device_descs(slots, rig.caps, origins, 0.0)
            descs["flags"][1] |= flags
            g.run_merged_cloud_msgs_to_device_ptrs(descs, n_parts, parts, None, 0, None, None)
        return fn

    def other_route(name):
        def fn():
            descs = g._device_descs(slots, [0] * B, origins, 0.0)
            descs["flags"][2] |= capi.SCAN_DEVICE_PART_COUNTS
            if name == "run_scans":
                capi._check(g._l.gg_run_scans(g._h, B, capi._ptr(descs), 0))
            elif name == "run_scans_device":
                g.run_scans_device(descs, [0] * B)
            elif name == "to_device":
                g.run_scans_to_device_ptrs(descs, [0] * B, None, 0, None, None)
            elif name == "msgs":
                g.run_cloud_msgs_to_device_ptrs(descs, [0] * B, 32, (0, 4, 8, 16, 20), None, None, 0, None, None)
            else:
                capi._check(g._l.gg_filter_cloud_batch(g._h, B, capi._ptr(descs), (C.c_void_p * B)(), None))
        return fn

    def raw_store(null_slots=False, null_counts=False):
        sl = np.ascontiguousarray(slots, np.int32)
        return lambda: capi._check(g._l.gg_set_part_counts_from_device(None if null_slots == "handle" else g._h, B,
                                                                       None if null_slots is True else capi._ptr(sl), P,
                                                                       None if null_counts else counts.data_ptr(), None))

    layer = g.layer_device_ptr("ground", slot=0)
    # before any store: a flagged scan is GG_E_STATE
    cases = [
        ("flagged scan without stored part counts", flagged_call(), STATE),
        ("null handle", raw_store(null_slots="handle"), ARG),
        ("null slots", raw_store(null_slots=True), ARG),
        ("null counts", raw_store(null_counts=True), ARG),
        ("count > n_slots", store(sl=list(range(B + 1)) + [0]), ARG),
        ("slot out of range", store(sl=[0, 1, 2, B + 1]), ARG),
        ("repeated slot", store(sl=[0, 1, 1, 3]), ARG),
        ("parts_per_slot 0", store(pps=0), ARG),
        ("parts_per_slot 17", store(pps=P + 1), ARG),
        ("misaligned", store(ptr=counts.data_ptr() + 2), ARG),
        ("overlaps the layers", store(ptr=layer), ARG),
        ("map not initialised", store(sl=[0, 1, 2, B]), STATE),
    ]
    for name in ("run_scans", "run_scans_device", "to_device", "msgs", "filter_cloud_batch"):
        cases.append((f"the flag on {name}", other_route(name), ARG))
    for name, fn, code in cases:
        l0 = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            fn()
        assert e.value.code == code, f"{name}: code {e.value.code} ({e.value})"
        assert g.kernel_launches == l0, f"{name}: something was launched"
    l0 = g.kernel_launches
    g.set_part_counts_from_device_ptrs([], P, None, None)
    assert g.kernel_launches == l0, "count 0 launched something"
    # stored for 4 parts: scan 1 has 5
    g.set_part_counts_from_device(slots, counts[:, :4].contiguous())
    torch.cuda.synchronize()
    for name, fn, code in (("more parts than stored", flagged_call(), STATE),
                           ("with GG_SCAN_DEVICE_COUNT", flagged_call(capi.SCAN_DEVICE_PART_COUNTS | capi.SCAN_DEVICE_COUNT), ARG),
                           ("GG_SCAN_DEVICE_COUNT alone", flagged_call(capi.SCAN_DEVICE_COUNT), ARG)):
        l0 = g.kernel_launches
        with pytest.raises(capi.GroundGridError) as e:
            fn()
        assert e.value.code == code and g.kernel_launches == l0, f"{name}: {e.value}"
    g.set_part_counts_from_device(slots, counts)
    flagged_call()()                                          # accepted once enough parts are stored
    torch.cuda.synchronize()
    g.close()

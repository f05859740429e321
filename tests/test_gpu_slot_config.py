"""Per-slot configuration (gg_set_slot_config) on the GPU: every slot of a batched handle runs with its own
GroundGridConfig, bit-exact against oracle instances that each carry that slot's configuration."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi, synth
from oracle import Oracle

pytestmark = pytest.mark.gpu

LIVE = ("points", "variance", "minGroundHeight", "ground", "groundpatch")
DEAD = ("m2", "meanVariance", "groundCandidates", "planeDist", "maxGroundHeight", "pointsRaw")

# Four configurations that differ in every field a kernel reads: ring cut-off (max_ring), confidence decay (both values
# of the floor shortcut: factor 2000 decays 0.001f to just above 0.000999), 3x3 / 5x5 split, label and outlier
# thresholds, patch-detection thresholds.
CFGS = [
    dict(),
    dict(max_ring=48, occupied_cells_decrease_factor=1.5, patch_size_change_distance=8.0, miminum_point_height_threshold=0.2,
         minimum_point_height_obstacle_threshold=0.05, outlier_tolerance=0.25, min_outlier_detection_ground_confidence=0.6,
         point_count_cell_variance_threshold=4),
    dict(max_ring=40, occupied_cells_decrease_factor=2000.0, patch_size_change_distance=30.0, distance_factor=0.0003,
         minimum_distance_factor=0.001, ground_patch_detection_minimum_point_count_threshold=0.15,
         occupied_cells_point_count_factor=8.0, outlier_tolerance=0.05),
    dict(occupied_cells_decrease_factor=1.5, patch_size_change_distance=12.0, outlier_tolerance=0.02,
         min_outlier_detection_ground_confidence=2.0, miminum_point_height_threshold=0.45,
         minimum_point_height_obstacle_threshold=0.2, point_count_cell_variance_threshold=20,
         ground_patch_detection_minimum_point_count_threshold=0.4, occupied_cells_point_count_factor=35.0),
]


def config_of(kw):
    c = capi.default_config()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def full(kw):
    """Every field of the configuration `kw` describes (defaults elsewhere): set_config(**kw) only changes the fields
    it is given, so a slot or oracle that ran another configuration before needs all of them."""
    c = config_of(kw)
    return {name: getattr(c, name) for name, _ in capi.Config._fields_}


def same_config(a, b):
    return bytes(a) == bytes(b)


# configurations no slot of the isolation tests starts with: moving a slot to one builds a variant (a new id, or the
# id the slot's previous configuration leaves unused, rebuilt)
FRESH = [dict(CFGS[2], outlier_tolerance=0.3), dict(CFGS[1], max_ring=56, outlier_tolerance=0.15)]


def set_slot_counting_builds(g, slot, kw):
    """set_config(slot=...) with a complete configuration; returns the detect tables it built (kernel launches)."""
    n0 = g.kernel_launches
    g.set_config(slot=slot, **full(kw))
    return g.kernel_launches - n0


def diff_report(name, a, b):
    bad = ~((a == b) | (np.isnan(a) & np.isnan(b)))
    if not bad.any():
        return None
    return f"{name}: {int(bad.sum())} cells differ"


def assert_slot_matches(g, slot, o, names, ctx):
    errs = [r for r in (diff_report(n, g.layer(n, slot=slot), o.layer(n)) for n in names) if r]
    assert not errs, f"{ctx}: " + " | ".join(errs)


def oracle_with(dim, res, kw):
    o = Oracle(dim, res)
    if kw:
        o.set_config(**full(kw))
    return o


def make_clouds(B, steps, seed):
    """[step][slot] -> (points, origin, ego xy, T): rolls, yaw, pitched base, pushed-down below-ground returns."""
    rng = np.random.default_rng(seed)
    scenes = [synth.make_scene(seed=seed + b, stream_len=10.0, undulation=0.2) for b in range(B)]
    out = []
    for k in range(steps):
        row = []
        for b in range(B):
            ex, ey, yaw = 0.8 * k + 0.05 * b, -0.35 * k * (b % 3), 0.04 * k * (1 + b % 2)
            pts, org = synth.lidar_scan(scenes[b], ego_xy=(ex, ey), yaw=yaw, beams=64, az_steps=768, seed=seed + 100 * k + b)
            if k:
                idx = rng.choice(len(pts), len(pts) // 200, replace=False)
                pts["z"][idx] -= rng.uniform(0.3, 1.2, len(idx)).astype(np.float32)
            row.append((pts, org, (ex, ey), synth.base_from_map(ex, ey, yaw, base_z=0.0, pitch=0.01)))
        out.append(row)
    return out


def test_the_four_configurations_cover_both_decay_floor_cases_and_differ_everywhere():
    consts = [capi.host_config_constants(config_of(kw)) for kw in CFGS]
    assert {c["decay_floor_ok"] for c in consts} == {0.0, 1.0}
    assert {c["max_ring"] for c in consts} == {1024.0, 48.0, 40.0}
    for name in consts[0]:
        if name != "decay_floor_ok":
            assert len({c[name] for c in consts}) >= 2, name


@pytest.mark.parametrize("dim,res,B,full_layers,path,pack", [
    (99.0, 0.33, 4, True, "device", None),      # N = 300: TMA patch detection, one thread per spiral lane
    (99.0, 0.33, 10, False, "batch", "0"),      # batch of ten: time-shared spiral layout, 32-byte records
    (99.0, 0.33, 10, True, "batch", "1"),       # packed host clouds
    (33.33, 0.33, 10, False, "device", None),   # N = 101: plain-load patch detection
    (33.33, 0.33, 4, True, "batch", "1"),
])
def test_mixed_configurations_in_one_batch(monkeypatch, dim, res, B, full_layers, path, pack):
    import torch

    if pack is not None:
        monkeypatch.setenv("GG_HOST_PACK", pack)
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536, full_layers=full_layers)
    kws = [CFGS[b % 4] for b in range(B)]        # interleaved: every stream group holds several configurations
    for b in range(B):
        g.set_config(slot=b, **full(kws[b]))
    oracles = [oracle_with(dim, res, kws[b]) for b in range(B)]
    steps = make_clouds(B, 3, seed=4000 + B)
    slots = np.arange(B, dtype=np.int32)
    names = LIVE + (DEAD if full_layers else ())
    for k, row in enumerate(steps):
        if k == 0:
            for b in range(B):
                g.init_map(row[b][2][0], row[b][2][1], 0.0, slot=b)
                oracles[b].init_map(row[b][2][0], row[b][2][1], 0.0)
        else:
            moved = g.update_pose_batch(slots, np.array([r[2] for r in row]), np.stack([r[3].reshape(12) for r in row]))
            for b in range(B):
                assert bool(moved[b]) == bool(oracles[b].update(row[b][2][0], row[b][2][1], row[b][3]))
        descs = g.make_descs(list(range(B)), [len(r[0]) for r in row], [r[1] for r in row], [0.02 * k] * B)
        if path == "device":
            dev = [torch.from_numpy(np.ascontiguousarray(r[0]).view(np.uint8).copy()).cuda() for r in row]
            torch.cuda.synchronize()
            g.run_scans_device(descs, [t.data_ptr() for t in dev])
            labels = [g.download_labels(len(r[0]), slot=b) for b, r in enumerate(row)]
            g.synchronize()
        else:
            hp = [torch.from_numpy(np.ascontiguousarray(r[0]).view(np.uint8).copy()).pin_memory() for r in row]
            hl = [torch.zeros(len(r[0]), dtype=torch.uint8).pin_memory() for r in row]
            g.filter_cloud_batch_ptrs(descs, [t.data_ptr() for t in hp], [t.data_ptr() for t in hl])
            labels = [t.numpy().copy() for t in hl]
        for b in range(B):
            want, want_idx, _ = oracles[b].filter_cloud(row[b][0], row[b][1], 0.02 * k, threads=1)
            assert np.array_equal(labels[b], want), f"step {k} slot {b}: {(labels[b] != want).sum()} labels differ"
            idx, _ = g.get_output(slot=b)
            assert np.array_equal(idx, want_idx), f"step {k} slot {b}: output order"
            assert_slot_matches(g, b, oracles[b], names, f"step {k} slot {b}")
        if path == "device":
            del dev
    g.close()


def test_per_phase_entries_use_the_slots_configuration():
    dim, res = 33.0, 0.33
    g = capi.GroundGridB200(dim, res, n_slots=3, max_points=40000, full_layers=True)
    g.set_config(**full(CFGS[1]))                  # handle-wide
    g.set_config(slot=0, **full(CFGS[3]))
    g.set_config(slot=2, **full(CFGS[2]))          # differs from slot 0 and from the handle-wide one
    assert same_config(g.get_config(), config_of(CFGS[1])) and same_config(g.get_config(slot=1), config_of(CFGS[1]))
    o = oracle_with(dim, res, CFGS[2])
    twin = capi.GroundGridB200(dim, res, n_slots=1, max_points=40000, full_layers=True)
    twin.set_config(**full(CFGS[2]))
    scene = synth.make_scene(seed=21, n_boxes=8, rmin=4.0, rmax=14.0)
    for m, kw in ((g, {"slot": 2}), (twin, {}), (o, {})):
        m.init_map(0.0, 0.0, 0.0, **kw)
    for k in range(2):
        pts, org = synth.lidar_scan(scene, beams=64, az_steps=512, seed=210 + k)
        if k:
            pts["z"][::41] -= 0.7
        g.run_single(pts, org, 0.25, slot=2, stop_after=1)
        o.filter_cloud(pts, org, 0.25, threads=1, stop_after=1)
        assert_slot_matches(g, 2, o, ("points", "minGroundHeight") + DEAD, f"scan {k} stage 1")
        g.detect_ground_patches(slot=2)
        g.synchronize()
        o.filter_cloud(pts, org, 0.25, threads=1, stop_after=2)   # stage 1 again on the same prior, then stage 2
        assert_slot_matches(g, 2, o, ("ground", "groundpatch", "variance"), f"scan {k} detect_ground_patches")
        g.spiral_ground_interpolation(0.25, slot=2)
        g.synchronize()
        o.spiral(0.25)
        assert_slot_matches(g, 2, o, ("ground", "groundpatch"), f"scan {k} spiral_ground_interpolation")
    # detect_ground_patch<3|5> on single cells: the same calls on a one-slot handle that runs CFGS[2] handle-wide
    pts, org = synth.lidar_scan(scene, beams=64, az_steps=512, seed=299)
    g.run_single(pts, org, 0.0, slot=2, stop_after=1)
    twin.set_layer("ground", g.layer("ground", slot=2))
    twin.set_layer("groundpatch", g.layer("groundpatch", slot=2))
    twin.run_single(pts, org, 0.0, stop_after=1)
    n = g.n
    for S in (3, 5):
        for i in range(n // 2 - 12, n // 2 + 12, 2):
            for j in range(n // 2 - 12, n // 2 + 12, 3):
                g.detect_ground_patch(S, i, j, slot=2)
                twin.detect_ground_patch(S, i, j)
    g.synchronize()
    twin.synchronize()
    for name in ("ground", "groundpatch"):
        assert np.array_equal(g.layer(name, slot=2), twin.layer(name)), f"detect_ground_patch: {name}"
    # interpolate_cell: the decay of CFGS[2] (factor 2000, no floor shortcut)
    rng = np.random.default_rng(3)
    G = rng.normal(0.0, 0.4, (n, n)).astype(np.float32)
    Cf = rng.uniform(0.0, 1.0, (n, n)).astype(np.float32)
    for name, arr in (("ground", G), ("groundpatch", Cf)):
        g.set_layer(name, arr, slot=2)
        o.set_layer(name, arr)
    for x, y in ((5, 7), (48, 49), (49, 49), (1, 1), (97, 97), (20, 80)):
        g.interpolate_cell(x, y, slot=2)
        o.interpolate_cell(x, y)
    g.synchronize()
    assert_slot_matches(g, 2, o, ("ground", "groundpatch"), "interpolate_cell")
    g.close()
    twin.close()


def run_device_step(g, torch, row, slots, k, sync=True):
    dev = [torch.from_numpy(np.ascontiguousarray(row[b][0]).view(np.uint8).copy()).cuda() for b in slots]
    torch.cuda.synchronize()
    if k:
        g.update_pose_batch(np.array(slots, np.int32), np.array([row[b][2] for b in slots]), np.stack([row[b][3].reshape(12) for b in slots]))
    descs = g.make_descs(list(slots), [len(row[b][0]) for b in slots], [row[b][1] for b in slots], [0.0] * len(slots))
    g.run_scans_device(descs, [t.data_ptr() for t in dev])
    if sync:
        g.synchronize()
    return dev


def test_reconfiguring_one_slot_leaves_every_other_slot_untouched():
    import torch

    dim, res, B = 66.0, 0.33, 8
    a = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536, full_layers=False)
    t = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536, full_layers=False)
    for h in (a, t):
        for b in range(B):
            h.set_config(slot=b, **full(CFGS[b % 4]))
    steps = make_clouds(B, 3, seed=6100)
    o3 = oracle_with(dim, res, CFGS[3])
    for b in range(B):
        for h in (a, t):
            h.init_map(steps[0][b][2][0], steps[0][b][2][1], 0.0, slot=b)
    o3.init_map(steps[0][3][2][0], steps[0][3][2][1], 0.0)
    for k, row in enumerate(steps):
        if k:
            # step 1: a configuration no slot uses (new variant); step 2: another one (the variant of step 1 is left
            # unused and rebuilt)
            assert set_slot_counting_builds(a, 3, FRESH[k - 1]) == 1
            o3.set_config(**full(FRESH[k - 1]))
        keep = [run_device_step(h, torch, row, list(range(B)), k) for h in (a, t)]
        if k:
            o3.update(row[3][2][0], row[3][2][1], row[3][3])
        want, _, _ = o3.filter_cloud(row[3][0], row[3][1], 0.0, threads=1)
        assert np.array_equal(a.download_labels(len(row[3][0]), slot=3), want), f"step {k}: reconfigured slot"
        for b in range(B):
            if b == 3:
                continue
            la, lt = a.download_labels(len(row[b][0]), slot=b), t.download_labels(len(row[b][0]), slot=b)
            a.synchronize()
            t.synchronize()
            assert np.array_equal(la, lt), f"step {k} slot {b}: labels"
            for name in LIVE:
                assert np.array_equal(a.layer(name, slot=b), t.layer(name, slot=b), equal_nan=True), f"step {k} slot {b}: {name}"
        del keep
    a.close()
    t.close()


def test_reconfiguring_a_slot_of_another_stream_group_while_scans_run():
    import torch

    dim, res, B = 99.0, 0.33, 8
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536, full_layers=False)
    assert g.n_streams > 1
    group = lambda s: s * g.n_streams // B   # noqa: E731  (slots are bound to streams in contiguous groups)
    for b in range(B):
        g.set_config(slot=b, **full(CFGS[b % 4]))
    oracles = [oracle_with(dim, res, CFGS[b % 4]) for b in range(B)]
    steps = make_clouds(B, 3, seed=7300)
    for b in range(B):
        g.init_map(steps[0][b][2][0], steps[0][b][2][1], 0.0, slot=b)
        oracles[b].init_map(steps[0][b][2][0], steps[0][b][2][1], 0.0)
    target = B - 1
    a_slots = [b for b in range(B) if group(b) != group(target)]
    for k, row in enumerate(steps):
        keep = run_device_step(g, torch, row, a_slots, k, sync=False)
        # group A's kernels are enqueued and not synchronised: a slot of another group changes its configuration.
        # Step 0: to one no slot uses (a new variant id is allocated and built); step 1: to another (the id of step 0
        # is left unused and rebuilt); step 2: to one other slots use (nothing is built).
        new_kw = [FRESH[0], FRESH[1], CFGS[0]][k]
        assert set_slot_counting_builds(g, target, new_kw) == (1 if k < 2 else 0)
        oracles[target].set_config(**full(new_kw))
        g.synchronize()
        for b in a_slots:
            if k:
                oracles[b].update(row[b][2][0], row[b][2][1], row[b][3])
            want, _, _ = oracles[b].filter_cloud(row[b][0], row[b][1], 0.0, threads=1)
            got = g.download_labels(len(row[b][0]), slot=b)
            g.synchronize()
            assert np.array_equal(got, want), f"step {k} slot {b}"
            assert_slot_matches(g, b, oracles[b], LIVE, f"step {k} slot {b}")
        keep2 = run_device_step(g, torch, row, [target], k)
        if k:
            oracles[target].update(row[target][2][0], row[target][2][1], row[target][3])
        want, _, _ = oracles[target].filter_cloud(row[target][0], row[target][1], 0.0, threads=1)
        assert np.array_equal(g.download_labels(len(row[target][0]), slot=target), want)
        g.synchronize()
        assert_slot_matches(g, target, oracles[target], LIVE, f"step {k} reconfigured slot")
        del keep, keep2
    g.close()


def test_slot_configuration_semantics():
    import torch

    dim, res, B = 33.0, 0.33, 4
    g = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536, full_layers=False)
    d = capi.default_config()
    assert all(same_config(g.get_config(slot=b), d) for b in range(B)) and same_config(g.get_config(), d)
    # round trip, thread_count included (accepted, unused)
    for b in range(B):
        g.set_config(slot=b, thread_count=b + 1, **CFGS[b])
        assert same_config(g.get_config(slot=b), config_of(dict(CFGS[b], thread_count=b + 1)))
    assert same_config(g.get_config(), d)
    # the configuration survives a new map
    steps = make_clouds(B, 1, seed=8800)
    row = steps[0]
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
        assert same_config(g.get_config(slot=b), config_of(dict(CFGS[b], thread_count=b + 1)))
    keep = run_device_step(g, torch, row, list(range(B)), 0)
    for b in range(B):
        o = oracle_with(dim, res, CFGS[b])
        o.init_map(0.0, 0.0, 0.0)
        want, _, _ = o.filter_cloud(row[b][0], row[b][1], 0.0, threads=1)
        assert np.array_equal(g.download_labels(len(row[b][0]), slot=b), want), f"slot {b} after init_map"
        g.synchronize()
    del keep
    # the handle-wide call replaces every slot's configuration
    g.set_config(**full(CFGS[2]))
    assert all(same_config(g.get_config(slot=b), config_of(CFGS[2])) for b in range(B))
    assert same_config(g.get_config(), config_of(CFGS[2]))
    # every slot set one by one to X == X set handle-wide, bit for bit
    p = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536, full_layers=False)
    q = capi.GroundGridB200(dim, res, n_slots=B, max_points=65536, full_layers=False)
    for b in range(B):
        p.set_config(slot=b, **full(CFGS[1]))
    q.set_config(**full(CFGS[1]))
    for h in (p, q):
        for b in range(B):
            h.init_map(0.0, 0.0, 0.0, slot=b)
    keep = [run_device_step(h, torch, row, list(range(B)), 0) for h in (p, q)]
    for b in range(B):
        lp, lq = p.download_labels(len(row[b][0]), slot=b), q.download_labels(len(row[b][0]), slot=b)
        p.synchronize()
        q.synchronize()
        assert np.array_equal(lp, lq)
        for name in LIVE:
            assert np.array_equal(p.layer(name, slot=b), q.layer(name, slot=b), equal_nan=True), (b, name)
    del keep
    # error codes
    L = capi.load()
    cfg = capi.default_config()
    assert L.gg_set_slot_config(None, 0, C.byref(cfg)) == -1
    assert L.gg_get_slot_config(None, 0, C.byref(cfg)) == -1
    assert L.gg_set_slot_config(g._h, 0, None) == -1
    assert L.gg_get_slot_config(g._h, 0, None) == -1
    for bad in (-1, B):
        assert L.gg_set_slot_config(g._h, bad, C.byref(cfg)) == -1
        assert L.gg_get_slot_config(g._h, bad, C.byref(cfg)) == -1
    with pytest.raises(capi.GroundGridError) as e:
        g.set_config(slot=B, max_ring=3)
    assert e.value.code == -1
    for h in (g, p, q):
        h.close()

"""Configurations at the limits of every GroundGridConfig field (tests/config_limits.py) through the CUDA path, bit for
bit (NaN-aware) against the reference's stored answers and against the oracle port: one slot configured on the host,
eight slots over three stream groups configured on the host and from device memory, the spiral's lane layouts on every
decrease factor of the cases, and a step plan whose configurations are rewritten before each replay."""
import numpy as np
import pytest

import config_limits as cl
import ref_scenarios as rs
import spiral_priors as sp
from groundgrid_b200 import capi, synth
from oracle import Oracle
from test_gpu_device_configs import EDGE
from test_gpu_device_outputs import DEAD, LIVE, torch_mod
from test_gpu_slot_config import config_of, full
from test_gpu_spiral_layouts import RES, _edge_scan, _planted_errors, dim_of, import_prior, layer_errors, layout_id

pytestmark = pytest.mark.gpu

B, GROUPS = 8, 3
NAMES = list(cl.CASES)
SPARSE = np.array([1, 0, 0, 1, 0, 1, 0, 0], np.int32)


def capacity(stream):
    return max(len(pts) for *_, pts, _ in stream)


def records(torch, pts):
    return torch.from_numpy(np.ascontiguousarray(pts).view(np.float32).reshape(-1, 8).copy()).cuda()


def check_slot(g, o, s, labels, index, cloud, want, names, ctx):
    """Labels, output order and cloud of one scan, and the layers `names` of slot s, against the oracle's."""
    wl, wi, wc = want
    assert np.array_equal(labels, wl), f"{ctx}: {(labels != wl).sum()} labels differ"
    assert np.array_equal(index.astype(np.int64), wi.astype(np.int64)), f"{ctx}: output order"
    got = np.frombuffer(cloud.tobytes(), synth.POINT_DTYPE)
    for f in rs.CLOUD_FIELDS:
        assert np.array_equal(got[f], wc[f], equal_nan=True), f"{ctx}: cloud.{f}"
    errs = layer_errors(g, o, names, slot=s)
    assert not errs, f"{ctx}: " + " | ".join(errs)


@pytest.mark.parametrize("n", list(rs.DENSE_GEOMETRY))
def test_single_slot_against_the_reference(n):
    """tests/ref_scenarios.py:config_limits through one slot configured with gg_set_config: every digest the reference
    stored (N = 100: the TMA detection and the skewed spiral; N = 101: plain-load detection on an odd map)."""
    cap = capacity(rs.config_limits_stream(n))
    rs.run("config_limits", lambda dim, res: rs.Cuda(dim, res, cap), n)


@pytest.mark.parametrize("full_layers", [False, True], ids=["live", "full"])
@pytest.mark.parametrize("how", ["host", "device"])
def test_batched_slots_against_the_oracle(monkeypatch, how, full_layers):
    """Eight slots over three stream groups, each on its own case, all cases in turn: configured with gg_set_slot_config
    (host) or with two gg_set_slot_configs_from_device calls under a sparse mask and its complement (device); then
    update_pose_batch and run_scans_to_device on three scans; every slot against its own oracle after every scan."""
    torch = torch_mod()
    monkeypatch.setenv("GG_STREAMS", str(GROUPS))
    stream = rs.config_limits_stream(100)
    g = capi.GroundGridB200(33.0, 0.33, n_slots=B, max_points=capacity(stream), full_layers=full_layers)
    assert g.n_streams == GROUPS
    names = LIVE + DEAD if full_layers else LIVE
    slots = [3, 6, 0, 5, 1, 7, 2, 4]
    clouds = [records(torch, pts) for *_, pts, _ in stream]
    for b in range(0, len(NAMES), B):
        batch = [NAMES[(b + j) % len(NAMES)] for j in range(B)]
        kws = [full(cl.CASES[nm]) for nm in batch]
        if how == "host":
            for s, kw in zip(slots, kws):
                g.set_config(slot=s, **kw)
        else:
            ct = capi.config_tensor(kws)
            for mask in (SPARSE, 1 - SPARSE):
                g.set_configs_from_device(slots, ct, torch.tensor(mask, device="cuda"))
        oracles = []
        for s, kw in zip(slots, kws):
            assert bytes(g.get_config(slot=s)) == bytes(config_of(kw)), f"slot {s}: stored configuration"
            g.init_map(0.0, 0.0, 0.0, slot=s)
            o = Oracle(33.0, 0.33)
            o.set_config(**kw)
            o.init_map(0.0, 0.0, 0.0)
            oracles.append(o)
        for k, (ex, ey, yaw, base_z, pts, org) in enumerate(stream):
            if k:
                T = synth.base_from_map(ex, ey, yaw, base_z=base_z, pitch=0.02)
                moved = g.update_pose_batch(slots, [(ex, ey)] * B, [T] * B)
                for j, o in enumerate(oracles):
                    assert int(moved[j]) == o.update(ex, ey, T), f"{batch[j]} roll {k}: moved"
            out = g.run_scans_to_device([clouds[k]] * B, slots, [org] * B, base_z, labels=True, select="all", index=True)
            torch.cuda.synchronize()
            cloud, index = out.trimmed()
            for j, (s, o) in enumerate(zip(slots, oracles)):
                want = o.filter_cloud(pts, org, base_z, threads=1, want_cloud=True)
                check_slot(g, o, s, out.labels[j].cpu().numpy(), index[j].cpu().numpy(), cloud[j].cpu().numpy(), want, names,
                           f"{how} [{batch[j]}] slot {s} scan {k}")
    g.close()


SPIRAL_SIZES = [12, 468, 1200, 1600]   # pipe, skew (two phases), pipe 1024, plain


@pytest.mark.parametrize("factor", cl.decay_factors(), ids=repr)
@pytest.mark.parametrize("n", SPIRAL_SIZES, ids=layout_id)
def test_spiral_paths_on_every_decrease_factor(n, factor):
    """A prior with confidences at and around 0.001f, -0, negative, denormal and FLT_MAX on cells of every kind the sweep
    treats apart (tests/spiral_priors.py), then gg_spiral_ground_interpolation and a scan, against the oracle: the decay's
    floor shortcut on both sides of its switch, and the factors it must not take it for (0, 0.5, negative, non-finite)."""
    dim = dim_of(n)
    planted = sp.edge_cases(n, RES)["dense finite"]
    G, C = sp.planted_prior(n, RES, planted, seed=n)
    pts, org = _edge_scan(n)
    cfg = dict(occupied_cells_decrease_factor=factor, thread_count=1)
    g = capi.GroundGridB200(dim, RES, n_slots=1, max_points=max(len(pts), 1024), full_layers=False)
    o = Oracle(dim, RES)
    g.set_config(**cfg)
    o.set_config(**cfg)
    g.init_map(0.0, 0.0, 0.0)
    o.init_map(0.0, 0.0, 0.0)
    import_prior((g, o), G, C)
    g.spiral_ground_interpolation(0.1)
    o.spiral(0.1)
    errs = layer_errors(g, o, ("ground", "groundpatch")) + _planted_errors(g, o, planted)
    assert not errs, f"N {n} factor {factor!r} spiral: " + " | ".join(errs[:3])
    labels = g.filter_cloud(pts, org, 0.1)
    want, _, _ = o.filter_cloud(pts, org, 0.1, threads=1)
    assert np.array_equal(labels, want), f"N {n} factor {factor!r} scan: {(labels != want).sum()} labels differ"
    errs = layer_errors(g, o, LIVE)
    assert not errs, f"N {n} factor {factor!r} scan: " + " | ".join(errs[:3])
    g.close()


def need_bound_planes(n, dim, res):
    """A configuration and imported planes that put the point-count bound of :364 on 2^24 + 1 at one cell (a double that
    float rounds to nearest down to 2^24) and the window sum there at exactly 2^24: the reference skips the cell, and so
    must the detect table's bound, rounded up to float.  Passing it would take the local-minimum branch (ground -1).
    Returns (config, planes, cell)."""
    o = Oracle(dim, res)
    i, j = n // 2 - 5, n // 2 - 3           # 3 x 3 window at the default patch_size_change_distance
    e = float(o.expected_points()[i, j])
    bound = 2.0**24 + 1.0
    gp = (bound + 0.5) / (3.0 * e)
    assert np.floor(gp * 3.0 * e) == bound and float(np.float32(bound)) == 2.0**24
    zero = np.zeros((n, n), np.float32)
    planes = {name: zero.copy() for name in ("points", "m2", "minGroundHeight", "ground", "groundpatch", "variance")}
    planes["points"][i, j] = 2.0**24
    planes["minGroundHeight"][i, j] = -1.0
    return dict(ground_patch_detection_minimum_point_count_threshold=gp, thread_count=1), planes, (i, j)


@pytest.mark.parametrize("n", list(rs.DENSE_GEOMETRY))
def test_detect_table_bound_above_2_24(n):
    """need_bound_planes through detect_ground_patches on a slot configured on the host and on one configured from device
    memory (its detect table rebuilt on the device): ground, groundpatch and variance against the oracle, which skips
    the cell."""
    torch = torch_mod()
    dim, res = rs.DENSE_GEOMETRY[n]
    cfg, planes, (i, j) = need_bound_planes(n, dim, res)
    o = Oracle(dim, res)
    o.set_config(**cfg)
    o.init_map(0.0, 0.0, 0.0)
    for name in ("groundCandidates", "m2", "variance"):
        o.add_layer(name, 0.0)
    for name, a in planes.items():
        o.set_layer(name, a)
    o.detect_ground_patches()
    assert o.layer("ground")[i, j] == 0.0, "the reference's bound skips the cell"
    g = capi.GroundGridB200(dim, res, n_slots=2, max_points=1024, full_layers=True)
    g.set_config(slot=0, **full(cfg))
    g.set_configs_from_device([1], capi.config_tensor([full(cfg)]), torch.ones(1, dtype=torch.int32, device="cuda"))
    for s in (0, 1):
        g.init_map(0.0, 0.0, 0.0, slot=s)
        for name, a in planes.items():
            g.set_layer(name, a, slot=s)
        g.detect_ground_patches(slot=s)
        errs = layer_errors(g, o, ("ground", "groundpatch", "variance"), slot=s)
        assert not errs, f"N {n} slot {s}: " + " | ".join(errs)
    g.close()


def test_step_plan_with_edge_configurations(monkeypatch):
    """One gg_step_plan_create_with_configs plan over eight slots in three stream groups, replayed six times with the edge
    configurations of tests/test_gpu_device_configs.py (NaN and +-inf in every double field, ring cut-offs of 0 and
    below, INT_MAX variance threshold, decay factors 0 and 0.5, moved patch-size boundaries) written into its config
    tensor before each replay, with a roll and a scan: every slot against its own oracle after each replay."""
    torch = torch_mod()
    monkeypatch.setenv("GG_STREAMS", str(GROUPS))
    replays = 6
    stream = rs.config_limits_stream(100, scans=replays)
    cap = capacity(stream)
    g = capi.GroundGridB200(33.0, 0.33, n_slots=B, max_points=cap, full_layers=True)
    assert g.n_streams == GROUPS
    slots = [5, 2, 7, 0, 3, 6, 1, 4]
    buf = [torch.zeros((cap, 8), dtype=torch.float32, device="cuda") for _ in slots]
    counts = torch.zeros(B, dtype=torch.int32, device="cuda")
    xy = torch.zeros((B, 2), dtype=torch.float64, device="cuda")
    T = torch.zeros((B, 12), dtype=torch.float64, device="cuda")
    pose_origins = torch.zeros((B, 3), dtype=torch.float32, device="cuda")
    pose_base_z = torch.zeros(B, dtype=torch.float64, device="cuda")
    ct = capi.config_tensor([{}] * B)
    oracles = []
    for s in slots:
        g.init_map(0.0, 0.0, 0.0, slot=s)
        o = Oracle(33.0, 0.33)
        o.init_map(0.0, 0.0, 0.0)
        oracles.append(o)
    plan = g.step_plan(slots, clouds=buf, counts=counts, xy=xy, T_base_from_map=T, pose_origins=pose_origins,
                       pose_base_z=pose_base_z, origins="device", labels=True, select="all", index=True, configs=ct)
    for r, (ex, ey, yaw, base_z, pts, org) in enumerate(stream):
        kws = [full(dict(EDGE[(r * B + j) % len(EDGE)], thread_count=1)) for j in range(B)]
        Tr = synth.base_from_map(ex, ey, yaw, base_z=base_z, pitch=0.02)
        dev = records(torch, pts)
        for b in buf:
            b[:len(pts)].copy_(dev)
        counts.fill_(len(pts))
        xy.copy_(torch.tensor([[ex, ey]] * B, dtype=torch.float64))
        T.copy_(torch.from_numpy(np.tile(Tr.reshape(1, 12), (B, 1))))
        pose_origins.copy_(torch.from_numpy(np.tile(np.asarray(org, np.float32).reshape(1, 3), (B, 1))))
        pose_base_z.fill_(base_z)
        ct.copy_(capi.config_tensor(kws))
        plan.launch()
        torch.cuda.synchronize()
        cloud, index = plan.outputs.trimmed()
        for j, (s, o) in enumerate(zip(slots, oracles)):
            ctx = f"replay {r} slot {s} {EDGE[(r * B + j) % len(EDGE)]}"
            o.set_config(**kws[j])
            o.update(ex, ey, Tr)
            want = o.filter_cloud(pts, org, base_z, threads=1, want_cloud=True)
            check_slot(g, o, s, plan.outputs.labels[j][:len(pts)].cpu().numpy(), index[j].cpu().numpy(), cloud[j].cpu().numpy(),
                       want, LIVE + DEAD, ctx)
            assert bytes(g.get_config(slot=s)) == bytes(config_of(kws[j])), f"{ctx}: stored configuration"
    plan.close()
    g.close()

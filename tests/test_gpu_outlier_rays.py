"""The outlier test of k_rasterize on the priors and rays of tests/outlier_rays.py, bit for bit against the oracle: labels,
output order and cloud, every live and dead layer, and the point classes after a rasterising-only scan (PC_OUTLIER on
exactly the oracle's outliers).  Each case's prior is imported with gg_set_layer or gg_set_layers_from_device, as a
migrated slot brings one; the rays sit on every decision of the march, including rays whose occluder lies past step
2^20 or whose origin lies 2e6 m outside the map, which k_rasterize finishes with its exact walk."""
import numpy as np
import pytest

import outlier_rays as orr
import ref_scenarios as rs
from groundgrid_b200 import capi
from oracle import Oracle
from test_gpu_parity import DEAD, LIVE, diff_report

pytestmark = pytest.mark.gpu

ALL = ("points",) + LIVE + DEAD
PC_OUTLIER = 5
SETS = {"n100": (100, (0.0, 0.0), True), "n101": (101, (0.0, 0.0), False), "n300": (300, (0.0, 0.0), False), "far": (100, orr.FAR, False)}
_cache = {}


def case_set(name):
    if name not in _cache:
        n, pos, heavy = SETS[name]
        _cache[name] = orr.cases(n, pos, heavy)
    return _cache[name]


def oracle_for(c):
    o = Oracle(c.dim, c.res)
    if c.cfg:
        o.set_config(**c.cfg)
    o.init_map(float(c.position[0]), float(c.position[1]), 0.0)
    o.set_layer("ground", c.G)
    o.set_layer("groundpatch", c.C)
    return o


def import_prior(g, c, slot, how):
    if how == "set_layer":
        g.set_layer("ground", c.G, slot=slot)
        g.set_layer("groundpatch", c.C, slot=slot)
    else:
        import torch

        src = torch.from_numpy(np.stack([c.G, c.C])[None].copy()).cuda()
        g.set_layers_from_device([slot], ("ground", "groundpatch"), src)
        torch.cuda.synchronize()


def prepare(g, c, slot=0, how="set_layer"):
    g.set_config(slot=slot, **dict(capi_default(), **c.cfg))
    g.init_map(float(c.position[0]), float(c.position[1]), 0.0, slot=slot)
    import_prior(g, c, slot, how)


def capi_default():
    import pyref

    return {k: v for k, v in pyref.DEFAULT_CFG.items() if k in ("min_outlier_detection_ground_confidence", "outlier_tolerance")}


def layer_errors(g, o, slot, ctx):
    return [f"{ctx}: {r}" for r in (diff_report(x, g.layer(x, slot=slot), o.layer(x)) for x in ALL) if r]


def check_case(g, c, how):
    """Rasterising-only scan (point classes) and a whole scan (labels, order, cloud, layers) of case c on slot 0."""
    errs = []
    pts = c.cloud()
    prepare(g, c, 0, how)
    o = oracle_for(c)
    g.run_single(pts, c.origin, 0.0, stop_after=1)
    o.filter_cloud(pts, c.origin, 0.0, threads=1, stop_after=1)
    outlier = (g.point_classes(len(pts)) >> 24) == PC_OUTLIER
    want = np.array([c.want[0]])
    if not np.array_equal(outlier, want):
        errs.append(f"{c.name}: gpu outlier={bool(outlier[0])} oracle={bool(want[0])} (hit step {c.want[1]})")
    errs += layer_errors(g, o, 0, f"{c.name} stop_after=1")
    prepare(g, c, 0, how)
    o = oracle_for(c)
    labels, index, cloud = g.filter_cloud(pts, c.origin, 0.0, want_index=True, want_cloud=True)
    lab_o, idx_o, cloud_o = o.filter_cloud(pts, c.origin, 0.0, threads=1, want_cloud=True)
    if not (np.array_equal(labels, lab_o) and np.array_equal(index, idx_o) and cloud.tobytes() == cloud_o.tobytes()):
        errs.append(f"{c.name}: labels / order / cloud gpu={labels.tolist()} {index.tolist()} cpu={lab_o.tolist()} {idx_o.tolist()}")
    errs += layer_errors(g, o, 0, f"{c.name} scan")
    return errs


@pytest.mark.parametrize("how", ["set_layer", "from_device"])
@pytest.mark.parametrize("which", list(SETS))
def test_every_case_against_the_oracle(which, how):
    cs = case_set(which)
    g = capi.GroundGridB200(cs[0].dim, cs[0].res, n_slots=1, max_points=1024, full_layers=True)
    assert g.n == cs[0].n
    fails = []
    for c in cs:
        fails += check_case(g, c, how)
    g.close()
    assert not fails, f"{which} {how}: {len(fails)} failing\n" + "\n".join(fails[:40])


def routed_labels(g, route, c, slot=0):
    import torch

    pts = c.cloud()
    if route == "filter_cloud":
        return g.filter_cloud(pts, c.origin, 0.0, slot=slot)
    if route.startswith("batch"):
        hp = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).pin_memory()
        hl = torch.zeros(len(pts), dtype=torch.uint8).pin_memory()
        g.filter_cloud_batch_ptrs(g.make_descs([slot], [len(pts)], [c.origin], [0.0]), [hp.data_ptr()], [hl.data_ptr()])
        return hl.numpy().copy()
    if route == "to_device":
        dev = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).cuda()
        out = g.run_scans_to_device([dev], [slot], [c.origin], 0.0, select="all", index=True)
    else:
        raw = np.zeros((len(pts), 18), np.uint8)
        for name, off, width in zip(("x", "y", "z", "intensity", "ring"), (0, 4, 8, 12, 16), (4, 4, 4, 4, 2)):
            raw[:, off:off + width] = np.ascontiguousarray(pts[name]).view(np.uint8).reshape(len(pts), width)
        dev = torch.from_numpy(raw).cuda()
        out = g.run_cloud_msgs_to_device([dev], 18, (0, 4, 8, 12, 16), None, [slot], [c.origin], 0.0, select="all", index=True)
    torch.cuda.synchronize()
    return out.labels[0].cpu().numpy()


@pytest.mark.parametrize("route", ["batch_packed", "batch_raw", "to_device", "cloud_msgs"])
def test_every_input_route(monkeypatch, route):
    if route.startswith("batch"):
        monkeypatch.setenv("GG_HOST_PACK", "1" if route == "batch_packed" else "0")
    cs = [c for c in case_set("n101") if c.regime.startswith(("long", "cell", "pretest", "direction"))]
    g = capi.GroundGridB200(cs[0].dim, cs[0].res, n_slots=1, max_points=1024, full_layers=True)
    fails = []
    for c in cs:
        prepare(g, c)
        o = oracle_for(c)
        labels = routed_labels(g, route, c)
        want, _, _ = o.filter_cloud(c.cloud(), c.origin, 0.0, threads=1)
        if not np.array_equal(labels, want):
            fails.append(f"{c.name}: labels {labels.tolist()} != {want.tolist()}")
        fails += layer_errors(g, o, 0, c.name)
    g.close()
    assert not fails, f"{route}: {len(fails)} failing\n" + "\n".join(fails[:40])


def test_batch_of_four_slots_over_two_stream_groups(monkeypatch):
    """Four slots, each with its own prior and ray, slots 1 and 3 with their own configuration, in one batched call per
    round; every round takes the next four cases."""
    import torch

    monkeypatch.setenv("GG_STREAMS", "2")
    cs = [c for c in case_set("n100") if not c.cfg]
    cfgs = {1: dict(min_outlier_detection_ground_confidence=0.6, outlier_tolerance=0.0), 3: dict(min_outlier_detection_ground_confidence=-1.0, outlier_tolerance=-0.3)}
    g = capi.GroundGridB200(cs[0].dim, cs[0].res, n_slots=4, max_points=1024, full_layers=True)
    assert g.n_streams == 2
    fails = []
    for r0 in range(0, len(cs) - 3, 4):
        group = cs[r0:r0 + 4]
        oracles = []
        for b, c in enumerate(group):
            c = orr.Case(c.name, c.n, c.position, c.G, c.C, c.origin, c.point, dict(cfgs.get(b, {})))
            group[b] = c
            prepare(g, c, b, "from_device" if b % 2 else "set_layer")
            oracles.append(oracle_for(c))
        hp = [torch.from_numpy(np.ascontiguousarray(c.cloud()).view(np.uint8).copy()).pin_memory() for c in group]
        hl = [torch.zeros(1, dtype=torch.uint8).pin_memory() for _ in group]
        g.filter_cloud_batch_ptrs(g.make_descs(list(range(4)), [1] * 4, [c.origin for c in group], [0.0] * 4),
                                  [t.data_ptr() for t in hp], [t.data_ptr() for t in hl])
        for b, (c, o) in enumerate(zip(group, oracles)):
            want, _, _ = o.filter_cloud(c.cloud(), c.origin, 0.0, threads=1)
            if not np.array_equal(hl[b].numpy(), want):
                fails.append(f"slot {b} {c.name}: labels {hl[b].numpy().tolist()} != {want.tolist()}")
            fails += layer_errors(g, o, b, f"slot {b} {c.name}")
    g.close()
    assert not fails, f"{len(fails)} failing\n" + "\n".join(fails[:40])


def test_roll_between_import_and_scan():
    """The imported prior rolled (the rolled prior seeds the exposed cells) before the scan, then a second scan on what
    the first left."""
    from groundgrid_b200 import synth

    cs = [c for c in case_set("n300") if c.regime.startswith(("long", "cell", "geometry"))]
    g = capi.GroundGridB200(cs[0].dim, cs[0].res, n_slots=1, max_points=1024, full_layers=True)
    fails = []
    for c in cs:
        prepare(g, c)
        o = oracle_for(c)
        ex, ey = float(c.position[0]) + 0.9, float(c.position[1]) - 0.7
        T = synth.base_from_map(ex, ey, 0.0, base_z=0.0, pitch=0.02)
        if int(g.update_pose(ex, ey, T)) != o.update(ex, ey, T):
            fails.append(f"{c.name}: moved")
        for k in range(2):
            labels = g.filter_cloud(c.cloud(), c.origin, 0.0)
            want, _, _ = o.filter_cloud(c.cloud(), c.origin, 0.0, threads=1)
            if not np.array_equal(labels, want):
                fails.append(f"{c.name} scan {k}: labels {labels.tolist()} != {want.tolist()}")
            fails += layer_errors(g, o, 0, f"{c.name} scan {k}")
    g.close()
    assert not fails, f"{len(fails)} failing\n" + "\n".join(fails[:40])


@pytest.mark.parametrize("n", rs.OUTLIER_SIZES)
def test_outlier_priors_against_the_reference_itself(n):
    """tests/ref_scenarios.py:outlier_priors on the CUDA path: every digest the reference stored."""
    rs.run("outlier_priors", lambda dim, res: rs.Cuda(dim, res, 1024), n)

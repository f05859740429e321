"""Patch detection on its own (gg_detect_ground_patches, gg_detect_ground_patch) on imported planes, bit for bit against
the oracle port, and the reference's stored answers replayed on the CUDA path.

Each case of tests/detect_planes.py is imported into slot 2 of a 3-slot handle, with and without GG_FLAG_FULL_LAYERS,
in three states of the slot: a fresh map, after a scan stopped after rasterising ("points" is then the kept-point count)
and after a complete scan ("points" is then the non-ground count).  The whole-map call must give the "ground",
"groundpatch" and "variance" the oracle's detect_ground_patches gives (NaN payloads canonical, the sign of zero kept), and
the one-cell call, at every planted cell and at the limits of the window, the oracle's detect_ground_patch<S>.  A handle
without the full layers keeps no "m2": it gets the variance m2 / (points + FLT_MIN) imported instead.  Slots 0 and 1
hold sentinel planes that must come back unchanged.

The sizes: N % 4 == 0 runs the TMA-staged kernel, the others the plain-load one; partial 32-column blocks, a last CTA
with 1 .. 3 of its 4 tiles, odd N (the upper section one row short), inner regions that are empty or tiny.
"""
import numpy as np
import pytest

import detect_planes as dp
import ref_scenarios as rs
from groundgrid_b200 import capi
from oracle import Oracle

pytestmark = pytest.mark.gpu

SIZES = [8, 12, 13, 96, 100, 101, 102, 132, 300, 364, 600, 1200, 1600]
STATES = ("fresh", "count", "scan")
SENTINEL_LAYERS = ("points", "ground", "groundpatch", "minGroundHeight", "variance")


def bits(a):
    a = np.ascontiguousarray(a, np.float32)
    u = a.view(np.uint32).copy()
    u[np.isnan(a)] = 0x7FC00000
    return u


def bit_errors(name, got, want, planted):
    bad = bits(got) != bits(want)
    if not bad.any():
        return []
    where = {(i, j): o for i, j, _, o in planted}
    ex = ", ".join(f"{tuple(int(v) for v in ij)} planted {where.get(tuple(int(v) for v in ij), '-')}: gpu={got[tuple(ij)]!r} cpu={want[tuple(ij)]!r}"
                   for ij in np.argwhere(bad)[:3])
    return [f"{name}: {int(bad.sum())} cells differ; e.g. {ex}"]


def imported(c, full):
    """The planes a handle with / without the full layers receives (the oracle gets the same, and always "m2")."""
    p = dict(c.planes)
    if not full:
        p["variance"] = dp.quotient(p["m2"], p["points"])
    return p


def oracle_for(c, planes):
    o = Oracle(c.dim, c.res)
    o.set_config(**c.config)
    o.init_map(0.0, 0.0, 0.0)
    for name in ("groundCandidates", "m2", "variance"):
        o.add_layer(name, 0.0)
    for name, a in planes.items():
        o.set_layer(name, a)
    return o


class Handle:
    """Slot 2 of a 3-slot handle of one geometry; slots 0 and 1 hold sentinel planes."""

    def __init__(self, dim, res, full):
        self.g = capi.GroundGridB200(dim, res, n_slots=3, max_points=8192, full_layers=full)
        self.full = full
        n = self.g.n
        rng = np.random.default_rng(n)
        self.sentinel = {}
        for s in (0, 1):
            self.g.init_map(0.0, 0.0, 0.0, slot=s)
            for name in SENTINEL_LAYERS:
                a = rng.normal(0.0, 1.0, (n, n)).astype(np.float32)
                self.g.set_layer(name, a, slot=s)
                self.sentinel[(s, name)] = a

    def prepare(self, c, state, planes):
        g = self.g
        g.set_config(slot=2, **{k: v for k, v in c.cfg.items()})
        g.init_map(0.0, 0.0, 0.0, slot=2)
        if state != "fresh":
            pts, org = rs.detection_scan(c.n, c.dim)
            if state == "count":
                keep = g.upload_points(pts, slot=2)
                g.run_scans(g.make_descs([2], [len(pts)], [org], [0.0]), stop_after=1)
                del keep
            else:
                g.filter_cloud(pts, org, 0.0, slot=2)
        for name, a in planes.items():
            if name == "m2" and not self.full:
                continue
            g.set_layer(name, a, slot=2)

    def sentinel_errors(self):
        return [f"slot {s} {name} changed" for (s, name), a in self.sentinel.items() if not np.array_equal(bits(self.g.layer(name, slot=s)), bits(a))]


@pytest.mark.parametrize("full", [True, False], ids=["full", "lean"])
@pytest.mark.parametrize("n", SIZES)
def test_detection_on_imported_planes(n, full):
    handles = {}
    fails = []
    for kind, cfg_name in dp.CASES:
        c = dp.make_case(kind, cfg_name, n)
        key = (c.dim, c.res)
        if key not in handles:
            handles[key] = Handle(c.dim, c.res, full)
        h = handles[key]
        assert h.g.n == n
        planes = imported(c, full)
        calls = [(S, i, j) for i, j, S, _ in c.planted] + dp.window_limit_cells(n)
        for state in STATES:
            errs = []
            h.prepare(c, state, planes)
            o = oracle_for(c, planes)
            h.g.detect_ground_patches(slot=2)
            o.detect_ground_patches()
            for name in ("ground", "groundpatch", "variance"):
                errs += bit_errors(f"patches {name}", h.g.layer(name, slot=2), o.layer(name), c.planted)
            h.prepare(c, state, planes)
            o = oracle_for(c, planes)
            for S, i, j in calls:
                h.g.detect_ground_patch(S, i, j, slot=2)
                o.detect_ground_patch(S, i, j)
            for name in ("ground", "groundpatch"):
                errs += bit_errors(f"patch {name}", h.g.layer(name, slot=2), o.layer(name), c.planted)
            if errs:
                fails.append(f"[{kind}/{cfg_name} {state}] " + " | ".join(errs[:3]))
    for h in handles.values():
        fails += h.sentinel_errors()
        h.g.close()
    assert not fails, f"N {n} {'full' if full else 'lean'}: {len(fails)} failing\n" + "\n".join(fails)


@pytest.mark.parametrize("n", rs.DETECT_SIZES)
def test_detect_planes_against_the_reference_itself(n):
    """tests/ref_scenarios.py:detect_planes on the CUDA path: every digest the reference stored."""
    rs.run("detect_planes", lambda dim, res: rs.Cuda(dim, res, 8192), n)

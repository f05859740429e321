"""Every launch layout of the spiral sweep on the device, and imported priors with confidences at the edges of the decay.

The spiral path of a map depends on its size N (tests/test_spiral_layouts.py:LAYOUTS): k_spiral_pipe for small and for
N 1108 .. 1283, k_spiral_skew with M lane threads per side and 1 .. 3 phases in between, the plain k_spiral above.  Each
row runs here at both of its ends (and the rows' neighbours just outside them) on a random prior over the whole map,
bit for bit against the oracle.  The priors of tests/spiral_priors.py (+-inf, NaN, -0, negative, denormal, FLT_MAX and
0.001 confidences on far, near, ring-corner, centre and border cells) run through the fused pipeline of each kind of
path and through the per-phase calls, for the default decrease factor and 1, 100 and 1000.
"""
import numpy as np
import pytest

import spiral_priors as sp
from groundgrid_b200 import capi, synth
from oracle import Oracle
from test_spiral_layouts import layout_of, spiral_plan

pytestmark = pytest.mark.gpu

RES = 0.33
LIVE = ("variance", "minGroundHeight", "ground", "groundpatch")
DEAD = ("m2", "meanVariance", "groundCandidates", "planeDist", "maxGroundHeight", "pointsRaw")
# both ends of every row of LAYOUTS, and the pipe / plain boundary
SIZES = [13, 14, 65, 66, 129, 130, 193, 194, 257, 258, 321, 322, 385, 386, 449, 450, 467, 468, 513, 514, 627, 628, 641, 642,
         787, 788, 947, 948, 1107, 1108, 1283, 1284]


def dim_of(n):
    d = round(n * RES, 4)
    assert capi.host_cells_per_side(d, RES) == n
    return d


def layout_id(n):
    kind, threads, M, phases = layout_of(n)
    return f"{n}-{kind}" + (f"-M{M}-ph{phases}" if kind == "skew" else f"-{threads}")


def diff_report(name, a, b):
    bad = ~((a == b) | (np.isnan(a) & np.isnan(b)))
    if not bad.any():
        return None
    idx = np.argwhere(bad)
    ex = ", ".join(f"{tuple(i)}: gpu={a[tuple(i)]!r} cpu={b[tuple(i)]!r}" for i in idx[:4])
    return f"{name}: {bad.sum()} cells differ; e.g. {ex}"


def layer_errors(g, o, names, slot=0):
    return [r for r in (diff_report(nm, g.layer(nm, slot=slot), o.layer(nm)) for nm in names) if r]


def import_prior(maps, G, C, slot=0):
    for m in maps:
        if isinstance(m, capi.GroundGridB200):
            m.set_layer("ground", G, slot=slot)
            m.set_layer("groundpatch", C, slot=slot)
        else:
            m.set_layer("ground", G)
            m.set_layer("groundpatch", C)


def test_sizes_cover_every_layout_twice():
    from test_spiral_layouts import LAYOUTS

    for lo, hi, *lay in LAYOUTS:
        tested = [n for n in SIZES + [10, 1200, 1600] if lo <= n <= hi]
        assert len(tested) >= 2 or lo == hi, (lo, hi)
        assert (lo in tested or lo == 3) and (hi in tested or hi == LAYOUTS[-1][1]), (lo, hi)
    assert {n % 4 for n in SIZES if n >= 300} == {0, 1, 2, 3}


@pytest.mark.parametrize("n", SIZES, ids=layout_id)
def test_every_layout_on_a_full_prior(n):
    """A random ground / groundpatch (C = uniform^4) over the whole map, imported into the handle and the oracle; a 64-beam
    scan, a roll with yaw, a second scan: labels and every layer bit-identical after each scan."""
    assert spiral_plan(n) == layout_of(n)
    dim = dim_of(n)
    g = capi.GroundGridB200(dim, RES, n_slots=1, max_points=140000, full_layers=True)
    o = Oracle(dim, RES)
    assert g.n == o.n == n
    g.init_map(0.0, 0.0, 0.0)
    o.init_map(0.0, 0.0, 0.0)
    import_prior((g, o), *sp.base_prior(n, seed=n))
    scene = synth.make_scene(seed=n)
    for k in range(2):
        ex, ey, yaw = 0.8 * k, -0.5 * k, 0.3 * k
        pts, org = synth.scan_64(scene, ego_xy=(ex, ey), yaw=yaw, seed=n + k)
        if k:
            T = synth.base_from_map(ex, ey, yaw, base_z=0.0, pitch=0.005)
            assert int(g.update_pose(ex, ey, T)) == o.update(ex, ey, T) == 1
            errs = layer_errors(g, o, ("ground", "groundpatch"))
            assert not errs, f"N {n} after the roll: " + " | ".join(errs)
        labels = g.filter_cloud(pts, org, 0.0)
        want, _, _ = o.filter_cloud(pts, org, 0.0, threads=1)
        assert np.array_equal(labels, want), f"N {n} scan {k}: {(labels != want).sum()} labels differ"
        errs = layer_errors(g, o, ("points",) + LIVE + DEAD)
        assert not errs, f"N {n} scan {k}: " + " | ".join(errs)
    g.close()


@pytest.mark.parametrize("n", [468, 1107], ids=layout_id)
def test_batch_over_two_stream_groups(monkeypatch, n):
    """Four slots over two stream groups, each on its own prior, through gg_run_scans_to_device twice with a batched roll in
    between: the per-slot offsets into the skewed copy and the per-slot shared memory at their largest for the layout."""
    import torch

    monkeypatch.setenv("GG_STREAMS", "2")
    B, dim = 4, dim_of(n)
    g = capi.GroundGridB200(dim, RES, n_slots=B, max_points=140000, full_layers=False)
    assert g.n_streams == 2
    oracles = [Oracle(dim, RES) for _ in range(B)]
    scenes = [synth.make_scene(seed=n + b) for b in range(B)]
    for b in range(B):
        g.init_map(0.1 * b, 0.0, 0.0, slot=b)
        oracles[b].init_map(0.1 * b, 0.0, 0.0)
        import_prior((g, oracles[b]), *sp.base_prior(n, seed=100 * n + b), slot=b)
    slots = np.arange(B, dtype=np.int32)
    for k in range(2):
        pos = [(0.1 * b + 0.9 * k, -0.6 * k) for b in range(B)]
        yaw = 0.25 * k
        if k:
            T = np.stack([synth.base_from_map(x, y, yaw, base_z=0.0, pitch=0.004) for x, y in pos])
            moved = g.update_pose_batch(slots, np.array(pos), T)
            for b in range(B):
                assert int(moved[b]) == oracles[b].update(pos[b][0], pos[b][1], T[b]) == 1
        scans = [synth.scan_64(scenes[b], ego_xy=pos[b], yaw=yaw, seed=10 * n + b + k) for b in range(B)]
        dev = [torch.from_numpy(np.ascontiguousarray(p).view(np.float32).reshape(-1, 8).copy()).cuda() for p, _ in scans]
        out = g.run_scans_to_device(dev, slots, [o_ for _, o_ in scans], 0.0, labels=True, select=None)
        torch.cuda.synchronize()
        for b in range(B):
            want, _, _ = oracles[b].filter_cloud(scans[b][0], scans[b][1], 0.0, threads=1)
            got = out.labels[b].cpu().numpy()
            assert np.array_equal(got, want), f"N {n} slot {b} scan {k}: {(got != want).sum()} labels differ"
            errs = layer_errors(g, oracles[b], ("ground", "groundpatch"), slot=b)
            assert not errs, f"N {n} slot {b} scan {k}: " + " | ".join(errs)
    g.close()


EDGE_SIZES = [10, 101, 300, 468, 1200, 1600]   # pipe, skew (one phase, odd and even), skew (two phases), pipe 1024, plain


def _edge_scan(n):
    scene = synth.make_scene(seed=7, n_boxes=6, rmin=1.0, rmax=min(30.0, 0.4 * n * RES))
    return synth.lidar_scan(scene, beams=16, az_steps=256, seed=n)


def _planted_errors(g, o, planted):
    Cg, Co = g.layer("groundpatch"), o.layer("groundpatch")
    return [f"groundpatch at the {kind} cell {(x, y)} planted {v!r}: gpu={Cg[x, y]!r} cpu={Co[x, y]!r}"
            for (x, y), kind, v in planted if not np.array_equal(Cg[x, y], Co[x, y], equal_nan=True)]


@pytest.mark.parametrize("factor", [None, 1.0, 100.0, 1000.0], ids=lambda f: "default" if f is None else f"factor{f:g}")
@pytest.mark.parametrize("n", EDGE_SIZES, ids=layout_id)
def test_edge_confidences_through_the_pipeline_and_the_phase_calls(n, factor):
    """Each case of spiral_priors.edge_cases imported into a fresh map, then (a) a scan through the fused pipeline,
    (b) gg_spiral_ground_interpolation alone, (c) gg_interpolate_cell at every planted cell: labels, ground and
    groundpatch against the oracle (NaN-aware), and groundpatch explicitly at every planted cell."""
    dim = dim_of(n)
    cfg = {} if factor is None else {"occupied_cells_decrease_factor": factor}
    pts, org = _edge_scan(n)
    g = capi.GroundGridB200(dim, RES, n_slots=1, max_points=max(len(pts), 1024), full_layers=False)
    if cfg:
        g.set_config(**cfg)
    fails = []
    for seed, (name, planted) in enumerate(sp.edge_cases(n, RES).items()):
        G, C = sp.planted_prior(n, RES, planted, seed=seed)
        for how in ("pipeline", "spiral", "interpolate_cell"):
            o = Oracle(dim, RES)
            if cfg:
                o.set_config(**cfg)
            g.init_map(0.0, 0.0, 0.0)
            o.init_map(0.0, 0.0, 0.0)
            import_prior((g, o), G, C)
            errs = []
            if how == "pipeline":
                labels = g.filter_cloud(pts, org, 0.1)
                want, _, _ = o.filter_cloud(pts, org, 0.1, threads=1)
                if not np.array_equal(labels, want):
                    errs.append(f"{(labels != want).sum()} labels differ")
            elif how == "spiral":
                g.spiral_ground_interpolation(0.1)
                o.spiral(0.1)
            else:
                for (x, y), _, _ in planted:
                    if 1 <= x < n - 1 and 1 <= y < n - 1:
                        g.interpolate_cell(x, y)
                        o.interpolate_cell(x, y)
            errs += layer_errors(g, o, ("ground", "groundpatch")) + _planted_errors(g, o, planted)
            if errs:
                fails.append(f"[{name} / {how}] " + " | ".join(errs[:3]))
    g.close()
    assert not fails, f"N {n} factor {factor or 'default'}: {len(fails)} failing cases\n" + "\n".join(fails)


def test_nonfinite_confidence_against_the_reference_itself():
    """tests/ref_scenarios.py:nonfinite_confidence on the CUDA path (N = 100, skewed layout): every digest the reference
    stored, its NaNs included."""
    import ref_scenarios as rs

    rs.run("nonfinite_confidence", lambda dim, res: rs.Cuda(dim, res, 4096))

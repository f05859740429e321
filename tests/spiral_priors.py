"""Imported priors for the spiral sweep with confidences at the edges of the decay's domain.

The spiral's far-cell decay is std::max(c - c / decrease_factor, 0.001) in fp64 (interpolate_cell :463-464): +-inf and
NaN decay to NaN, -0, negative values and denormals land on the 0.001 floor, FLT_MAX stays finite.  Scans alone never
leave such values in `groundpatch`; gg_set_layer / gg_set_layers_from_device (slot migration) can.  Each case plants
values at cells of every kind the sweep treats differently:
  far     visited once, beyond minDistSquared: the visit stores the decay
  corner  a ring corner, visited twice and beyond minDistSquared: the decay of the decay
  near    visited, inside minDistSquared: keeps its confidence
  border  never visited, only read as a neighbour: keeps its confidence
  centre  the spiral's start: set to 1 before the sweep
One non-finite confidence makes most of the terrain the sweep computes after it NaN, so each non-finite value gets its
own case on cells near the outer rings; the finite edge values share one dense case.
"""
import numpy as np

from groundgrid_b200 import capi

f32 = np.float32
FLT_MAX = f32(np.finfo(np.float32).max)
FLOOR = f32(0.001)
FINITE_EDGES = (f32(-0.0), f32(0.0), f32(-0.5), -FLT_MAX, f32(np.finfo(np.float32).smallest_subnormal), FLT_MAX, FLOOR,
                np.nextafter(FLOOR, f32(0.0)), np.nextafter(FLOOR, f32(1.0)), f32(1.0))
NONFINITE = {"+inf": f32(np.inf), "-inf": f32(-np.inf), "nan": f32(np.nan)}
KINDS = ("far", "corner", "near", "border", "centre")
# occupied_cells_decrease_factor: the ends of GroundGrid.cfg's range (1, 100) and the default (5) take the floor shortcut
# of decay_confidence (CfgConst::decay_floor_ok = 1); 1000 does not
FACTORS = (1.0, 5.0, 100.0, 1000.0)


def is_far(n, res, x, y):
    """interpolate_cell's distance test (:463) for cells (x, y) of an n x n map."""
    c = f32(n // 2 - 1)
    fx = (np.asarray(x, np.float32) - c).astype(np.float64)
    fy = (np.asarray(y, np.float32) - c).astype(np.float64)
    return (fx * fx + fy * fy) * np.float64(f32(res)) ** 2 > 12.0


def cell_kinds(n, res):
    """Cells of each kind, the outermost first (by ring around the centre); far / corner / near come from the schedule.
    A map of less than 3.5 m has no far cell."""
    _, vs = capi.host_spiral_schedule(n)
    cnt = np.zeros((n, n), np.int32)
    np.add.at(cnt, (vs[:, 0], vs[:, 1]), 1)
    c = n // 2 - 1
    ii, jj = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    ring = np.maximum(np.abs(ii - c), np.abs(jj - c))
    far = is_far(n, res, ii, jj)
    read = np.zeros((n, n), bool)
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            read[vs[:, 0] + dx, vs[:, 1] + dy] = True
    masks = {"far": (cnt == 1) & far, "corner": (cnt == 2) & far, "near": (cnt >= 1) & ~far,
             "border": read & (cnt == 0) & (ring > 1)}
    out = {}
    for k, m in masks.items():
        x, y = np.nonzero(m)
        order = np.lexsort((y, x, -ring[x, y]))
        out[k] = [(int(a), int(b)) for a, b in zip(x[order], y[order])]
    out["centre"] = [(c, c)]
    return out


def base_prior(n, seed):
    """Random terrain and uniform^4 confidences, so that every visit does real arithmetic."""
    rng = np.random.default_rng(seed)
    return rng.uniform(-1, 1, (n, n)).astype(np.float32), (rng.uniform(0, 1, (n, n)) ** 4).astype(np.float32)


def edge_cases(n, res):
    """name -> [((x, y), kind, confidence)].  Non-finite values one per case, on an outer-ring cell of each kind (the near one
    as far out as minDistSquared allows); the dense case holds every finite edge value on cells of every kind."""
    kinds = cell_kinds(n, res)
    cases = {}
    for vname, v in NONFINITE.items():
        for kind in KINDS:
            if not kinds[kind]:
                continue
            cases[f"{vname}@{kind}"] = [(kinds[kind][2 if kind in ("far", "border") else 0], kind, v)]
    dense = []
    for kind in KINDS:
        cells = kinds[kind]
        step = max(1, len(cells) // (3 * len(FINITE_EDGES)))
        for i, v in enumerate(FINITE_EDGES * 3):
            if i * step < len(cells) and cells[i * step] not in {c for c, _, _ in dense}:
                dense.append((cells[i * step], kind, v))
    cases["dense finite"] = dense
    return cases


def planted_prior(n, res, planted, seed):
    G, C = base_prior(n, seed)
    for (x, y), _, v in planted:
        C[x, y] = v
    return G, C


def expected_confidence(kind, v, decay):
    """What the sweep leaves at a planted cell of a kind: decay(c), decay(decay(c)), c, or 1 at the centre."""
    return {"centre": f32(1.0), "corner": decay(decay(v)), "far": decay(v)}.get(kind, v)

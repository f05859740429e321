"""CPU-side checks of the product library: it loads, exports every symbol the header declares,
refuses to compute without a GPU, and its host-side logic (expectedPoints table, map-move
arithmetic, spiral wavefront schedule) agrees with the oracle."""
import os
import re

import numpy as np
import pytest

import spiral_priors as sp
from groundgrid_b200 import capi
from oracle import Oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
FLT_MIN = f32(np.finfo(np.float32).tiny)


def header_symbols():
    text = open(os.path.join(ROOT, "include", "groundgrid_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(gg_[a-z_0-9]+)\s*\(", text)))


def test_library_loads_and_exports_every_declared_symbol():
    lib = capi.load()
    names = header_symbols()
    assert len(names) >= 25
    for name in names:
        assert hasattr(lib, name), f"{name} declared in include/groundgrid_b200.h but not exported"


def test_struct_layouts_match_the_header():
    import ctypes as C

    assert C.sizeof(capi.Config) == 8 + 11 * 8 + 8        # 2 ints, 11 doubles, int + padding
    assert C.sizeof(capi.ScanDesc) == 40
    assert capi.POINT_DTYPE.itemsize == 32
    cfg = capi.Config()
    capi.load().gg_default_config(C.byref(cfg))
    assert (cfg.point_count_cell_variance_threshold, cfg.max_ring, cfg.thread_count) == (10, 1024, 8)
    assert (cfg.distance_factor, cfg.minimum_distance_factor, cfg.patch_size_change_distance) == (0.0001, 0.0005, 20.0)
    assert (cfg.occupied_cells_decrease_factor, cfg.occupied_cells_point_count_factor) == (5.0, 20.0)
    assert cfg.min_outlier_detection_ground_confidence == 1.25 and cfg.outlier_tolerance == 0.1


def test_no_cpu_fallback():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is for machines without one")
    with pytest.raises(capi.GroundGridError) as e:
        capi.GroundGridB200(99.0, 0.33)
    assert e.value.code == -2 and "no CPU fallback" in str(e.value)


@pytest.mark.parametrize("dim,res,n", [(120.0, 0.33, 364), (99.0, 0.33, 300), (120.0, 0.2, 600), (33.0, 0.33, 100)])
def test_expected_points_table_matches_oracle(dim, res, n):
    assert capi.host_cells_per_side(dim, res) == n
    E = capi.host_expected_points(dim, res)
    assert np.array_equal(E, Oracle(dim, res).expected_points())


def test_move_map_matches_oracle():
    rng = np.random.default_rng(9)
    res = float(np.float32(0.33))
    o = Oracle(33.0, 0.33)
    o.init_map(1.5, -2.5, 0.0)
    pos = o.position().copy()
    T = np.eye(4)[:3]
    for _ in range(200):
        target = pos + rng.uniform(-3, 3, 2) * res * rng.choice([0.1, 1.0, 5.0])
        moved, new_pos, shift = capi.host_move_map(res, pos, target)
        A = (np.arange(o.n)[:, None] * o.n + np.arange(o.n)[None, :]).astype(np.float32)
        o.set_layer("ground", A)
        assert o.update(target[0], target[1], T) == int(moved)
        assert np.array_equal(o.position(), new_pos)
        if moved:
            # oracle content shift must equal the reported index shift: new(r,c) = old(r+si, c+sj)
            Gn = o.layer("ground")
            r = np.arange(o.n)[:, None] + shift[0]
            c = np.arange(o.n)[None, :] + shift[1]
            ok = (r >= 0) & (r < o.n) & (c >= 0) & (c < o.n)
            want = (r * o.n + c).astype(np.float32)
            assert np.array_equal(Gn[ok], want[ok])
            assert np.all(o.layer("groundpatch")[~ok] == 0.0)
        pos = new_pos


def decay_confidence(c, factor=5.0):
    """gg_internal.h:decay_confidence (the decay k_skew / k_detect store for the skewed and the pipelined spiral) for
    occupied_cells_decrease_factor = factor, elementwise on the host."""
    import ctypes as C

    L = capi.load()
    L.gg_host_decay_confidence.restype = C.c_int
    L.gg_host_decay_confidence.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    cfg = capi.default_config()
    cfg.occupied_cells_decrease_factor = factor
    c = np.ascontiguousarray(c, np.float32)
    out = np.empty_like(c)
    assert L.gg_host_decay_confidence(C.byref(cfg), c.ctypes.data, c.size, out.ctypes.data) == 0
    return out


def skew_visit_confidence(d, occ):
    """The confidence a visit of k_spiral_skew leaves, from its SD entry d (the decay, or the near-cell sentinel)."""
    import ctypes as C

    L = capi.load()
    L.gg_host_skew_visit_confidence.restype = C.c_int
    L.gg_host_skew_visit_confidence.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    d, occ = np.ascontiguousarray(d, np.float32), np.ascontiguousarray(occ, np.float32)
    out = np.empty_like(d)
    assert L.gg_host_skew_visit_confidence(d.ctypes.data, occ.ctypes.data, d.size, out.ctypes.data) == 0
    return out


def _tree9(v):
    return ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + (v[7] + v[8])))


def run_level_schedule(G, C, base_z, level_start, visits, res_f, dec_factor=5.0):
    """Executes the spiral as the GPU does: level by level, all visits of a level read first, then write."""
    n = G.shape[0]
    c = n // 2 - 1
    G = G.copy()
    C = C.copy()
    C[c, c] = 1.0
    G[c, c] = f32(base_z)
    res2 = np.float64(f32(res_f)) ** 2
    for lvl in range(len(level_start) - 1):
        vs = visits[level_start[lvl]:level_start[lvl + 1]]
        x, y = vs[:, 0], vs[:, 1]
        cc = [C[x - 1 + k % 3, y - 1 + k // 3] for k in range(9)]
        gg = [G[x - 1 + k % 3, y - 1 + k // 3] for k in range(9)]
        s = _tree9(cc) + FLT_MIN
        avg = _tree9([a * b for a, b in zip(cc, gg)]) / s
        occ = cc[4]
        G[x, y] = (f32(1.0) - occ) * avg + occ * gg[4]
        fx = (x.astype(np.float32) - f32(c)).astype(np.float64)
        fy = (y.astype(np.float32) - f32(c)).astype(np.float64)
        far = (fx * fx + fy * fy) * res2 > 12.0
        o64 = occ.astype(np.float64)
        dec = o64 - o64 / np.float64(dec_factor)
        with np.errstate(invalid="ignore"):
            dec = np.where(dec < 0.001, 0.001, dec).astype(np.float32)   # std::max(dec, 0.001): NaN stays NaN
        C[x[far], y[far]] = dec[far]
    return G, C


@pytest.mark.parametrize("dim,res,levels", [(33.0, 0.33, None), (99.0, 0.33, 743), (120.0, 0.33, 903)])
def test_spiral_wavefront_schedule_is_exact(dim, res, levels):
    o = Oracle(dim, res)
    n = o.n
    ls, vs = capi.host_spiral_schedule(n)
    c = n // 2 - 1
    assert len(vs) == sum(4 * 2 * (c - p) + 2 for p in range(1, c))       # SURVEY App. C visit count
    if levels is not None:
        assert len(ls) - 1 == levels                                       # SURVEY App. C DAG depth
    # no two visits of a level may touch each other's 3x3 neighbourhood writes
    for lvl in range(0, len(ls) - 1, max(1, (len(ls) - 1) // 40)):
        v = vs[ls[lvl]:ls[lvl + 1]]
        cells = v[:, 0] * n + v[:, 1]
        assert len(np.unique(cells)) == len(cells)
        written = set(cells.tolist())
        for (x, y) in v:
            for dx in (-1, 0, 1):
                for dy in (-1, 0, 1):
                    if dx or dy:
                        assert (x + dx) * n + (y + dy) not in written
    rng = np.random.default_rng(21)
    o.init_map(0.0, 0.0, 0.0)
    G = rng.uniform(-1, 1, (n, n)).astype(np.float32)
    C = (rng.uniform(0, 1, (n, n)) ** 4).astype(np.float32)
    o.set_layer("ground", G)
    o.set_layer("groundpatch", C)
    o.spiral(0.3)
    Gs, Cs = run_level_schedule(G, C, 0.3, ls, vs, res)
    assert np.array_equal(o.layer("ground"), Gs)
    assert np.array_equal(o.layer("groundpatch"), Cs)


def host_spiral_records(n, res, dist):
    import ctypes as C

    L = capi.load()
    L.gg_host_spiral_records.restype = C.c_int
    L.gg_host_spiral_records.argtypes = [C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    ls, vs = capi.host_spiral_schedule(n)
    recs = np.zeros(4 * len(vs), np.uint32)
    mr = C.c_int(0)
    ok = L.gg_host_spiral_records(n, np.float32(res), dist, recs.ctypes.data_as(C.c_void_p), recs.size, C.byref(mr))
    return ok, mr.value, ls, recs.reshape(-1, 4)


@pytest.mark.parametrize("dist", [1, 2, 3])
@pytest.mark.parametrize("dim,res", [(33.0, 0.33), (99.0, 0.33)])
def test_pipelined_spiral_records_emulation(dim, res, dist):
    """Emulates k_spiral_pipe on the CPU: neighbourhoods are snapshotted `dist` levels before the
    visit, the entries named by the record come from the exchange ring instead, the decay comes
    from the table.  Must reproduce the oracle's sequential sweep bit for bit."""
    o = Oracle(dim, res)
    n = o.n
    rng = np.random.default_rng(4)
    o.init_map(0.0, 0.0, 0.0)
    G = rng.uniform(-1, 1, (n, n)).astype(np.float32)
    C = (rng.uniform(0, 1, (n, n)) ** 4).astype(np.float32)
    o.set_layer("ground", G)
    o.set_layer("groundpatch", C)
    o.spiral(0.3)
    G, C = emulate_pipe(n, res, dist, G, C, 0.3)
    assert np.array_equal(o.layer("ground"), G)
    assert np.array_equal(o.layer("groundpatch"), C)


def emulate_pipe(n, res, dist, G, C, base_z, factor=5.0):
    """k_detect's decay table (D1, and D2 for the second visit of a ring corner) -> k_spiral_pipe with `dist` levels of
    prefetch, on the CPU; returns the sweep's (ground, groundpatch)."""
    ok, max_recent, ls, recs = host_spiral_records(n, res, dist)
    assert ok == 1 and max_recent <= 4
    L = len(ls) - 1
    c = n // 2 - 1
    G, C = G.copy(), C.copy()
    D1 = decay_confidence(C, factor)
    D2 = decay_confidence(D1, factor)
    C[c, c] = 1.0
    G[c, c] = f32(base_z)
    ring = {}       # level -> (newg, newc) arrays by slot
    snaps = {}      # level -> (cc[9], gg[9]) snapshot taken dist levels ahead

    def snapshot(lvl):
        r = recs[ls[lvl]:ls[lvl + 1]]
        x, y = (r[:, 0] & 0xFFFF).astype(np.int64), (r[:, 0] >> 16).astype(np.int64)
        snaps[lvl] = ([C[x - 1 + q % 3, y - 1 + q // 3].copy() for q in range(9)], [G[x - 1 + q % 3, y - 1 + q // 3].copy() for q in range(9)])

    for lvl in range(min(dist, L)):
        snapshot(lvl)                      # prologue: before level 0 runs
    for lvl in range(L):
        if lvl + dist < L:
            snapshot(lvl + dist)           # prefetch issued at the top of level lvl
        r = recs[ls[lvl]:ls[lvl + 1]]
        x, y = (r[:, 0] & 0xFFFF).astype(np.int64), (r[:, 0] >> 16).astype(np.int64)
        cc, gg = snaps.pop(lvl)
        ents = np.stack([r[:, 1] & 0xFFFF, r[:, 1] >> 16, r[:, 2] & 0xFFFF, r[:, 2] >> 16], axis=1)
        for e in ents.T:
            back = (e >> 14).astype(np.int64)
            q = ((e >> 10) & 15).astype(np.int64)
            slot = (e & 1023).astype(np.int64)
            for b in (1, 2, 3):
                m = back == b
                if not m.any():
                    continue
                assert b <= dist
                src_g, src_c = ring[lvl - b]
                for qq in range(9):
                    mm = m & (q == qq)
                    gg[qq][mm] = src_g[slot[mm]]
                    cc[qq][mm] = src_c[slot[mm]]
        s = _tree9(cc) + FLT_MIN
        avg = _tree9([a * b for a, b in zip(cc, gg)]) / s
        occ = cc[4]
        newg = (f32(1.0) - occ) * avg + occ * gg[4]
        far = (r[:, 3] & 1).astype(bool)
        second = (r[:, 3] & 2).astype(bool)
        newc = np.where(far, np.where(second, D2[x, y], D1[x, y]), occ).astype(np.float32)
        ring[lvl] = (newg.copy(), newc.copy())
        ring.pop(lvl - dist - 1, None)
        G[x, y] = newg
        C[x[far], y[far]] = newc[far]
    return G, C


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 16383, 16384, 16385, 40001])
def test_host_cloud_packing(n):
    """gg_filter_cloud_batch repacks PointXYZIR records as x | y | z | ring before the H2D copy."""
    import ctypes as C

    from groundgrid_b200 import synth

    rng = np.random.default_rng(n)
    pts = np.zeros(n, synth.POINT_DTYPE)
    pts.view(np.uint8)[:] = 0xCD          # junk in the padding bytes of the records
    for c in "xyz":
        pts[c] = rng.standard_normal(n).astype(np.float32)
    pts["intensity"] = 7.0
    pts["ring"] = rng.integers(0, 65536, n)
    n_pad = (n + 7) & ~7
    raw = np.full(14 * n_pad + 64, 0xAB, np.uint8)
    off = (-raw.ctypes.data) % 32
    dst = raw[off:off + 14 * n_pad]
    L = capi.load()
    L.gg_host_pack_cloud.restype = C.c_int
    L.gg_host_pack_cloud.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    assert L.gg_host_pack_cloud(pts.ctypes.data_as(C.c_void_p), n, dst.ctypes.data_as(C.c_void_p)) == 0
    f = dst[:12 * n_pad].view(np.float32)
    assert np.array_equal(f[:n], pts["x"]) and np.array_equal(f[n_pad:n_pad + n], pts["y"]) and np.array_equal(f[2 * n_pad:2 * n_pad + n], pts["z"])
    assert np.array_equal(dst[12 * n_pad:].view(np.uint16)[:n], pts["ring"])
    assert np.all(f[n:n_pad] == 0) and np.all(dst[12 * n_pad:].view(np.uint16)[n:] == 0)
    assert np.all(raw[off + 14 * n_pad:] == 0xAB)


def host_spiral_skew(n):
    import ctypes as C

    L = capi.load()
    fn = L.gg_host_spiral_skew
    fn.restype = C.c_int
    fn.argtypes = [C.c_int] + [C.c_void_p] * 7 + [C.c_int]
    hdr = np.zeros(10, np.int32)
    fn(n, hdr.ctypes.data, None, None, None, None, None, None, 0)
    if not hdr[0]:
        return None
    K, KP, rows, levels, row0, lanes, n_irr = (int(v) for v in hdr[1:8])
    pattern = np.zeros(36, np.int32)
    lb, le = np.zeros(lanes, np.int32), np.zeros(lanes, np.int32)
    home = np.zeros(n * n * 4, np.int32)
    ils = np.zeros(levels + 1, np.int32)
    recs = np.zeros(n_irr * 16, np.uint32)
    assert fn(n, hdr.ctypes.data, pattern.ctypes.data, lb.ctypes.data, le.ctypes.data, home.ctypes.data, ils.ctypes.data, recs.ctypes.data, recs.size) == 1
    return dict(K=K, KP=KP, rows=rows, levels=levels, row0=row0, lanes=lanes, pattern=pattern.reshape(4, 9), lane_begin=lb, lane_end=le,
                home=home.reshape(n * n, 4), irr_level_start=ils, irr=recs.reshape(-1, 16))


@pytest.mark.parametrize("dim,res", [(13.2, 0.33), (33.0, 0.33), (99.0, 0.33), (120.0, 0.33), (120.0, 0.2),
                                     (33.33, 0.33), (30.5, 0.5), (81.2, 0.4)])   # the last three: odd cell counts (101, 61, 203)
def test_skewed_spiral_tables_emulation(dim, res):
    """CPU emulation of k_skew -> k_spiral_skew -> k_unskew: lane threads follow the fixed offset
    pattern in (level, ring) space, the irregular warp follows explicit records, neighbourhoods are
    read one level ahead, values written one level ago arrive through the per-lane exchange buffer.
    Must equal the oracle's sequential sweep bit for bit."""
    o = Oracle(dim, res)
    n = o.n
    rng = np.random.default_rng(17)
    o.init_map(0.0, 0.0, 0.0)
    G = rng.uniform(-1, 1, (n, n)).astype(np.float32)
    C = (rng.uniform(0, 1, (n, n)) ** 4).astype(np.float32)
    o.set_layer("ground", G)
    o.set_layer("groundpatch", C)
    o.spiral(0.3)
    G, C = emulate_skew(n, res, G, C, 0.3)
    assert np.array_equal(o.layer("ground"), G)
    assert np.array_equal(o.layer("groundpatch"), C)


def emulate_skew(n, res, G, C, base_z, factor=5.0, t=None, lanes_at=None):
    """k_skew (the skewed copy and its SD table, fused into k_detect) -> k_spiral_skew -> k_unskew on the CPU; returns
    the sweep's (ground, groundpatch).  lanes_at(level): the lanes whose regular visit of that level runs (default: the
    lanes whose [lane_begin, lane_end) holds it), e.g. from a replay of the lane threads."""
    t = host_spiral_skew(n) if t is None else t
    assert t is not None
    KP, rows, row0, lanes, L = t["KP"], t["rows"], t["row0"], t["lanes"], t["levels"]
    prev_q = [1, 3, 7, 5]

    # ---- k_skew (column-major cell index = i + j * n)
    c = n // 2 - 1
    Gf, Cf = G.reshape(-1, order="F").copy(), C.reshape(-1, order="F").copy()
    Gf[c + c * n] = f32(base_z)
    Cf[c + c * n] = 1.0
    D1 = decay_confidence(Cf, factor)
    D2 = decay_confidence(D1, factor)
    ii, jj = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    fx = (ii.astype(np.float32) - f32(c)).astype(np.float64)
    fy = (jj.astype(np.float32) - f32(c)).astype(np.float64)
    far = ((fx * fx + fy * fy) * np.float64(f32(res)) ** 2 > 12.0).reshape(-1, order="F")
    nslots = 4 * rows * KP
    SKg, SKc, SD = np.zeros(nslots, np.float32), np.zeros(nslots, np.float32), np.full(nslots, -1.0, np.float32)
    home = t["home"]
    for h in range(4):
        m = home[:, h] >= 0
        SKg[home[m, h]] = Gf[m]
        SKc[home[m, h]] = Cf[m]
        if h < 2:
            SD[home[m, h]] = np.where(far[m], (D1 if h == 0 else D2)[m], f32(-1.0))
    # ---- k_spiral_skew
    lane = np.arange(lanes)
    side, kcol = lane // KP, lane % KP
    xg, xc = np.zeros((2, lanes), np.float32), np.zeros((2, lanes), np.float32)
    irr, ils = t["irr"], t["irr_level_start"]

    def reg_lanes(lvl):
        if lanes_at is not None:
            return np.asarray(lanes_at(lvl), np.int64)
        return lane[(t["lane_begin"] <= lvl) & (lvl < t["lane_end"])]

    def fetch(lvl):  # what the prefetch of level `lvl` sees
        rl = reg_lanes(lvl)
        own = (side[rl] * rows + lvl + row0) * KP + kcol[rl]
        idx = own[:, None] + t["pattern"][side[rl]]
        r = irr[ils[lvl]:ils[lvl + 1]]
        iidx = r[:, 1:10].astype(np.int64)
        return (rl, own, SKg[idx].copy(), SKc[idx].copy(), SD[own].copy(), r, SKg[iidx].copy(), SKc[iidx].copy(), SD[r[:, 0].astype(np.int64)].copy())

    def tree(v):
        return ((v[:, 0] + v[:, 1]) + (v[:, 2] + v[:, 3])) + ((v[:, 4] + v[:, 5]) + (v[:, 6] + (v[:, 7] + v[:, 8])))

    def visit(gg, cc, dd):
        s = tree(cc) + FLT_MIN
        avg = tree(cc * gg) / s
        occ = cc[:, 4]
        newg = (f32(1.0) - occ) * avg + occ * gg[:, 4]
        return newg.astype(np.float32), skew_visit_confidence(dd, occ)

    nxt = fetch(0)
    for lvl in range(L):
        cur = nxt
        if lvl + 1 < L:
            nxt = fetch(lvl + 1)       # issued before this level's stores
        rl, own, gg, cc, dd, r, igg, icc, idd = cur
        pb = (lvl - 1) & 1
        # regular lanes: the previous cell of the lane comes from the exchange buffer
        if len(rl) and lvl > 0:
            pq = np.array(prev_q)[side[rl]]
            gg[np.arange(len(rl)), pq] = xg[pb, rl]
            cc[np.arange(len(rl)), pq] = xc[pb, rl]
        ng, nc = visit(gg, cc, dd)
        # irregular visits: recents name (neighbour, producer lane)
        for w in (10, 11):
            for sh in (0, 16):
                e = (r[:, w] >> sh) & 0xFFFF
                m = e != 0xFFFF
                q = np.where(m, e >> 12, 0).astype(np.int64)
                pl = (e & 4095).astype(np.int64)
                igg[m, q[m]] = xg[pb, pl[m]]
                icc[m, q[m]] = xc[pb, pl[m]]
        ing, inc = visit(igg, icc, idd)
        # stores
        SKg[own], SKc[own] = ng, nc
        xg[lvl & 1, rl], xc[lvl & 1, rl] = ng, nc
        io = r[:, 0].astype(np.int64)
        SKg[io], SKc[io] = ing, inc
        mir = r[:, 12].astype(np.int32)
        mm = mir >= 0
        SKg[mir[mm]], SKc[mir[mm]] = ing[mm], inc[mm]
        il = r[:, 13].astype(np.int64)
        xg[lvl & 1, il], xc[lvl & 1, il] = ing, inc
    # ---- k_unskew
    m = home[:, 0] >= 0
    Gf[m], Cf[m] = SKg[home[m, 0]], SKc[home[m, 0]]
    return Gf.reshape(n, n, order="F"), Cf.reshape(n, n, order="F")


def reference_decay(c, factor):
    """interpolate_cell :464 as the reference writes it: std::max(c - c / F, 0.001) in double, std::max(a, b) = a < b ? b : a
    (so a NaN difference stays NaN), stored as float."""
    o = np.float64(c)
    with np.errstate(invalid="ignore"):
        d = o - o / np.float64(factor)
        return f32(0.001) if d < 0.001 else f32(d)


def test_decay_confidence_at_the_edges_of_its_domain():
    """The decay every spiral path stores for a far cell, against the reference's expression, on both sides of the
    floor shortcut (decay_floor_ok = 1 for factors 1 .. 100, 0 for 1000)."""
    vals = np.array(list(sp.FINITE_EDGES) + list(sp.NONFINITE.values()) + [f32(-1.0), f32(1e-30), f32(2e-3), f32(1e30)], np.float32)
    for factor in sp.FACTORS:
        consts = capi.host_config_constants(_config(occupied_cells_decrease_factor=factor))
        assert consts["decay_floor_ok"] == (0 if factor == 1000.0 else 1), factor
        got = decay_confidence(vals, factor)
        want = np.array([reference_decay(v, factor) for v in vals], np.float32)
        assert np.array_equal(got, want, equal_nan=True), (factor, got, want)
    assert np.isnan(decay_confidence(np.array([np.inf, -np.inf, np.nan], np.float32), 5.0)).all()
    # the skewed layout's table: a decay (>= 0.001 or NaN) is stored; only the near-cell sentinel keeps the cell's value
    d = np.array([np.nan, 0.001, 7.0, -1.0], np.float32)
    occ = np.array([np.inf, -np.inf, 0.5, np.inf], np.float32)
    assert np.array_equal(skew_visit_confidence(d, occ), np.array([np.nan, 0.001, 7.0, np.inf], np.float32), equal_nan=True)


def _config(**kw):
    cfg = capi.default_config()
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _nan_equal_report(name, a, b):
    bad = ~((a == b) | (np.isnan(a) & np.isnan(b)))
    if not bad.any():
        return None
    idx = np.argwhere(bad)
    return f"{name}: {bad.sum()} cells differ, e.g. " + ", ".join(f"{tuple(i)}: emulated={a[tuple(i)]!r} oracle={b[tuple(i)]!r}" for i in idx[:4])


EDGE_PATHS = ("plain", "pipe", "skew")


@pytest.mark.parametrize("factor", sp.FACTORS)
@pytest.mark.parametrize("path", EDGE_PATHS)
@pytest.mark.parametrize("dim,res", [(33.0, 0.33), (33.33, 0.33)])   # N = 100, 101
def test_spiral_emulations_on_edge_confidences(dim, res, path, factor):
    """Imported priors with +-inf, NaN, -0, negative, denormal, FLT_MAX and 0.001 (and its neighbours) confidences on far,
    near, ring-corner, centre and border cells (tests/spiral_priors.py), through the plain level schedule, the pipelined
    records (two levels ahead) and the skewed tables with their decay tables: NaN-aware equal to the oracle's sweep, and
    at every planted cell the value the reference's decay gives."""
    n = Oracle(dim, res).n
    ls, vs = capi.host_spiral_schedule(n)
    t = host_spiral_skew(n) if path == "skew" else None
    fails = []
    for seed, (name, planted) in enumerate(sp.edge_cases(n, res).items()):
        G, C = sp.planted_prior(n, res, planted, seed=seed)
        o = Oracle(dim, res)
        o.set_config(occupied_cells_decrease_factor=factor)
        o.init_map(0.0, 0.0, 0.0)
        o.set_layer("ground", G)
        o.set_layer("groundpatch", C)
        o.spiral(0.3)
        with np.errstate(invalid="ignore", over="ignore"):   # inf - inf, FLT_MAX sums: the arithmetic under test
            if path == "plain":
                Ge, Ce = run_level_schedule(G, C, 0.3, ls, vs, res, dec_factor=factor)
            elif path == "pipe":
                Ge, Ce = emulate_pipe(n, res, 2, G, C, 0.3, factor)
            else:
                Ge, Ce = emulate_skew(n, res, G, C, 0.3, factor, t=t)
        Go, Co = o.layer("ground"), o.layer("groundpatch")
        errs = [r for r in (_nan_equal_report("ground", Ge, Go), _nan_equal_report("groundpatch", Ce, Co)) if r]
        for (x, y), kind, v in planted:
            want = sp.expected_confidence(kind, v, lambda c: reference_decay(c, factor))
            for who, got in (("oracle", Co[x, y]), ("emulation", Ce[x, y])):
                if not np.array_equal(got, want, equal_nan=True):
                    errs.append(f"{who} groundpatch at {kind} cell {(x, y)} planted {v!r}: {got!r}, the reference's decay gives {want!r}")
        if errs:
            fails.append(f"[{name}] " + " | ".join(errs[:4]))
    assert not fails, f"{path}, N {n}, factor {factor}: " + "\n".join(fails)


# Parent-build values: the choice gg_create made before it moved into plan_spiral (skew tables, records, and the
# smallest time-shared M, replayed from the gg_host_spiral_skew / gg_host_spiral_records exports).
@pytest.mark.parametrize("n,kind,threads,M,phases", [(10, "pipe", 512, 0, 0), (16, "skew", 192, 32, 1), (100, "skew", 320, 64, 1),
                                                    (300, "skew", 704, 160, 1), (364, "skew", 832, 192, 1), (600, "skew", 576, 128, 3),
                                                    (1200, "pipe", 1024, 0, 0), (1600, "plain", 512, 0, 0)])
def test_spiral_plan_picks_the_path_of_each_map_size(n, kind, threads, M, phases):
    """gg_host_spiral_plan: the skewed layout while one CTA holds it (one lane thread per lane, time-shared rings from
    N ~ 500), the pipelined kernel where the skew tables do not fit (small maps, N = 1200), the plain wavefront where a
    level has more than 1024 visits."""
    import ctypes as C

    fn = capi.load().gg_host_spiral_plan
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_float, C.c_void_p]
    out = np.zeros(4, np.int32)
    assert fn(n, 0.33, out.ctypes.data) == 0
    assert (["plain", "pipe", "skew"][out[0]], int(out[1]), int(out[2]), int(out[3])) == (kind, threads, M, phases)


@pytest.mark.parametrize("threads,n_jobs,n_points,ring,rounds,lag", [(4, 40, 20000, 8, 4, 3), (3, 17, 50001, 4, 3, 1),
                                                                     (6, 64, 3000, 5, 6, 4), (2, 9, 100, 2, 3, 0),
                                                                     (8, 96, 16385, 32, 5, 6)])
def test_packer_pool_ring_claims_and_cancel(threads, n_jobs, n_points, ring, rounds, lag):
    """The worker pool of gg_filter_cloud_batch without CUDA: ragged clouds through a small staging ring whose slots
    are released `lag` jobs late, jobs taken away from the back (raw path), a cancelled batch, several rounds."""
    import ctypes as C

    L = capi.load()
    f = L.gg_host_packer_selftest
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_size_t, C.c_int, C.c_int, C.c_int]
    for _ in range(3):
        assert f(threads, n_jobs, n_points, ring, rounds, lag) == 0


def test_bench_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (no GPU involved): one JSON line with impl = reference, the metric / unit of the GPU arm, a
    cpu_baseline describing the run and an e2e object repeating the value; it runs the reference's own sources (oracle/_ref)
    whenever that library is available."""
    import json
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1", "--pool", "2"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "Mpoints/s" and d["higher_is_better"] is True and d["value"] > 0
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["cpu_baseline"]["value"] == d["value"] and d["cpu_baseline"]["cores"] >= 1
    from oracle import ref as refmod

    assert d["cpu_baseline"]["kind"] == ("reference" if refmod.available() else "port")

"""The launch layouts of the spiral sweep (gg_host.cpp:plan_spiral) and the lane threads of k_spiral_skew, on the CPU.

plan_spiral picks, per map size N, a kernel (pipe, skew, plain) and for the skewed layout the lane threads per side M
and the number of phases (rings a lane thread walks one after the other).  LAYOUTS pins that choice for every N from 3
to 1699 (a sweep of gg_host_spiral_plan at resolution 0.33; the layout depends on N only); tests/test_gpu_spiral_layouts.py
runs every row on the device.  The replay below follows skew_lane_thread (gg_kernels.cu) thread by thread: the phase
switch, the per-warp level window, the one-level-ahead register loads, and composes the visits it makes with the lane
emulation of test_host_logic.py.
"""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi
from oracle import Oracle
from test_host_logic import emulate_skew, host_spiral_skew

# (first N, last N, kind, CTA threads, M, phases); rows cover 3 .. 1699 without a gap
LAYOUTS = [
    (3, 13, "pipe", 512, 0, 0),
    (14, 65, "skew", 192, 32, 1),
    (66, 129, "skew", 320, 64, 1),
    (130, 193, "skew", 448, 96, 1),
    (194, 257, "skew", 576, 128, 1),
    (258, 321, "skew", 704, 160, 1),
    (322, 385, "skew", 832, 192, 1),
    (386, 449, "skew", 960, 224, 1),
    (450, 467, "skew", 448, 96, 3),
    (468, 513, "skew", 576, 128, 2),
    (514, 627, "skew", 576, 128, 3),
    (628, 641, "skew", 704, 160, 2),
    (642, 787, "skew", 704, 160, 3),
    (788, 947, "skew", 832, 192, 3),
    (948, 1107, "skew", 960, 224, 3),
    (1108, 1283, "pipe", 1024, 0, 0),
    (1284, 1699, "plain", 512, 0, 0),
]
PF_FAR, PF_NEAR = 8, 2     # prefetch distances of skew_lane_thread


def layout_of(n):
    for lo, hi, *lay in LAYOUTS:
        if lo <= n <= hi:
            return tuple(lay)
    raise KeyError(n)


def spiral_plan(n, res=0.33):
    fn = capi.load().gg_host_spiral_plan
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_float, C.c_void_p]
    out = np.zeros(4, np.int32)
    assert fn(n, res, out.ctypes.data) == 0
    return (["plain", "pipe", "skew"][out[0]], int(out[1]), int(out[2]), int(out[3]))


def test_layout_table_is_contiguous():
    assert LAYOUTS[0][0] == 3 and all(a[1] + 1 == b[0] for a, b in zip(LAYOUTS, LAYOUTS[1:]))
    assert len({tuple(r[2:]) for r in LAYOUTS}) == len(LAYOUTS)   # no layout appears in two rows


@pytest.mark.parametrize("lo,hi,kind,threads,M,phases", LAYOUTS)
def test_spiral_plan_of_each_layout_row(lo, hi, kind, threads, M, phases):
    """Both ends of a row and the sizes just outside them (the neighbouring rows' layouts), and the row's midpoint."""
    for n in sorted({lo, hi, (lo + hi) // 2}):
        assert spiral_plan(n) == (kind, threads, M, phases), n
    for n in (lo - 1, hi + 1):
        if 3 <= n <= LAYOUTS[-1][1]:
            assert spiral_plan(n) == layout_of(n) != (kind, threads, M, phases), n
    if kind == "skew":
        t = host_spiral_skew(lo)
        assert M % 32 == 0 and phases == -(-t["KP"] // M) and threads == 4 * M + 64


def test_spiral_plan_does_not_depend_on_the_resolution():
    for n in (14, 449, 450, 641, 1107, 1108, 1284):
        assert {spiral_plan(n, res) for res in (0.1, 0.2, 0.33, 0.5)} == {layout_of(n)}, n


def replay_lane_threads(n):
    """skew_lane_thread for every thread (side, m) of the layout plan_spiral picks for N, vectorised over the threads.
    Returns (lanes visited per level, the number of (thread, level) visits).  Asserts on the way:
      - a visit runs on the registers loaded for its level (the one-level-ahead load; a phase's first level included),
      - no iteration a warp skips (outside its [w_first, w_last) window) holds a visit, load or prefetch of a thread,
      - a phase's first level is loaded by the thread after it switched to that phase (the kGap margin of plan_spiral)."""
    kind, _, M, phases = spiral_plan(n)
    assert kind == "skew"
    t = host_spiral_skew(n)
    KP, L = t["KP"], t["levels"]
    # the [phase][side][m] tables plan_spiral builds for the kernel
    PB = np.zeros((phases, 4, M), np.int64)
    PE = np.zeros((phases, 4, M), np.int64)
    for ph in range(phases):
        for sd in range(4):
            cols = ph * M + np.arange(M)
            ok = cols < KP
            PB[ph, sd, ok] = t["lane_begin"][sd * KP + cols[ok]]
            PE[ph, sd, ok] = t["lane_end"][sd * KP + cols[ok]]
    T = 4 * M
    side, m = np.arange(T) // M, np.arange(T) % M
    ph = np.zeros(T, np.int64)
    lb, le = PB[0, side, m].copy(), PE[0, side, m].copy()
    BIG = np.iinfo(np.int64).max

    def window():
        f = np.where(lb < le, lb - PF_FAR, BIG).reshape(-1, 32).min(axis=1)
        last = np.where(lb < le, le, -1).reshape(-1, 32).max(axis=1)
        return np.repeat(np.maximum(f, 0) & ~1, 32), np.repeat(last, 32)

    w_first, w_last = window()
    reg = {0: np.full(T, -1), 1: np.full(T, -1)}      # register sets A, B: the level each holds
    reg[0][(lb == 0) & (le > 0)] = 0
    switched_at = {}                                   # (thread, phase) -> loop level of the switch
    loaded = set()
    visits = {}
    n_visits = 0
    for l in range(0, L, 2):
        if phases > 1:
            moved = np.zeros(T, bool)
            while True:
                go = (ph + 1 < phases) & (l >= le)
                if not go.any():
                    break
                ph[go] += 1
                lb[go], le[go] = PB[ph[go], side[go], m[go]], PE[ph[go], side[go], m[go]]
                moved |= go
                for i in np.nonzero(go)[0]:
                    switched_at[(int(i), int(ph[i]))] = l
            wm = np.repeat(moved.reshape(-1, 32).any(axis=1), 32)
            if wm.any():
                nf, nl = window()
                w_first[wm], w_last[wm] = nf[wm], nl[wm]
        skip = (l < w_first) | (l >= w_last)
        for ll, cur, nxt in ((l, 0, 1), (l + 1, 1, 0)):
            if ll >= L:
                break
            busy = np.zeros(T, bool)
            for d in (PF_FAR, PF_NEAR, 1, 0):
                busy |= (ll + d >= lb) & (ll + d < le)
            bad = np.nonzero(skip & busy)[0]
            assert not len(bad), f"N {n}: thread {bad[0]} has work at level {ll} outside its warp's window"
            act = ~skip
            ld = act & (ll + 1 >= lb) & (ll + 1 < le)
            vis = act & (ll >= lb) & (ll < le)
            stale = np.nonzero(vis & (reg[cur] != ll))[0]
            assert not len(stale), f"N {n}: thread {stale[0]} visits level {ll} on registers of level {reg[cur][stale[0]]}"
            reg[nxt][ld] = ll + 1
            loaded.update(zip(np.nonzero(ld)[0].tolist(), [ll + 1] * int(ld.sum())))
            i = np.nonzero(vis)[0]
            col = ph[i] * M + m[i]
            assert np.all(col < KP)
            visits[ll] = np.sort(side[i] * KP + col)
            n_visits += len(i)
    # every later phase's first level: the thread switched to it before the level ahead of it, and loaded it then
    for p in range(1, phases):
        for i in range(T):
            b, e = PB[p, side[i], m[i]], PE[p, side[i], m[i]]
            if b < e:
                assert switched_at[(i, p)] <= b - 1 and (i, int(b)) in loaded, (n, i, p, b)
    return visits, n_visits, t


SKEW_SIZES = [40, 100, 160, 230, 300, 364, 449, 450, 467, 468, 513, 600, 628, 641, 700, 800, 948, 1107]


def test_replay_sizes_cover_every_skew_layout():
    assert {layout_of(n) for n in SKEW_SIZES} == {tuple(r[2:]) for r in LAYOUTS if r[2] == "skew"}


@pytest.mark.parametrize("n", SKEW_SIZES)
def test_lane_threads_run_every_regular_visit_once(n):
    """Every regular visit of every lane runs exactly once, on thread (side, col mod M) in phase col / M, at its level;
    composed with the lane emulation, the sweep equals the oracle's bit for bit."""
    visits, n_visits, t = replay_lane_threads(n)
    lane = np.arange(t["lanes"])
    total = 0
    for lvl in range(t["levels"]):
        want = lane[(t["lane_begin"] <= lvl) & (lvl < t["lane_end"])]
        assert np.array_equal(visits.get(lvl, np.zeros(0, np.int64)), want), f"N {n}: level {lvl}"
        total += len(want)
    assert n_visits == total == int((t["lane_end"] - t["lane_begin"]).sum())
    res = 0.33
    dim = n * res
    o = Oracle(dim, res)
    assert o.n == n
    rng = np.random.default_rng(n)
    G = rng.uniform(-1, 1, (n, n)).astype(np.float32)
    Cc = (rng.uniform(0, 1, (n, n)) ** 4).astype(np.float32)
    o.init_map(0.0, 0.0, 0.0)
    o.set_layer("ground", G)
    o.set_layer("groundpatch", Cc)
    o.spiral(0.3)
    Ge, Ce = emulate_skew(n, res, G, Cc, 0.3, t=t, lanes_at=lambda lvl: visits.get(lvl, np.zeros(0, np.int64)))
    assert np.array_equal(o.layer("ground"), Ge)
    assert np.array_equal(o.layer("groundpatch"), Ce)

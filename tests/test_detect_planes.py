"""The generators of tests/detect_planes.py hit what they claim, checked with pyref's one-cell restatement of
detect_ground_patch<S> (:343-395, the sequential minCoeff fold) on the variance detect_ground_patches computes first.

Every planted cell must take the branch it was built for, and every case of a map of at least 100 cells per side must
have planted cells of both window sizes in all five outcomes.  The boundary cells must sit exactly on their boundary,
and the ring cells exactly on patch_size_change_distance.
"""
import math

import numpy as np
import pytest

import detect_planes as dp
import pyref

SIZES = [12, 100, 101, 102, 300, 364]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind,cfg_name", dp.CASES, ids=[f"{k}-{c}" for k, c in dp.CASES])
def test_planted_cells_take_their_branch(n, kind, cfg_name):
    c = dp.make_case(kind, cfg_name, n)
    assert dp.cells_per_side(c.dim, c.res) == n
    for name in dp.PLANES:
        assert c.planes[name].shape == (n, n) and c.planes[name].dtype == np.float32
    wrong, reached = [], set()
    for i, j, S, want in c.planted:
        assert c.inner(i, j) and S == c.size(i, j)
        got, g, cc = dp.outcome(c, i, j, S)
        if want is not None and got != want:
            wrong.append(f"({i}, {j}) S={S}: {got}, planted for {want}")
        if want is not None:
            reached.add((S, got))
    assert not wrong, f"{kind}/{cfg_name} N {n}: " + "; ".join(wrong[:6])
    if n >= 100:
        missing = [(S, o) for S in (3, 5) for o in dp.OUTCOMES if (S, o) not in reached]
        assert not missing, f"{kind}/{cfg_name} N {n}: no planted cell for {missing}"


def test_window_minimum_is_the_sequential_fold():
    """A NaN heading a later column of the window does not hide the minimum further down it; one at element 0 is the
    minimum (what the reference's minCoeff returns)."""
    c = dp.make_case("nonfinite", "default", 100)
    (i1, j1, S1, o1), (i0, j0, S0, o0) = [p for p in c.planted if p[3] is not None][10:12]
    M = c.planes["minGroundHeight"]
    assert np.isnan(M[c.window(i1, j1, S1)[S1]]) and not np.isnan(M[c.window(i1, j1, S1)[0]])
    got, g, _ = dp.outcome(c, i1, j1, S1)
    assert (got, g) == ("localmin", c.planes["ground"][i1, j1] - np.float32(1.0))
    assert np.isnan(M[c.window(i0, j0, S0)[0]])
    assert dp.outcome(c, i0, j0, S0)[0] == "unchanged"


@pytest.mark.parametrize("n", [100, 101, 364])
@pytest.mark.parametrize("cfg_name", ["default", "low", "high"])
def test_boundary_cells_sit_on_their_boundary(n, cfg_name):
    c = dp.make_case("boundaries", cfg_name, n)
    var = dp.quotient(c.planes["m2"], c.planes["points"])
    P = c.planes["points"]
    sums = {}
    for i, j, S, _ in c.planted:
        h = S // 2
        sums[(i, j)] = pyref.tree_sum(pyref.block(P, i - h, j - h, S))
    special = c.planted[10:]
    need_eq, need_below = special[0], special[1]
    assert pyref.f64(sums[need_eq[:2]]) == c.need(*need_eq[:3])
    assert pyref.f64(sums[need_below[:2]]) == c.need(*need_below[:3]) - 1
    T = c.cfg["point_count_cell_variance_threshold"]
    assert P[special[2][:2]] == T and P[special[3][:2]] == T - 1
    og, gl = dp._equal_after_tol(c.cfg["outlier_tolerance"])
    assert pyref.f64(gl) == pyref.f64(og) + c.cfg["outlier_tolerance"]
    for i, j, S, _ in special[4:10]:
        assert c.planes["ground"][i, j] == og and c.planes["minGroundHeight"][i, j] in (gl, np.nextafter(gl, np.float32(np.inf)),
                                                                                       np.nextafter(gl, np.float32(-np.inf)))
    below, above = special[10], special[11]
    for (i, j, S, _), sign in ((below, -1), (above, 1)):
        q = var[i, j]
        assert np.sign(pyref.f64(q) * pyref.f64(q) - pyref.f64(c.vt(i, j))) == sign
        assert np.sign(pyref.f64(np.nextafter(q, np.float32(-sign * np.inf))) ** 2 - pyref.f64(c.vt(i, j))) != sign
    assert [var[p[:2]] for p in special[12:15]] == [0.0, 0.0, dp.DENORM]
    assert math.copysign(1.0, var[special[13][:2]]) == -1.0


@pytest.mark.parametrize("n", [100, 364, 1600])
def test_cap_cells_straddle_a_bound_above_two_to_the_24(n):
    c = dp.make_case("cap", "cap", n)
    cap = [(i, j, S, o) for i, j, S, o in c.planted[10:]]
    assert {o for *_, o in cap} == {"need", "localmin"}
    for i, j, S, o in cap:
        need = c.need(i, j, S)
        assert need > 2.0 ** 24 and (c.planes["points"][i, j] < need) == (o == "need")
        assert float(np.float32(c.planes["points"][i, j])) != need or o == "localmin"


@pytest.mark.parametrize("n", [100, 101, 300, 364])
@pytest.mark.parametrize("kind", ["ring", "ring+", "ring-"])
def test_ring_cells_sit_on_the_patch_size_switch(n, kind):
    c = dp.make_case(kind, "default", n)
    psc = c.cfg["patch_size_change_distance"]
    ring = [p for p in c.planted if p[3] in ("need", "localmin") and p[3] == ("need" if p[2] == 3 else "localmin")]
    t, exact = dp._ring_distance(c)
    on = []
    for i, j, S, _ in c.planted:
        di, dj = pyref.f64(i) - pyref.f64(n) / 2.0, pyref.f64(j) - pyref.f64(n) / 2.0
        if pyref.f64(pyref.f32((di * di + dj * dj) * (pyref.f64(c.res_f) ** 2))) == t:
            on.append((i, j, S))
    assert len(on) >= 2 and ring
    assert exact * exact == t
    assert {S for _, _, S in on} == ({5} if kind == "ring-" else {3})
    assert psc == {"ring": exact, "ring+": math.nextafter(exact, math.inf), "ring-": math.nextafter(exact, -math.inf)}[kind]

"""The adversarial families of tests/neighbour_reference.py land where they claim, the CPU oracle agrees with float64
distances outside a few-ulp band on all of them, and numpy restatements with one planted mistake each are caught by
their family.  No GPU needed: these pin the inputs that tests/test_gpu_neighbour_geometry.py runs on the device."""
import numpy as np
import pytest

import neighbour_reference as NR
from oracle import oracle as O

F32 = np.float32
N = 16384


@pytest.fixture(scope="module")
def shell():
    return NR.shell(N, 2)


@pytest.fixture(scope="module")
def caps():
    return NR.caps(N, 5)


def test_dist2_binding_is_the_fma_order():
    a = np.array([[0.1, 0.2, 0.3]], F32)
    b = np.array([[0.7, -0.4, 1.9]], F32)
    dx, dy, dz = (a - b)[0].astype(np.float64)
    want = F32(dz * dz + float(F32(dx * dx + float(F32(dy * dy)))))   # each fma rounds once; products exact in float64
    assert O.dist2(a, b)[0] == want


def test_shell_points_sit_on_the_fp32_radius(shell):
    cloud, centres, placements = shell
    levels = {}
    for k, ci, r, level, axes in placements:
        d = O.dist2(centres[ci], cloud[k])
        r2 = F32(r) * F32(r)
        assert np.sign(d - r2) == level, (k, r, level)
        levels.setdefault(level, set()).add(axes)
        if level == 0:
            assert d == r2
    assert levels[0] == {1, 2, 3} and levels[-1] >= {1, 2, 3} and levels[1] >= {1, 2, 3}
    for r in NR.ALL_RADII:                                     # every radius has an exact d2 == r2 pair
        assert any(p[2] == r and p[3] == 0 for p in placements), r


def test_lidar_scene_is_dense_where_the_grid_caps_bite():
    xyz = NR.lidar(N, 1)
    assert np.isfinite(xyz).all() and len(np.unique(xyz, axis=0)) > N - 10
    cent = xyz[O.fps(xyz[None], 4096)[0]]
    d = ((cent[:, None, :].astype(np.float64) - xyz[None]) ** 2).sum(-1)
    cnt = (d < 0.25).sum(1)
    assert (cnt > 128).sum() > 50, "SA1 centres with more than BQ_CAP candidates at r = 0.5"
    assert ((cnt > 0) & (cnt <= 32)).sum() > 100 and ((cnt > 32) & (cnt <= 128)).sum() > 100
    ground = np.abs(xyz[:, 1] - F32(1.7)) < 0.01
    assert ground.mean() > 0.3, "a ground plane"
    assert (xyz[:, 2] >= 40).sum() > 0 and (xyz[:, 2] < 40).sum() > N // 2


def test_caps_clusters_hit_every_dispatch_boundary(caps):
    cloud, centres, sizes = caps
    r0, rmax = 0.1, 0.5
    h = NR.bq_cell(rmax)
    for c, size in zip(centres, sizes):
        d = O.dist2(np.broadcast_to(c, cloud.shape), cloud)
        if size > 0:
            assert (d < F32(r0) * F32(r0)).sum() == size and (d < F32(rmax) * F32(rmax)).sum() == size
        else:
            cells = np.floor(cloud.astype(np.float64) / h).astype(np.int64)
            block = np.all(np.abs(cells - np.floor(c.astype(np.float64) / h)) <= 1, axis=1)
            assert block.sum() > 512 and (d < F32(rmax) * F32(rmax)).sum() == 0, "list walk overflow, no hit"
    assert {32, 33, 128, 129, 16, 17}.issubset(sizes)


def test_cell_edge_centres_sit_on_cell_boundaries():
    cloud, centres = NR.cell_edge(N, 3)
    h = NR.bq_cell(0.5)
    q = centres.astype(np.float64) / h
    off = np.abs(centres.astype(np.float64) - np.round(q) * h)
    assert (off <= 1.5 * np.spacing(np.abs(centres))).all(), "every centre coordinate is k*h to within an ulp"
    below = np.floor(q) != np.round(q)
    assert below.any() and (~below).any(), "centres on both sides of a boundary"


def test_nn_cell_edge_probes_straddle_the_certification_radius():
    unknown, known, npk = NR.nn_cell_edge(N, 4096, 4)
    h = NR.nn_cell(known)
    cert = F32(F32(F32(h) * F32(0.9999)) ** 2)
    d2, idx = O.three_nn(unknown[None, :npk], known[None])
    third = d2[0, :, 2]
    assert (third < cert).any() and (third == cert).any() and (third > cert).any()


def test_ties_family_has_ties_at_the_fps_argmax():
    xyz = NR.ties(4096, 6)
    idx, nties = NR.fps_replay(xyz, 256)
    assert np.array_equal(idx, O.fps(xyz[None], 256)[0])
    assert (nties > 1).sum() > 100, "most rounds pick among exact ties"
    sph = NR.sphere_around_zero(4097, 7)
    idx, nties = NR.fps_replay(sph, 8)
    assert nties[1] > 1000 and np.array_equal(idx, O.fps(sph[None], 8)[0])


@pytest.mark.parametrize("family", ["lidar", "shell", "cell_edge", "caps", "ties", "far3e4", "far1e6", "flat", "collinear",
                                    "nonfinite"])
def test_oracle_ball_query_agrees_with_float64_outside_the_band(family):
    xyz, centres = scene(family, 4096)
    for r, ns in ((0.1, 16), (0.5, 32), (2.0, 32)):
        idx = O.ball_query(r, ns, xyz[None], centres[None])[0]
        assert NR.ball_query_f64_violations(xyz, centres, r, ns, idx) == 0, (family, r)


@pytest.mark.parametrize("family", ["lidar", "ties", "far3e4", "flat", "collinear", "nn_cell_edge"])
def test_oracle_three_nn_agrees_with_float64_outside_the_band(family):
    if family == "nn_cell_edge":
        unknown, known, _ = NR.nn_cell_edge(4096, 1024, 4)
    else:
        unknown, _ = scene(family, 4096)
        known = np.ascontiguousarray(unknown[::4])
    d2, idx = O.three_nn(unknown[None], known[None])
    assert NR.three_nn_f64_violations(unknown, known, idx[0]) == 0


def scene(family, n, seed=0):
    """(cloud (n, 3), centres (k, 3)) of one family: its own centres first, then FPS picks"""
    own = None
    if family == "lidar":
        xyz = NR.lidar(n, 11 + seed)
    elif family == "shell":
        xyz, own, _ = NR.shell(n, 2 + seed)
    elif family == "cell_edge":
        xyz, own = NR.cell_edge(n, 3 + seed)
    elif family == "caps":
        xyz, own, _ = NR.caps(n, 5 + seed)
    elif family == "ties":
        xyz = NR.ties(n, 6 + seed)
    elif family == "far3e4":
        xyz = NR.far(n, 7 + seed, 3e4)
    elif family == "far1e6":
        xyz = NR.far(n, 8 + seed, 1e6)
    elif family == "flat":
        xyz = NR.flat(n, 9 + seed)
    elif family == "collinear":
        xyz = NR.collinear(n, 10 + seed)
    elif family == "nonfinite":
        xyz = NR.nonfinite(n, 12 + seed)
    else:
        raise ValueError(family)
    picks = xyz[O.fps(xyz[None], 256)[0]]
    centres = picks if own is None else np.concatenate([own, picks])
    return xyz, np.ascontiguousarray(centres[:256])


# ------------------------------------------------------------------------------------------------ mutants
def _disagree(a, b):
    return int(np.any(a != b, axis=-1).sum())


def test_mutant_non_strict_radius_is_caught_by_the_shell(shell):
    cloud, centres, _ = shell
    caught = 0
    for ci, r in enumerate(NR.ALL_RADII):
        want = O.ball_query(r, 16, cloud[None], centres[None, ci:ci + 1])[0]
        assert _disagree(NR.ball_query_np(cloud, centres[ci:ci + 1], r, 16), want) == 0
        caught += _disagree(NR.ball_query_np(cloud, centres[ci:ci + 1], r, 16, strict=False), want)
    assert caught == len(NR.ALL_RADII), "every radius's centre selects its d2 == r2 points under <="


def test_mutant_unfused_distance_is_caught_by_the_shell():
    cloud, centres, placements = NR.shell(N, 2, n2=24, n3=24)
    caught = 0
    for ci, r in enumerate(NR.ALL_RADII):
        want = O.ball_query(r, 64, cloud[None], centres[None, ci:ci + 1])[0]
        caught += _disagree(NR.ball_query_np(cloud, centres[ci:ci + 1], r, 64, fused=False), want)
    assert caught >= 3, caught


def test_mutant_larger_rank_wins_ties_is_caught_by_the_ties():
    xyz = NR.ties(4096, 6)
    want = O.fps(xyz[None], 256)[0]
    got, _ = NR.fps_replay(xyz, 256, larger_rank_wins=True)
    assert (got != want).sum() > 0


def test_cell_edge_margin_is_not_load_bearing_for_fp32_inputs():
    """The grid's 1.0001 cell margin and the 3-NN's 0.9999 certification factor guard against rounding, but with fp32
    coordinates and the FMA distance no placement needs them: every hit has |fl(dx)| < r on each axis (fl(dx*dx) alone
    already reaches fl(r*r) otherwise, and the other terms only add), so a cell edge of exactly r still holds it in the
    3x3x3 block; and a point outside the 3-NN block has fl(d2) >= fl(fl(h)^2), so certifying at h accepts nothing
    wrong.  The families that sit on those boundaries show it: the margin-free restatements agree with the oracle."""
    cloud, centres = NR.cell_edge(N, 3)
    for r in (0.5,):
        want = O.ball_query(r, 32, cloud[None], centres[None])[0]
        assert _disagree(NR.ball_query_grid_np(cloud, centres, r, 32, float(F32(r))), want) == 0
        assert _disagree(NR.ball_query_grid_np(cloud, centres, r, 32, NR.bq_cell(r)), want) == 0
    unknown, known, npk = NR.nn_cell_edge(2048, 1024, 4)
    d_o, i_o = O.three_nn(unknown[None], known[None])
    for cert in (0.9999, 1.0):
        d, i, ok = NR.three_nn_grid_np(unknown, known, cert=cert)
        assert np.array_equal(i, i_o[0]) and np.array_equal(d, d_o[0])
        assert ok.any() and (~ok).any()

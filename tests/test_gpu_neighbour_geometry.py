"""FPS, ball query and 3-NN on the device, bit for bit against the CPU oracle, on the adversarial families of
tests/neighbour_reference.py at the batch-16 shapes of the network: every scene batch mixes one scene of each family
with ray-cast LiDAR scenes.  Every kernel path a prb_option selects is compared with the same oracle result, computed
once per module."""
import numpy as np
import pytest
import torch

import neighbour_reference as NR
from oracle import oracle as O

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import _cabi, config  # noqa: E402
from pointrcnn_b200.ext import pointnet2_cuda  # noqa: E402
from pointrcnn_b200.pointnet2 import pointnet2_utils as pu  # noqa: E402

B = 16
FAMILIES = ("shell", "cell_edge", "caps", "ties", "far3e4", "far1e6", "flat", "collinear", "nonfinite")


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _family(kind, n, radii, seed):
    """(cloud (n, 3), own centres (k, 3) or None)"""
    if kind == "shell":
        xyz, own, _ = NR.shell(n, seed, radii=tuple(sorted(set(radii))), n2=2, n3=2)
        return xyz, own
    if kind == "cell_edge":
        return NR.cell_edge(n, seed, rmax=max(radii), radii=radii)
    if kind == "caps":
        xyz, own, _ = NR.caps(n, seed, radii=radii)
        return xyz, own
    if kind == "ties":
        return NR.ties(n, seed), None
    if kind == "far3e4":
        return NR.far(n, seed, 3e4), None
    if kind == "far1e6":
        return NR.far(n, seed, 1e6), None
    if kind == "flat":
        return NR.flat(n, seed), None
    if kind == "collinear":
        return NR.collinear(n, seed), None
    if kind == "nonfinite":
        xyz = NR.nonfinite(n, seed)
        own = xyz[:8].copy()
        own[1, 0], own[2, 1], own[3] = np.nan, np.inf, -np.inf      # non-finite centres too
        return xyz, own
    return NR.lidar(n, seed), None


def batch(n, m, radii, seed, families=FAMILIES):
    """(xyz (B, n, 3), centres (B, m, 3)): one scene per family, LiDAR scenes for the rest; a scene's own centres first,
    then its leading points"""
    xyz, cen = [], []
    if n < 4096:                                              # the cap clusters and cell-edge rings need room
        families = [f for f in families if f not in ("caps", "cell_edge")]
    kinds = list(families) + ["lidar"] * (B - len(families))
    for s, kind in enumerate(kinds):
        x, own = _family(kind, n, radii, seed + 17 * s)
        c = x[:m] if own is None else np.concatenate([own, x[: m - len(own)]])
        xyz.append(x)
        cen.append(c[:m])
    return np.ascontiguousarray(np.stack(xyz)), np.ascontiguousarray(np.stack(cen))


def pooled(n, m, seed):
    """RCNN SA input: per scene a box's worth of a LiDAR scan, duplicate-padded to n points as roipool3d pads"""
    rng = np.random.default_rng(seed)
    xyz = []
    for s in range(B):
        if s == 0:
            x = NR.ties(n, seed) * np.float32(0.1)
        elif s == 1:
            x, _, _ = NR.shell(n, seed, radii=NR.RCNN_RADII, n2=2, n3=2)
        else:
            scan = NR.lidar_scan(seed + s)
            c = scan[rng.integers(len(scan))]
            inside = np.where(np.all(np.abs(scan - c) < np.array([2.0, 1.5, 3.0]), axis=1))[0][:n]
            k = np.arange(n) % len(inside)
            x = scan[inside][k]
        xyz.append(x)
    xyz = np.ascontiguousarray(np.stack(xyz), dtype=np.float32)
    return xyz, np.ascontiguousarray(xyz[:, :m])


# ------------------------------------------------------------------------------------------------ ball query
BQ_SHAPES = {                     # level: (n, m, radii, nsamples)
    "sa1": (16384, 4096, (0.1, 0.5), (16, 32)),
    "sa2": (4096, 1024, (0.5, 1.0), (16, 32)),
    "sa3": (1024, 256, (1.0, 2.0), (16, 32)),
    "sa4": (256, 64, (2.0, 4.0), (16, 32)),
}


@pytest.fixture(scope="module")
def bq_cases():
    out = {}
    for level, (n, m, radii, nss) in BQ_SHAPES.items():
        xyz, cen = batch(n, m, radii, 100 + n)
        want = [O.ball_query(r, ns, xyz, cen) for r, ns in zip(radii, nss)]
        out[level] = (xyz, cen, radii, nss, want)
    for m, r in ((128, 0.2), (32, 0.4)):
        xyz, cen = pooled(512, m, 7 + m)
        out["rcnn%d" % m] = (xyz, cen, (r,), (NR.RCNN_NSAMPLE,), [O.ball_query(r, NR.RCNN_NSAMPLE, xyz, cen)])
    return out


def _bq(x, c, radii, nss):
    if len(radii) == 2:
        return list(pu.ball_query_msg2(radii, nss, x, c))
    return [pu.ball_query(radii[0], nss[0], x, c)]


@pytest.mark.parametrize("level", list(BQ_SHAPES) + ["rcnn128", "rcnn32"])
@pytest.mark.parametrize("path", ["grid", "grid_csr", "brute_msg2", "brute_single"])
def test_ball_query_bits_on_adversarial_families(cuda, bq_cases, level, path):
    xyz, cen, radii, nss, want = bq_cases[level]
    x, c = T(xyz, cuda), T(cen, cuda)
    old = pu.GRID_MIN_POINTS_BQ
    pu.GRID_MIN_POINTS_BQ = 1 if path.startswith("grid") else old
    try:
        with _cabi.options(grid_csr=int(path == "grid_csr")), config.override(disable_grid=path.startswith("brute")):
            if path == "brute_single":
                got = [pu.ball_query(r, ns, x, c) for r, ns in zip(radii, nss)]
            else:
                got = _bq(x, c, radii, nss)
    finally:
        pu.GRID_MIN_POINTS_BQ = old
    for g, w, r in zip(got, want, radii):
        g = g.cpu().numpy()
        bad = np.where(np.any(g != w, axis=2))
        assert bad[0].size == 0, "r=%g: %d centres differ, first (scene, centre) %s" % (r, bad[0].size, list(zip(*bad))[:4])


def test_ball_query_batch_equals_per_scene(cuda, bq_cases):
    """overflow-list entries and workspace offsets are per scene: the batch answer is each scene's own answer"""
    xyz, cen, radii, nss, _ = bq_cases["sa1"]
    x, c = T(xyz, cuda), T(cen, cuda)
    for csr in (0, 1):
        with _cabi.options(grid_csr=csr):
            full = _bq(x, c, radii, nss)
            for s in (0, 2, 5, 8, 15):                        # shell, caps, far1e6, nonfinite, lidar
                one = _bq(x[s:s + 1].contiguous(), c[s:s + 1].contiguous(), radii, nss)
                for a, b in zip(full, one):
                    assert torch.equal(a[s:s + 1], b), (csr, s)


# ------------------------------------------------------------------------------------------------ three_nn
NN_SHAPES = ((16384, 4096), (4096, 1024), (1024, 256), (256, 64))


@pytest.fixture(scope="module")
def nn_cases():
    out = {}
    for n, m in NN_SHAPES:
        xyz, _ = batch(n, 1, (0.5, 1.0), 300 + n, families=("ties", "far3e4", "far1e6", "flat", "collinear", "nonfinite"))
        unknown = xyz.copy()
        known = np.ascontiguousarray(xyz[:, :: n // m][:, :m])
        if m >= 512:                                          # certification pockets and cell-boundary queries
            for s, seed in ((6, 1), (7, 2)):
                unknown[s], known[s], _ = NR.nn_cell_edge(n, m, seed)
        d2, idx = O.three_nn(unknown, known)
        out[(n, m)] = (unknown, known, d2, idx)
    return out


NN_MODES = {"plain": {}, "sorted_queries": {"nn_sort_queries": 1}, "walk": {"nn_walk": 1}, "csr": {"grid_csr": 1},
            "cell_0.5": {"nn_cell": 0.5}, "cell_4.0": {"nn_cell": 4.0}, "brute": None}


@pytest.mark.parametrize("n,m", NN_SHAPES)
@pytest.mark.parametrize("mode", list(NN_MODES))
def test_three_nn_bits_on_adversarial_families(cuda, nn_cases, n, m, mode):
    unknown, known, d2, idx = nn_cases[(n, m)]
    opts = NN_MODES[mode]
    with _cabi.options(**(opts or {})), config.override(disable_grid=opts is None):
        got_d2, got_idx, w = pu.three_nn_weights(T(unknown, cuda), T(known, cuda))
    gi = got_idx.cpu().numpy()
    bad = np.where(np.any(gi != idx, axis=2))
    assert bad[0].size == 0, "%d queries differ, first %s" % (bad[0].size, list(zip(*bad))[:4])
    assert np.array_equal(got_d2.cpu().numpy(), d2, equal_nan=True)
    np.testing.assert_allclose(w.cpu().numpy(), O.interp_weights(d2), rtol=2e-6, atol=1e-7, equal_nan=True)


@pytest.mark.parametrize("mode", ["plain", "csr"])
def test_three_nn_grid_query_at_infinity_lists_point_zero(cuda, mode):
    """every distance from a query at infinity is inf (or NaN), so the reference's cascade, started at 1e40, takes none of
    them and answers indices (0, 0, 0) at distance inf.  The grid sends such a query to its exhaustive kernel, which
    used to fill its empty slots through the index tie-break (inf == inf) and answer (0, 1, 2)."""
    known = NR.lidar(1024, 41)[None]
    unknown = NR.lidar(2048, 42)[None].copy()
    unknown[0, 5] = np.inf
    unknown[0, 9, 0] = -np.inf
    unknown[0, 17, 2] = np.inf
    d2, idx = O.three_nn(unknown, known)
    assert (idx[0, [5, 9, 17]] == 0).all() and np.isinf(d2[0, [5, 9, 17]]).all()
    with _cabi.options(**NN_MODES[mode]):
        got_d2, got_idx, _ = pu.three_nn_weights(T(unknown, cuda), T(known, cuda))
    assert np.array_equal(got_idx.cpu().numpy(), idx)
    assert np.array_equal(got_d2.cpu().numpy(), d2)


def test_three_nn_batch_equals_per_scene(cuda, nn_cases):
    unknown, known, _, _ = nn_cases[(16384, 4096)]
    u, k = T(unknown, cuda), T(known, cuda)
    full = pu.three_nn_weights(u, k)
    for s in (0, 5, 6, 15):
        one = pu.three_nn_weights(u[s:s + 1].contiguous(), k[s:s + 1].contiguous())
        for a, b in zip(full, one):
            assert np.array_equal(a[s:s + 1].cpu().numpy(), b.cpu().numpy(), equal_nan=True), s


# ------------------------------------------------------------------------------------------------ FPS
@pytest.fixture(scope="module")
def fps_cases():
    out = {}
    for n, m in ((16384, 4096), (4097, 1024)):
        xyz, _ = batch(n, 1, (0.5, 1.0), 500 + n)
        xyz[3] = NR.sphere_around_zero(n, 3)                  # a tie of n - 1 points in the first round
        want, temp = O.fps(xyz, m, return_temp=True)
        out[(n, m)] = (xyz, want, temp)
    return out


FPS_OPTS = {"default": {}, "prune1": {"fps_prune": 1}, "prune2": {"fps_prune": 2}, "prune_1024": {"fps_prune": 1, "fps_threads": 1024},
            "cluster1": {"fps_prune": 0, "fps_cluster": 1}, "cluster2": {"fps_prune": 0, "fps_cluster": 2},
            "cluster4": {"fps_prune": 0, "fps_cluster": 4}, "cluster8": {"fps_prune": 0, "fps_cluster": 8},
            "generic": {"fps_prune": 0, "fps_generic": 1}}


@pytest.mark.parametrize("n,m", [(16384, 4096), (4097, 1024)])
@pytest.mark.parametrize("variant", list(FPS_OPTS))
def test_fps_bits_on_adversarial_families(cuda, fps_cases, n, m, variant):
    xyz, want, want_temp = fps_cases[(n, m)]
    x = T(xyz, cuda)
    with _cabi.options(**FPS_OPTS[variant]):
        idx, new_xyz = pu.furthest_point_sample_xyz(x, m, ordered=False)
        temp = torch.full((B, n), 1e10, device=cuda)
        idx2 = torch.empty((B, m), dtype=torch.int32, device=cuda)
        pointnet2_cuda.furthest_point_sampling_wrapper(B, n, m, x, temp, idx2)
    got = idx.cpu().numpy()
    bad = np.where(np.any(got != want, axis=1))[0]
    assert bad.size == 0, "scenes %s differ from the oracle" % bad.tolist()
    assert torch.equal(idx, idx2)
    assert np.array_equal(new_xyz.cpu().numpy(), np.stack([xyz[b][want[b]] for b in range(B)]), equal_nan=True)
    assert np.array_equal(temp.cpu().numpy(), want_temp, equal_nan=True)


def test_fps_ordered_shortcut_over_nested_lidar_levels(cuda):
    xyz = np.stack([NR.lidar(16384, 700 + s) for s in range(4)])
    x = T(xyz, cuda)
    for m in NR.RPN_NPOINTS:
        idx_o, nx_o = pu.furthest_point_sample_xyz(x, m, ordered=True)
        want = O.fps(x.cpu().numpy(), m)
        assert np.array_equal(idx_o.cpu().numpy(), want), m
        x = nx_o

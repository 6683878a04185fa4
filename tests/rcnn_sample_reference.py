"""Crafted IoU matrices for the RCNN RoI sampler (prb_rcnn_sample_rois, csrc/rcnn_sample.cu) and their scenes.

The sampler takes the RoI x GT IoU matrix as an input, so every selection decision can be put on an edge without
geometry: exact ties along a row and a column, IoUs on np.float32 of each threshold and one ulp either side, NaN, +-inf
and -0.0, every branch (fg+bg, fg only, bg only, status 1, status 2), hard only / easy only / both, fg counts around the
quota, HARD_BG_RATIO products just under an integer, RoI and GT counts below the buffer sizes with NaN behind them, and
the layer recipe's trailing zero GT rows.  The RoIs and GT boxes are distinct boxes whose geometry the sampler does not
look at (it copies them); a row's box identifies its source.

Used by oracle/make_golden_rcnn_sample_edges.py (the reference's own sampling on every `cases()` matrix),
tests/test_cpu_rcnn_sample_edges.py and tests/test_gpu_rcnn_sample_edges.py.
"""
import contextlib

import numpy as np

from oracle import rcnn_offline as RO

f32 = np.float32
# tools/cfgs/default.yaml; fg_thresh = min(REG_FG_THRESH, CLS_FG_THRESH)
LO, BG, FG, CLS = f32(0.05), f32(0.45), f32(0.55), f32(0.6)
THRESHOLDS = (LO, BG, FG, CLS)
NAN, INF = f32(np.nan), f32(np.inf)


def up(x):
    return np.nextafter(f32(x), f32(np.inf))


def dn(x):
    return np.nextafter(f32(x), f32(-np.inf))


def rois(m, scene=0):
    """m distinct RoIs: [x, y, z, h, w, l, ry], each field a function of the row"""
    i = np.arange(m, dtype=np.float64)
    b = np.stack([0.125 * i - 20.0 + scene, 1.5 + 0.001 * (i % 97), 30.0 + 0.0625 * (i % 211), np.full(m, 1.5), np.full(m, 1.6),
                  3.5 + 0.001 * (i % 503), 0.01 * (i % 300) - 1.5], 1)
    return b.astype(np.float32)


def gts(g, scene=0):
    """g distinct GT boxes, none of them all zero"""
    j = np.arange(g, dtype=np.float64)
    b = np.stack([0.5 * j - 60.0 + scene, np.full(g, 1.6), 12.0 + 0.25 * j, np.full(g, 1.52), np.full(g, 1.63), np.full(g, 3.88),
                  0.02 * j + 0.25], 1)
    return b.astype(np.float32)


def mat(rows, g, fill=0.0):
    """rows: lists of leading values (the rest of the row is `fill`) -> (len(rows), g) float32"""
    M = np.full((len(rows), g), fill, np.float32)
    for i, r in enumerate(rows):
        M[i, :len(r)] = np.asarray(r, np.float32)
    return M


def _case(name, M, R=16, cfg=None, roi_count=None, gt_count=None, zero_gt=(), golden=True):
    """one scene: the (m, g) matrix M, ROI_PER_IMAGE R, config overrides, the loader's counts (None: every row / column),
    the GT rows set to all zero (the layer trims the trailing ones), and whether the reference runs it (limit sizes do not)"""
    return dict(name=name, iou=np.asarray(M, np.float32), R=R, cfg=dict(cfg or {}), roi_count=roi_count, gt_count=gt_count,
                zero_gt=tuple(zero_gt), golden=golden)


def cases():
    """the small crafted scenes, run by the reference, the oracle and the device"""
    out = []
    z, nz = 0.0, -0.0
    # ties along a row (first max: the GT of lowest index), all-zero rows (GT 0), ties below the fg threshold
    out.append(_case("row_ties", mat([[0.7, 0.7, 0.1], [0.2, 0.8, 0.8], [0.9, 0.1, 0.9], [0.3, 0.3, 0.3], [z, z, z], [z, z, z],
                                      [0.02, 0.02, 0.01], [0.5, 0.2, 0.5], [0.1, 0.4, 0.4]], 3)))
    # ties along a column below the fg threshold: every GT's first-max RoI is row 0 (the loader appends it four times)
    out.append(_case("column_ties", mat([[0.3, 0.2, 0.4, 0.4], [0.3, 0.1, 0.4, 0.1], [0.1, 0.2, 0.1, 0.4], [0.01] * 4, [z] * 4,
                                         [0.2, 0.2, 0.2, 0.2], [0.04, 0.03, 0.02, 0.01]], 4)))
    # duplicate GT columns 1 and 3: a row's GT is column 1
    d = np.array([[0.1, 0.7, 0.2, 0.7], [0.3, 0.35, 0.1, 0.35], [0.6, 0.65, 0.0, 0.65], [0.0, 0.01, 0.02, 0.01], [0.2, 0.05, 0.1, 0.05]])
    out.append(_case("duplicate_gts", mat(d, 4)))
    # every threshold on f32(t) and one ulp either side, in column 0 and column 1
    vals = [v for t in THRESHOLDS for v in (dn(t), t, up(t))] + [f32(0), f32(1)]
    out.append(_case("thresholds", mat([[v, 0.0] for v in vals] + [[0.0, v] for v in vals], 2), R=32))
    # the same values with R = 8: fg above the quota of 4
    out.append(_case("thresholds_quota", mat([[v] for v in vals], 1), R=8))
    # NaN: in column 0, in a later column, in a later row of a column whose finite maximum comes first
    out.append(_case("nan", mat([[NAN, 0.7, 0.1], [0.3, NAN, 0.7], [0.8, 0.1, 0.1], [0.2, 0.1, 0.0], [0.01, 0.0, 0.0],
                                 [0.9, 0.2, NAN], [0.4, 0.3, 0.2], [0.02, 0.0, 0.0]], 3)))
    # NaN rows only in later columns, no other fg: the NaN rows must not become fg (nor the column maxima behind them)
    out.append(_case("nan_later", mat([[0.1, 0.9, NAN], [0.3, NAN, 0.6], [0.2, 0.1, 0.1], [0.0, 0.0, 0.01], [0.4, 0.0, 0.0]], 3)))
    # +-inf and signed zeros
    out.append(_case("inf_signed_zero", mat([[INF, 0.1], [-INF, -INF], [0.3, INF], [-INF, 0.2], [z, nz], [nz, z], [nz, nz],
                                             [0.6, 0.1], [-INF, 0.01], [0.2, -INF]], 2)))
    out.append(_case("signed_zero_bg", mat([[nz, z, z], [z, nz, nz], [nz, nz, nz], [z, z, nz], [-0.5, nz, z]], 3), R=12))
    # branches
    out.append(_case("fg_only", mat([[0.6, 0.1], [0.2, 0.9], [FG, 0.0], [1.0, 1.0]], 2)))
    out.append(_case("hard_only", mat([[0.7, 0.1], [0.2, 0.3], [LO, 0.0], [dn(BG), 0.1], [0.1, 0.1]], 2)))
    out.append(_case("easy_only", mat([[0.7, 0.1], [0.02, 0.03], [dn(LO), 0.0], [z, z], [nz, 0.01]], 2)))
    out.append(_case("no_fg_hard", mat([[0.2, 0.3], [LO, 0.0], [dn(BG), 0.1], [0.1, 0.1]], 2)))
    out.append(_case("no_fg_easy", mat([[z, z], [nz, -0.25], [-1.0, z]], 2), R=10))
    out.append(_case("no_fg_both", mat([[0.2, 0.3], [0.0, 0.01], [dn(BG), 0.1], [-0.5, 0.0], [0.1, 0.1], [dn(LO), 0.0]], 2)))
    out.append(_case("gap_only", mat([[BG, 0.0], [dn(FG), 0.3], [0.5, 0.5]], 2)))          # the layer: status 1
    out.append(_case("status1", mat([[z, z], [z, nz], [nz, nz]], 2), cfg=dict(CLS_BG_THRESH=0.0, CLS_BG_THRESH_LO=0.0)))
    out.append(_case("all_nan", np.full((4, 3), NAN, np.float32)))
    out.append(_case("no_rois", np.zeros((0, 3), np.float32)))
    out.append(_case("no_gts", np.zeros((5, 0), np.float32)))
    # counts below the buffer sizes (the loader); NaN behind them, which must not be read
    M = mat([[0.7, 0.1, 0.2], [0.3, 0.2, 0.1], [0.0, 0.01, 0.0], [0.9, 0.1, 0.6], [0.2, 0.5, 0.0]], 3)
    P = np.full((8, 5), NAN, np.float32)
    P[:5, :3] = M
    out.append(_case("counts", P, roi_count=5, gt_count=3))
    out.append(_case("roi_count_zero", P, roi_count=0, gt_count=3))
    out.append(_case("gt_count_zero", P, roi_count=5, gt_count=0))
    # the layer's GT trimming: a zero row in the middle stays (IoU 0 with every RoI), the trailing zero rows go
    T = mat([[0.7, 0.0, 0.1, 0.0, 0.0], [0.3, 0.0, 0.5, 0.0, 0.0], [0.0, 0.0, 0.01, 0.0, 0.0], [0.1, 0.0, 0.8, 0.0, 0.0],
             [0.2, 0.0, 0.2, 0.0, 0.0]], 5)
    out.append(_case("zero_gt_rows", T, zero_gt=(1, 3, 4)))
    out.append(_case("zero_gt_all", T, zero_gt=(0, 1, 2, 3, 4)))
    # fg counts around the quota (8 of R = 16): k rows over the threshold, the rest hard bg; the loader adds one GT-max RoI
    for k in (6, 7, 8, 9, 16):
        out.append(_case("fg_%d" % k, mat([[0.6 + 0.01 * i] for i in range(k)] + [[0.2]] * 4, 1)))
    # HARD_BG_RATIO: 0, 1, and 0.29 / 0.57 of 100 bg rows (float64 products 28.999999999999996 and 56.99999999999999)
    H = mat([[0.7]] * 28 + [[0.3], [0.2], [0.1]] + [[0.01], [0.0]], 1)
    for ratio in (0.0, 1.0, 0.29, 0.57):
        out.append(_case("ratio_%g" % ratio, H, R=128, cfg=dict(HARD_BG_RATIO=ratio)))
    return out


def _palette_matrix(rng, m, g, p_fg):
    """an (m, g) matrix of signed zeros with four overlaps per row: exact ties, values on and next to the bg thresholds and
    uniform IoUs below FG; about p_fg of the rows also get one overlap of 0.7, FG or one ulp over it"""
    low = np.array([0.0, -0.0, 0.3, 0.3, 0.3, dn(LO), LO, up(LO), dn(BG), BG, up(BG), dn(FG)], np.float32)
    M = np.where(rng.random((m, g)) < 0.5, f32(0.0), f32(-0.0)).astype(np.float32)
    for q in range(4):
        cols = rng.integers(0, g, m)
        M[np.arange(m), cols] = np.where(rng.random(m) < 0.6, low[rng.integers(0, len(low), m)], rng.random(m).astype(np.float32) * 0.5)
    fg_rows = np.nonzero(rng.random(m) < p_fg)[0]
    hi = np.array([0.7, 0.7, FG, up(FG)], np.float32)
    M[fg_rows, rng.integers(0, g, fg_rows.size)] = hi[rng.integers(0, len(hi), fg_rows.size)]
    return M


def big_cases():
    """the kernel's limits: m = 4096 RoIs, g = 256 GT boxes, R = 1024 rows (the device only)"""
    rng = np.random.default_rng(4096)
    m, g, R = 4096, 256, 1024
    out = [_case("limit_mixed", _palette_matrix(rng, m, g, 0.1), R=R, golden=False)]
    every = np.full((m, g), 0.01, np.float32)                   # every row fg, every GT's max RoI appended: n + ng candidates
    every[np.arange(m), np.arange(m) % g] = np.float32(0.9)
    out.append(_case("limit_every_fg", every, R=R, golden=False))
    # all rows but one fg: fg+bg with the quota of 512 taken without replacement from ~4350 candidates
    near = every.copy()
    near[17] = 0.01
    out.append(_case("limit_one_bg", near, R=R, golden=False))
    return out


def batch_cases():
    """scenes of one shape (m = 64, g = 8, R = 64) that take different branches in one launch"""
    rng = np.random.default_rng(8)
    m, g = 64, 8
    mixed = _palette_matrix(rng, m, g, 0.2)
    fg_only = np.full((m, g), 0.7, np.float32)
    bg_only = np.where(rng.random((m, g)) < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
    hard = np.full((m, g), 0.2, np.float32)
    status1 = np.full((m, g), 0.5, np.float32)                 # the gap: status 1 for the layer, fg via GT-max for the loader
    nan = _palette_matrix(rng, m, g, 0.2)
    nan[rng.random((m, g)) < 0.1] = NAN
    return [_case("batch_%d" % i, M, R=64, golden=False) for i, M in enumerate([mixed, fg_only, bg_only, hard, status1, nan])]


def scene(case, index=0):
    """-> rois (m, 7), gts (g, 7), iou (m, g) float32 of one case; with counts, NaN behind them in all three; zero_gt rows
    all zero"""
    M = case["iou"]
    m, g = M.shape
    r, t = rois(m, index), gts(g, index)
    if case["roi_count"] is not None:
        r[case["roi_count"]:] = NAN
    if case["gt_count"] is not None:
        t[case["gt_count"]:] = NAN
    for j in case["zero_gt"]:
        t[j] = 0.0
    return r, t, M.copy()


@contextlib.contextmanager
def no_jitter():
    """both recipes with 0 jitter tries: every row keeps its source box and IoU (the loader's 10 / 1 tries are fixed)"""
    orig = RO.recipe_values
    RO.recipe_values = lambda c, which: dict(orig(c, which), fg_aug_times=0, bg_aug_times=0)
    try:
        yield
    finally:
        RO.recipe_values = orig


def oracle_inputs(case, recipe, index=0):
    """the scene and IoU matrix sample_scene gets: the loader's counted rows and columns, the layer's every row"""
    r, t, M = scene(case, index)
    if recipe == "loader":
        n = len(r) if case["roi_count"] is None else case["roi_count"]
        ng = len(t) if case["gt_count"] is None else case["gt_count"]
        r, t, M = r[:n], t[:ng], M[:n, :ng]
    z = np.zeros((1, 3), np.float32)
    return dict(rpn_xyz=z, rpn_features=z[:, :1], rpn_intensity=z[:, 0], seg_mask=z[:, 0], roi_boxes3d=r, gt_boxes3d=t), M


def run_oracle(case, recipe, draw="hash", rng=np.random, seed=0, index=0):
    sc, M = oracle_inputs(case, recipe, index)
    cfg = dict(case["cfg"], ROI_PER_IMAGE=case["R"], NUM_POINTS=1, ROI_FG_AUG_TIMES=0)
    with no_jitter():
        return RO.sample_scene(sc, cfg, draw=draw, iou="fp32", rng=rng, seed=seed, scene_index=index, train=False, recipe=recipe, iou3d=M)


def bits(a):
    return np.asarray(a, np.float32).view(np.int32)

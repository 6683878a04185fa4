"""Seeded RPN outputs (scores (N,), reg (N, 76), xyz (N, 3)) that put the proposal layer's data-dependent branches on their
edges, for csrc/proposal.cu (decode_proposals_kernel, proposal_select_nms_kernel, proposal_pack_kernel) and its numpy
restatement oracle/proposal.py.

The channel layout is the default configuration's: LOC_SCOPE 3.0, LOC_BIN_SIZE 0.5, 12 heading bins, so
  x bins 0-11, z bins 12-23, x residuals 24-35, z residuals 36-47, y offset 48, heading bins 49-60, heading residuals
  61-72, sizes 73-75.
Most rows are "placed": x and z bin 5 with residual 0.5 decode to px = pz = 0 exactly, so the box centre is xyz's x and
z, heading bin 0 with residual 0 gives ry = 0 and size residual 0 the anchor size.  The edge rows of a scene come first
and carry the highest scores; random background rows with distinct lower scores fill the scene to N.

Families (`scene(family, variant, n, seed)`):
  range_edges       decoded z exactly 0, 40 and 80 and one ulp either side, z < 0 and z > 80
  tied_scores       a handful of score values; every score 0; groups of identical boxes with identical scores
  argmax_edges      equal maxima, an all-zero group, all -inf, +inf, NaN at position 0 and later, in the x, z and heading
                    bins (z around 40, so the bin decides the range)
  heading_wrap      ry before the wrap exactly 0, pi, 2 pi, -pi and one ulp either side, and large residuals
  degenerate_sizes  h, w or l exactly 0, negative sizes, boxes 1e3 m wide or long
  non_finite        NaN / +-inf scores, residuals, y offset and xyz
  quota_edges       near / far counts at and around the 6300 / 2700 caps, the far range empty (the near range's fallback
                    slice) below, at, between and above the caps, and the near range empty
  nms_clusters      dense clusters, suppression chains inside and across 32-candidate chunks, IoU within a few ulps
                    of 0.8 and 0.85, and isolated boxes where post_nms_top_n is reached at a chunk boundary or mid-chunk
Every score is distinct except in tied_scores.
"""
import numpy as np

from neighbour_reference import ulp_steps

F = np.float32
NB, NH, C = 12, 12, 76
XB, ZB, XR, ZR, YO, HB, HR, SZ = 0, 12, 24, 36, 48, 49, 61, 73
ANCHOR = np.array([1.52563191462, 1.62856739989, 3.88311640418], dtype=F)     # tools/cfgs/default.yaml:19
APC = F((2 * np.pi) / NH)
HALF_APC = F((2 * np.pi) / NH / 2)
PI, TWO_PI = F(np.pi), F(2 * np.pi)
TEST = dict(pre_nms_top_n=9000, post_nms_top_n=100, nms_thresh=0.8)             # default.yaml:163-165
TRAIN = dict(pre_nms_top_n=9000, post_nms_top_n=512, nms_thresh=0.85)           # default.yaml:156-158
MODES = {"test_normal": dict(TEST, nms_type="normal", distance_based=True),
         "test_rotate": dict(TEST, nms_type="rotate", distance_based=True),
         "train_normal": dict(TRAIN, nms_type="normal", distance_based=True),
         "train_rotate": dict(TRAIN, nms_type="rotate", distance_based=True),
         "score_based": dict(TEST, nms_type="rotate", distance_based=False)}
PRE0, PRE1 = 6300, 2700
N = 16384


def _top(k):
    """k distinct scores, descending, above every background score"""
    return (F(64) - np.arange(k, dtype=F) * F(2 ** -8)).astype(F)


def placed(n, rng, x=None, y=None, z=None):
    """(reg, xyz) of n placed rows (see the module docstring): the other bins get lower logits and random residuals, so
    that a wrong bin choice gives a different box"""
    reg = np.zeros((n, C), F)
    for lo, res, b, r in ((XB, XR, 5, 0.5), (ZB, ZR, 5, 0.5), (HB, HR, 0, 0.0)):
        reg[:, lo:lo + NB] = rng.uniform(-3, 0.5, (n, NB))
        reg[:, lo + b] = 1
        reg[:, res:res + NB] = rng.normal(0, 0.5, (n, NB))
        reg[:, res + b] = r
    xyz = np.stack([rng.uniform(-35, 35, n) if x is None else x, rng.uniform(-1, 2, n) if y is None else y,
                    rng.uniform(1, 79, n) if z is None else z], 1).astype(F)
    return reg, xyz


def background(n, rng):
    xyz = np.stack([rng.uniform(-40, 40, n), rng.uniform(-1, 3, n), rng.uniform(0.5, 79.5, n)], 1).astype(F)
    reg = rng.normal(0, 1.0, (n, C)).astype(F)
    reg[:, YO] *= F(0.3)
    reg[:, SZ:] *= F(0.1)
    scores = (F(-20) + rng.permutation(n).astype(F) * F(2 ** -10)).astype(F)
    return scores, reg, xyz


def _compose(n, rng, reg, xyz, scores=None):
    """edge rows first (top scores in row order unless given), background behind; truncated to n"""
    k = min(len(reg), n)
    s_bg, r_bg, x_bg = background(n - k, rng)
    s = _top(k) if scores is None else np.asarray(scores, F)[:k]
    return (np.concatenate([s, s_bg]).astype(F), np.concatenate([reg[:k], r_bg]).astype(F),
            np.concatenate([xyz[:k], x_bg]).astype(F))


def _shuffled(rng, *arrays):
    p = rng.permutation(len(arrays[0]))
    return [a[p] for a in arrays]


# ------------------------------------------------------------------------------------------------ families
RANGE_VALUES = [v for e in (0.0, 40.0, 80.0) for v in (np.nextafter(F(e), F(-np.inf)), F(e), np.nextafter(F(e), F(np.inf)))]
RANGE_VALUES += [F(-3.0), F(83.0)]


def range_edges(n, rng, variant):
    z = np.repeat(np.array(RANGE_VALUES, F), 40)
    reg, xyz = placed(len(z), rng, z=z)
    return _compose(n, rng, *_shuffled(rng, reg, xyz))


def tied_scores(n, rng, variant):
    if variant == "dup_boxes":                                  # 150 groups of 4 identical rows with one score
        reg, xyz = placed(150, rng)
        reg[:, HR] = rng.normal(0, 0.3, 150)
        reg, xyz = np.repeat(reg, 4, 0), np.repeat(xyz, 4, 0)
        reg, xyz, s = _shuffled(rng, reg, xyz, np.repeat(_top(150), 4))
        return _compose(n, rng, reg, xyz, s)
    s, reg, xyz = background(n, rng)
    s = rng.choice(np.array([0.5, 1.0, 1.5, 2.0, 2.5], F), n) if variant == "few_values" else np.zeros(n, F)
    return s.astype(F), reg, xyz


ARGMAX_KINDS = ("tie", "zeros", "neginf", "posinf", "posinf2", "nan0", "nan_late", "nan2")


def _argmax_logits(kind, rng):
    v = rng.uniform(-3, 1, NB).astype(F)
    p, q = sorted(rng.choice(NB, 2, replace=False))
    if kind == "tie":
        v[p] = v[q] = 2
    elif kind == "zeros":
        v[:] = 0
    elif kind == "neginf":
        v[:] = -np.inf
    elif kind == "posinf":
        v[q] = np.inf
    elif kind == "posinf2":
        v[p] = v[q] = np.inf
    elif kind == "nan0":
        v[0], v[q] = np.nan, 5
    elif kind == "nan_late":                                    # finite maxima before and after a NaN
        a = int(rng.integers(1, NB - 1))
        v[0], v[a], v[a + 1] = 4, np.nan, 5
    elif kind == "nan2":
        v[p] = v[q] = np.nan
    return v


def argmax_edges(n, rng, variant):
    rows = []
    for lo, res in ((XB, XR), (ZB, ZR), (HB, HR)):
        for kind in ARGMAX_KINDS:
            reg, xyz = placed(12, rng, z=rng.uniform(37, 43, 12))
            for r in range(12):
                reg[r, lo:lo + NB] = _argmax_logits(kind, rng)
                reg[r, res:res + NB] = rng.normal(0, 0.5, NB)
            rows.append((reg, xyz))
    reg, xyz = np.concatenate([r for r, _ in rows]), np.concatenate([x for _, x in rows])
    return _compose(n, rng, *_shuffled(rng, reg, xyz))


def pre_wrap_ry(reg):
    """the heading before torch.remainder: bin * angle_per_class + residual * angle_per_class / 2, in fp32"""
    reg = np.asarray(reg, F)
    b = np.argmax(reg[:, HB:HB + NH], axis=1)
    res = np.take_along_axis(reg[:, HR:HR + NH], b[:, None], axis=1)[:, 0]
    return (b.astype(F) * APC + res * HALF_APC).astype(F)


def _heading_for(target):
    """(bin, residual) whose decode puts ry exactly on target before the wrap"""
    for b in range(NH):
        base = F(b) * APC
        r0 = (np.float64(target) - np.float64(base)) / np.float64(HALF_APC)
        cand = ulp_steps(np.full(257, r0, F), np.arange(-128, 129))
        hit = np.nonzero((base + cand * HALF_APC).astype(F) == F(target))[0]
        if hit.size:
            return b, cand[hit[0]]
    raise ValueError("no residual decodes to %r" % target)


def wrap_targets():
    t = [F(0)]
    for v in (F(0), PI, TWO_PI, -PI):
        t += [np.nextafter(v, F(-np.inf)), np.nextafter(v, F(np.inf))] + ([] if v == 0 else [v])
    return t


def heading_wrap(n, rng, variant):
    regs, xyzs = [], []
    for t in wrap_targets():
        b, r = _heading_for(t)
        reg, xyz = placed(16, rng)
        reg[:, HB:HB + NH] = rng.uniform(-3, 0.5, (16, NH))
        reg[:, HB + b], reg[:, HR + b] = 1, r
        regs.append(reg)
        xyzs.append(xyz)
    for r in (37.5, -37.5, 1e3, -1e3, 1e6, -1e6, 3e38, -3e38):
        reg, xyz = placed(16, rng)
        reg[:, HR:HR + NH] = F(r)
        regs.append(reg)
        xyzs.append(xyz)
    return _compose(n, rng, *_shuffled(rng, np.concatenate(regs), np.concatenate(xyzs)))


SIZE_KINDS = {"h0": (-1, 0, 0), "w0": (0, -1, 0), "l0": (0, 0, -1), "all0": (-1, -1, -1), "neg": (0, -2.5, -2.5),
              "negl": (0, 0, -3), "wide": (0, 1e3 / ANCHOR[1] - 1, 0), "long": (0, 0, 1e3 / ANCHOR[2] - 1),
              "huge": (0, 1e3 / ANCHOR[1] - 1, 1e3 / ANCHOR[2] - 1)}


def degenerate_sizes(n, rng, variant):
    regs, xyzs = [], []
    for res in SIZE_KINDS.values():
        reg, xyz = placed(16, rng)
        reg[:, SZ:SZ + 3] = np.array(res, F)
        regs.append(reg)
        xyzs.append(xyz)
    return _compose(n, rng, *_shuffled(rng, np.concatenate(regs), np.concatenate(xyzs)))


NONFINITE_KINDS = {"x_res_nan": ("reg", XR, NB, np.nan), "z_res_inf": ("reg", ZR, NB, np.inf),
                   "z_res_neginf": ("reg", ZR, NB, -np.inf), "y_off_nan": ("reg", YO, 1, np.nan),
                   "y_off_inf": ("reg", YO, 1, np.inf), "h_inf": ("reg", SZ, 1, np.inf), "w_neginf": ("reg", SZ + 1, 1, -np.inf),
                   "l_nan": ("reg", SZ + 2, 1, np.nan),
                   "ry_res_nan": ("reg", HR, NH, np.nan), "ry_res_inf": ("reg", HR, NH, np.inf),
                   "x_nan": ("xyz", 0, 1, np.nan), "z_nan": ("xyz", 2, 1, np.nan), "y_inf": ("xyz", 1, 1, np.inf),
                   "x_inf": ("xyz", 0, 1, np.inf), "x_neginf": ("xyz", 0, 1, -np.inf)}


def non_finite(n, rng, variant):
    regs, xyzs = [], []
    for where, lo, cnt, v in NONFINITE_KINDS.values():
        reg, xyz = placed(12, rng)
        (reg if where == "reg" else xyz)[:, lo:lo + cnt] = v
        regs.append(reg)
        xyzs.append(xyz)
    reg, xyz = _shuffled(rng, np.concatenate(regs), np.concatenate(xyzs))
    s = _top(len(reg))
    pos = rng.choice(len(reg), 3, replace=False)                # one NaN, one +inf, one -inf score: no two tie
    s[pos] = np.array([np.nan, np.inf, -np.inf], F)
    return _compose(n, rng, reg, xyz, s)


QUOTA = {  # near count, far count, far rows score above every near row
    "near_eq": (PRE0, 1500, False), "near_m1": (PRE0 - 1, 1500, False), "near_p1": (PRE0 + 1, 1500, False),
    "far_eq": (3000, PRE1, True), "far_m1": (3000, PRE1 - 1, True), "far_p1": (3000, PRE1 + 1, True),
    "fb_below": (5000, 0, False), "fb_p1": (PRE0 + 1, 0, False), "fb_mid": (7500, 0, False),
    "fb_above": (PRE0 + PRE1 + 3000, 0, False), "near_empty": (0, 3000, False)}


def quota_edges(n, rng, variant):
    near, far, far_top = QUOTA[variant]
    assert near + far <= n
    out = n - near - far
    z = np.concatenate([rng.uniform(0.5, 39.5, near), rng.uniform(40.5, 79.5, far),
                        np.where(np.arange(out) % 2 == 0, 90.0, -2.0)]).astype(F)
    reg, xyz = placed(n, rng, z=z)
    s = (F(-20) + rng.permutation(n).astype(F) * F(2 ** -10)).astype(F)
    if far_top:
        s[near:near + far] = _top(far)
    return s, reg, xyz


# nms_clusters: boxes on a grid of 6 m cells never overlap (anchor size, ry = 0)
def _cells(rng, far):
    cx, cz = np.meshgrid(np.arange(-33.0, 34.0, 6.0), np.arange(43.0, 80.0, 6.0) if far else np.arange(3.0, 40.0, 6.0))
    c = np.stack([cx.ravel(), cz.ravel()], 1)
    return c[rng.permutation(len(c))]


def _at(rng, xz):
    xz = np.asarray(xz, np.float64).reshape(-1, 2)
    return placed(len(xz), rng, x=xz[:, 0], y=np.zeros(len(xz)), z=xz[:, 1])


def _isolated(rng, far, n_rows, n_dups):
    """n_rows rows in score order: n_rows - n_dups boxes in distinct cells, and n_dups exact copies of earlier rows
    (suppressed: IoU 1); the last row is a new box"""
    kinds = np.array(["n"] + list(rng.permutation(["d"] * n_dups + ["n"] * (n_rows - n_dups - 2))) + ["n"])
    cells, xz, used = _cells(rng, far), [], 0
    for k in kinds:
        if k == "n":
            xz.append(cells[used])
            used += 1
        else:
            xz.append(xz[int(rng.integers(0, len(xz)))])
    return _at(rng, xz)


def _chains(rng, far):
    """rows in score order: fillers and triples A, B, C 0.3 m apart along the box length (IoU(A, B) = IoU(B, C) = 0.857,
    IoU(A, C) = 0.73): A keeps, B goes, C stays.  Triple positions 31-33 and 62-64 straddle chunk boundaries, 34-36
    and 65-79 sit inside a chunk"""
    cells = _cells(rng, far)
    xz, used = [], 0

    def fill(k):
        nonlocal used
        for _ in range(k):
            xz.append(cells[used])
            used += 1

    def chain():
        nonlocal used
        for t in range(3):
            xz.append(cells[used] + np.array([0.3 * t - 0.3, 0.0]))
        used += 1
    fill(31)
    chain()
    chain()
    fill(62 - len(xz))
    for _ in range(6):
        chain()
    return _at(rng, xz)


def _size_residual(anchor, target):
    """a size residual whose decode r * anchor + anchor is exactly target"""
    r0 = (np.float64(target) - np.float64(anchor)) / np.float64(anchor)
    cand = ulp_steps(np.full(257, r0, F), np.arange(-128, 129))
    hit = np.nonzero((cand * F(anchor) + F(anchor)).astype(F) == F(target))[0]
    return cand[hit[0]]


THRESH_STEP = 2.0 ** -22


def _threshold_pairs(rng):
    """pairs A (score above) and B of 4 x 2 m boxes, ry = 0, B shifted by d = k 2^-22 m along x from x = 0.5: every bev
    coordinate, area and union is exact in fp32, so the axis-aligned IoU (4 - d) / (4 + d) is one rounding, and k runs
    over the 7 values around the threshold for 0.8 and for 0.85"""
    xz = []
    j = 0
    for t in (0.8, 0.85):
        k0 = int(round(4 * (1 - t) / (1 + t) / THRESH_STEP))
        for k in range(k0 - 3, k0 + 4):
            z = 1.5 + 3 * j if j < 13 else 43.5 + 3 * (j - 13)
            xz += [(0.5, z), (0.5 + k * THRESH_STEP, z)]
            j += 1
    reg, xyz = _at(rng, xz)
    reg[:, SZ + 1] = _size_residual(ANCHOR[1], 2.0)
    reg[:, SZ + 2] = _size_residual(ANCHOR[2], 4.0)
    return reg, xyz


def nms_clusters(n, rng, variant):
    if variant == "dense":                                      # 48 clusters of 32: half in score blocks, half interleaved
        centres = np.stack(np.meshgrid(np.arange(-30.0, 31.0, 10.0), np.arange(5.0, 76.0, 10.0)), -1).reshape(-1, 2)[:48]
        xz = np.repeat(centres, 32, 0) + rng.normal(0, 0.12, (48 * 32, 2))
        reg, xyz = _at(rng, xz)
        flip = rng.random(len(reg)) < 0.2
        reg[:, HR] = rng.normal(0, 0.05, len(reg))
        reg[flip, HB], reg[flip, HB + 6], reg[flip, HR + 6] = 0, 2, rng.normal(0, 0.05, flip.sum())
        rank = np.arange(len(reg))
        inter = rank >= 24 * 32
        rank[inter] = 24 * 32 + (rank[inter] - 24 * 32) % 32 * 24 + (rank[inter] - 24 * 32) // 32
        return _compose(n, rng, reg, xyz, _top(len(reg))[rank])
    if variant == "chains":
        parts = [_chains(rng, False), _chains(rng, True)]
    elif variant == "thresh":
        parts = [_threshold_pairs(rng)]
    elif variant == "isolated_boundary":                       # TEST: post 70 / 30 reached at candidate 96 / 128
        parts = [_isolated(rng, False, 96, 26), _isolated(rng, True, 128, 98)]
    else:                                                       # isolated_mid: every box kept
        parts = [_isolated(rng, False, 84, 0), _isolated(rng, True, 84, 0)]
    return _compose(n, rng, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]))


FAMILIES = {"range_edges": range_edges, "tied_scores": tied_scores, "argmax_edges": argmax_edges,
            "heading_wrap": heading_wrap, "degenerate_sizes": degenerate_sizes, "non_finite": non_finite,
            "quota_edges": quota_edges, "nms_clusters": nms_clusters}
VARIANTS = {"tied_scores": ("few_values", "all_zero", "dup_boxes"), "quota_edges": tuple(QUOTA),
            "nms_clusters": ("dense", "chains", "thresh", "isolated_boundary", "isolated_mid")}
SCENES = [(f, v) for f in FAMILIES for v in VARIANTS.get(f, ("",))]
TIED = ("tied_scores",)
# two batches of 16 scenes, each scene from another family or variant, topped up with reseeded edge families
_EXTRA = [("range_edges", ""), ("argmax_edges", ""), ("heading_wrap", ""), ("degenerate_sizes", ""), ("non_finite", ""),
          ("nms_clusters", "dense"), ("nms_clusters", "chains"), ("nms_clusters", "thresh"), ("tied_scores", "dup_boxes")]
BATCHES = [(SCENES + _EXTRA)[:16], (SCENES + _EXTRA)[16:32]]


def scene(family, variant="", n=N, seed=0):
    rng = np.random.default_rng([seed, list(FAMILIES).index(family), (VARIANTS.get(family, ("",)) + ("",)).index(variant)])
    return FAMILIES[family](n, rng, variant)


def batch(k, n=N, seed=0):
    """BATCHES[k] as (scores (16, n), reg (16, n, 76), xyz (16, n, 3)); scene s is seeded with seed + 16 k + s"""
    rows = [scene(f, v, n, seed + 16 * k + s) for s, (f, v) in enumerate(BATCHES[k])]
    return tuple(np.ascontiguousarray(np.stack([r[i] for r in rows])) for i in range(3))

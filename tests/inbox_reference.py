"""A float64 reference of the point-in-box decisions of the device kernels, a derived bound on how far any fp32 evaluation
of them can be from it, and seeded point / box families that put points where an fp32 predicate goes wrong.

Boxes are [x, y, z, h, w, l, ry] in the rectified camera frame, y the bottom face.  With dx = x_p - x, dz = z_p - z,
  x_rot = dx cos ry - dz sin ry,  z_rot = dx sin ry + dz cos ry,
a point is inside iff every condition of its rule holds (closed faces):
  pool   pt_in_box3d (csrc/roipool3d.cu pt_in_box, oracle orc_pt_in_box3d): |dx| <= 10, |dz| <= 10 (the cap),
         |y_p - cy| <= h/2 with cy = y - h/2, |x_rot| <= l/2, |z_rot| <= w/2
  label  in_box of csrc/kitti_io.cu (the hull test of generate_rpn_training_labels): -h <= y_p - y <= 0, |x_rot| <= l/2,
         |z_rot| <= w/2, no cap
  paste  the pool rule on the box with h + 2 (added in fp32, as gt_paste.cu does)

membership() evaluates each condition in float64 on the fp32 inputs, with the kernels' comparisons, so NaN decides as on
the device: a rejecting test (`|dx| > 10`, `dy > 0`, ...) is false on NaN and keeps the point, an accepting test
(`|x_rot| <= l/2`, ...) is false on NaN and drops it.  A condition's slack is limit - |value|; margin is the smallest
slack, the distance in metres to the nearest decision boundary (>= 0 exactly when inside); a NaN slack counts as +inf
where its test keeps the point and -inf where it drops it.

band() bounds |fp32 slack - float64 slack| of every condition, U = 2^-24 the unit roundoff of fp32, to first order:
  differences  dx = fl(x_p - x): |err| <= U |dx|; likewise dz, and dy of the label rule
  cy           pool rule: the kernels round y - h/2 to fp32 (|err| <= U |cy|), then dy = fl(y_p - cy) adds U |dy|
  cos, sin     device cosf / sinf / sincosf are within 2 ulp (build.py does not use fast math), host cosf and
               (float)cos(double) within less; an ulp of v is at most 2U |v|, so |err| <= 4U |cos ry|, 4U |sin ry|
  rotation     x_rot = a - b with a = dx cos, b = dz sin: each product inherits (U + 4U) of its size from its inputs and
               U from its own rounding unless an FMA contracts it, the sum U of |a| + |b|: |err| <= 7U (|a| + |b|) whether
               or not the compiler contracts (the label kernel leaves that to it); likewise z_rot
  limits       10, h/2, l/2 and w/2 are exact (double halves in the pool kernels, fp32 * 0.5 in the label kernel)
The band of a pair is the largest of its conditions' bounds times (1 + 2^-10) for the second-order terms.  Each term is
U times a coordinate difference, a box coordinate or a rotated extent, so the band follows the ulp of the coordinates
and stays valid at far range.  A point is certain-inside when margin > band, certain-outside when margin < -band; in
between any fp32 evaluation may go either way.

delaunay=True widens the label band for the reference's own labels, which test the point against the hull of the fp32
corners of boxes3d_to_corners3d (a float32 matmul with numpy's float32 cos / sin, then + centre): a corner moves by at
most 10U (|l/2 cos| + |w/2 sin|) + U (|x| + |l/2| + |w/2|) in x and z (numpy's float32 cos / sin within 4 ulp) and
U |y - h| in y, the hull by no more than its corners, and qhull's find_simplex adds a tolerance of a few 1e-13 m.
"""
import numpy as np

U = 2.0 ** -24
CAP = 10.0
RULES = ("pool", "label", "paste")
FAMILIES = ("random", "faces", "edges", "corners", "headings", "cap", "degenerate", "far", "overlap")


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def rule_boxes(boxes, rule):
    """the fp32 boxes the kernel of `rule` tests against"""
    b = f32(boxes).reshape(-1, 7).copy()
    if rule == "paste":
        b[:, 3] = b[:, 3] + np.float32(2)
    return b


def _conditions(pts, boxes, rule):
    """-> list of (slack, passes, err), each (M, N) float64 / bool / float64"""
    assert rule in RULES, rule
    p = f32(pts).reshape(-1, 3).astype(np.float64)[None]
    b = rule_boxes(boxes, rule).astype(np.float64)[:, None]
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    cx, by, cz, h, w, l, ry = (b[..., k] for k in range(7))
    with np.errstate(invalid="ignore", over="ignore"):
        c, s = np.cos(ry), np.sin(ry)
        dx, dz = x - cx, z - cz
        xr, zr = dx * c - dz * s, dx * s + dz * c
        rot = 7 * U * (np.abs(dx * c) + np.abs(dz * s))
        rot_z = 7 * U * (np.abs(dx * s) + np.abs(dz * c))
        hl, hw = l / 2, w / 2
        out = []
        if rule == "label":
            dy = y - by
            out.append((-dy, ~(dy > 0), U * np.abs(dy)))
            out.append((dy + h, ~(dy < -h), U * np.abs(dy)))
        else:
            hh = h / 2
            cy = by - hh
            dy = y - cy
            out.append((CAP - np.abs(dx), ~(np.abs(dx) > CAP), U * np.abs(dx)))
            out.append((CAP - np.abs(dz), ~(np.abs(dz) > CAP), U * np.abs(dz)))
            out.append((hh - np.abs(dy), ~(np.abs(dy) > hh), U * (np.abs(cy) + np.abs(dy))))
        out.append((hl - np.abs(xr), (xr >= -hl) & (xr <= hl), rot))
        out.append((hw - np.abs(zr), (zr >= -hw) & (zr <= hw), rot_z))
    return out


def membership(pts, boxes, rule):
    """(N,3) points, (M,7) boxes -> inside (M,N) bool, margin (M,N) float64 (metres to the nearest decision boundary,
    >= 0 inside)"""
    conds = _conditions(pts, boxes, rule)
    inside = np.logical_and.reduce([ok for _, ok, _ in conds])
    margin = np.full(inside.shape, np.inf)
    for slack, ok, _ in conds:
        margin = np.minimum(margin, np.where(np.isnan(slack), np.where(ok, np.inf, -np.inf), slack))
    assert np.array_equal(margin >= 0, inside)
    return inside, margin


def band(pts, boxes, rule, delaunay=False):
    """(M,N) bound on |fp32 slack - float64 slack| over the pair's conditions (module docstring)"""
    conds = _conditions(pts, boxes, rule)
    e = np.zeros(conds[0][0].shape)
    for _, _, err in conds:
        e = np.maximum(e, np.where(np.isfinite(err), err, 0.0))
    if delaunay:
        assert rule == "label"
        b = rule_boxes(boxes, rule).astype(np.float64)
        with np.errstate(invalid="ignore"):
            c, s = np.abs(np.cos(b[:, 6])), np.abs(np.sin(b[:, 6]))
        hl, hw = np.abs(b[:, 5]) / 2, np.abs(b[:, 4]) / 2
        corner = 10 * U * (hl * c + hw * s) + U * (np.maximum(np.abs(b[:, 0]), np.abs(b[:, 2])) + hl + hw)
        corner = np.maximum(corner, U * np.abs(b[:, 1] - b[:, 3]))
        e = e + np.where(np.isfinite(corner), corner, 0.0)[:, None] + 1e-9
    return e * (1 + 2.0 ** -10)


def classify(pts, boxes, rule, delaunay=False):
    """-> inside (float64), certain_in, certain_out, all (M,N)"""
    inside, margin = membership(pts, boxes, rule)
    bnd = band(pts, boxes, rule, delaunay)
    return inside, margin > bnd, margin < -bnd


def frustum(lidar, calib, use_range=True):
    """the validity test of csrc/kitti_io.cu kitti_prepare_kernel (get_valid_flag of the reference) in float64 on the fp32
    inputs: lidar (N, >= 3), calib the 32 floats the kernel reads (Calibration.pack: M (4x3) with rect = [x y z 1] . M,
    P2 (3x4), image height and width, range box x0 x1 y0 y1 z0 z1).  Conditions: 0 <= u < W, 0 <= v < H, depth >= 0
    with u, v = P2 row 0, 1 . [rect 1] / rect z and depth = P2 row 2 . [rect 1] - P2[2,3], and, with use_range, rect
    inside the range box.  -> valid (N,) bool, certain_valid, certain_invalid.

    Bound of each condition, U = 2^-24, first order times (1 + 2^-10):
      rect_k       four products and sums, each one rounding, in any order or contraction: 4U T_k with T_k the sum of
                   the absolute terms |x M0k| + |y M1k| + |z M2k| + |M3k|
      h_k          the rect errors through P2 (sum_j |P_kj| e_j) plus 4U of its own absolute terms
      u, v         h / rect z: (e_h + |u| e_z) / |rect z| + U |u|; a point whose rect z is within twice its error of 0
                   is never certain
      depth, box   e_h2 + U |depth|; e_rect_k for a range-box face"""
    p = f32(lidar)[:, :3].astype(np.float64)
    c = f32(calib).astype(np.float64)
    M, P = c[0:12].reshape(4, 3), c[12:24].reshape(3, 4)
    H, W = c[24], c[25]
    terms = np.abs(p[:, :, None] * M[None, 0:3]).sum(1) + np.abs(M[3])[None]
    r = p @ M[0:3] + M[3]
    er = 4 * U * terms
    hom = np.concatenate([r, np.ones((len(r), 1))], 1)
    h = hom @ P.T
    eh = er @ np.abs(P[:, 0:3]).T + 4 * U * (np.abs(r[:, None, :] * P[None, :, 0:3]).sum(2) + np.abs(P[:, 3])[None])
    z, ez = r[:, 2], er[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = h[:, 0] / z, h[:, 1] / z
        eu = (eh[:, 0] + np.abs(u) * ez) / np.abs(z) + U * np.abs(u)
        ev = (eh[:, 1] + np.abs(v) * ez) / np.abs(z) + U * np.abs(v)
    fragile = np.abs(z) <= 2 * ez
    eu, ev = np.where(fragile, np.inf, eu), np.where(fragile, np.inf, ev)
    depth = h[:, 2] - P[2, 3]
    ed = eh[:, 2] + U * np.abs(depth)
    conds = [(u, eu), (W - u, eu), (v, ev), (H - v, ev), (depth, ed)]
    if use_range:
        for k in range(3):
            conds += [(r[:, k] - c[26 + 2 * k], er[:, k]), (c[27 + 2 * k] - r[:, k], er[:, k])]
    strict = {1, 3}                                          # u < W and v < H; every other test is closed
    valid = np.logical_and.reduce([s > 0 if i in strict else s >= 0 for i, (s, _) in enumerate(conds)])
    k = 1 + 2.0 ** -10
    certain_valid = np.logical_and.reduce([s > k * e for s, e in conds])
    certain_invalid = np.logical_or.reduce([s < -k * e for s, e in conds])
    return valid, certain_valid, certain_invalid


# ------------------------------------------------------------------------------------------------ checks shared by tests
def rows_to_index(rows, *columns):
    """pooled rows (..., W) that are bit copies of the rows of the point table [columns...] (each (N, k), W = sum of k) ->
    the point index of each row (-1: no such point); equal points map to the lowest index"""
    n = len(columns[0])
    table = np.concatenate([f32(c).reshape(n, -1) for c in columns], 1)
    width = table.shape[1]
    lut = {}
    for i, key in enumerate(map(bytes, table.view(np.uint32))):
        lut.setdefault(key, i)
    r = f32(rows).reshape(-1, width).view(np.uint32)
    return np.array([lut.get(bytes(k), -1) for k in r], np.int64).reshape(np.shape(rows)[:-1])


def check_pool_selection(idx, empty, pts, boxes, rule="pool", where=""):
    """idx (M,S) point index of every pooled row of one scene (anything for an empty box), empty (M,): the rows must be the
    first S inside points in index order, padded with slot k % cnt, and every decision must agree with the float64
    membership outside the band.  Returns (number of boxes, number of in-band pairs among the decisions)"""
    idx, empty = np.asarray(idx), np.asarray(empty).astype(bool)
    M, S = idx.shape
    _, cin, cout = classify(pts, boxes, rule)
    for m in range(M):
        tag = "%s box %d" % (where, m)
        ci = np.nonzero(cin[m])[0]
        if empty[m]:
            assert len(ci) == 0, "%s: empty, but points %s are certainly inside" % (tag, ci[:8])
            continue
        seq = idx[m]
        assert (seq >= 0).all(), "%s: a pooled row is not a copy of a scene point" % tag
        up = np.nonzero(np.diff(seq) <= 0)[0]
        cnt = int(up[0]) + 1 if len(up) else S
        sel = seq[:cnt]
        pad = np.arange(cnt, S)
        assert np.array_equal(seq[pad], sel[pad % cnt]), "%s: rows past cnt = %d are not slot k %% cnt" % (tag, cnt)
        bad = sel[cout[m, sel]]
        assert len(bad) == 0, "%s: selected points %s are certainly outside" % (tag, bad[:8])
        skipped = np.setdiff1d(ci[ci < sel[-1]] if cnt == S else ci, sel)
        assert len(skipped) == 0, "%s: certainly inside points %s were skipped (cnt %d of S %d)" % (tag, skipped[:8], cnt, S)
    return M, int((~cin & ~cout).sum())


def label_replay(pts, boxes, extra=0.2, count=None, delaunay=False):
    """generate_rpn_training_labels' loop (boxes in order, later boxes overwrite; fg -> 1, fg != enlarged -> -1) replayed
    with every certain decision fixed and every in-band one free.  count=None skips all-zero size rows as the batched
    kernel does without gt_count; else the first `count` rows are the boxes.  -> possible (N, 3) bool over the labels
    (-1, 0, 1), certain (N,) every decision of the point is certain, last (N,) the last box the point is certainly in
    among the kept rows (-1 none), rows (the kept boxes)"""
    b = f32(boxes).reshape(-1, 7)
    keep = ~((b[:, 3] == 0) & (b[:, 4] == 0) & (b[:, 5] == 0)) if count is None else np.arange(len(b)) < count
    b = b[keep]
    big = b.copy()
    big[:, 1] = b[:, 1] + np.float32(extra)
    big[:, 3:6] = b[:, 3:6] + np.float32(2 * extra)
    n = len(f32(pts).reshape(-1, 3))
    possible = np.zeros((n, 3), bool)
    possible[:, 1] = True
    certain = np.ones(n, bool)
    last = np.full(n, -1)
    if len(b):
        fin, fi, fo = classify(pts, b, "label", delaunay)
        _, bi, bo = classify(pts, big, "label", delaunay)
        for k in range(len(b)):
            a11, a00 = ~fo[k] & ~bo[k], ~fi[k] & ~bi[k]
            amix = (~fo[k] & ~bi[k]) | (~fi[k] & ~bo[k])
            pm, p0, p1 = possible.T
            possible = np.stack([amix | (a00 & pm), a00 & p0, a11 | (a00 & p1)], 1)
            certain &= (fi[k] | fo[k]) & (bi[k] | bo[k])
            last = np.where(fin[k], k, last)
    return possible, certain, last, b


def reg_labels(pts, rows, last):
    """the regression targets of csrc/kitti_io.cu rpn_labels_kernel in numpy fp32 (each op one rounding): centre - point
    with the centre's y at y - h * 0.5, then h, w, l, ry of the last box the point is in (zeros when none)"""
    p = f32(pts).reshape(-1, 3)
    reg = np.zeros((len(p), 7), np.float32)
    fg = last >= 0
    b = f32(rows)[last[fg]]
    reg[fg, 0] = b[:, 0] - p[fg, 0]
    reg[fg, 1] = (b[:, 1] - b[:, 3] * np.float32(0.5)) - p[fg, 1]
    reg[fg, 2] = b[:, 2] - p[fg, 2]
    reg[fg, 3:7] = b[:, 3:7]
    return reg


def check_labels(cls, reg, pts, boxes, count=None, delaunay=False, where=""):
    """every label is one the float64 replay allows; where every decision is certain, the regression targets equal
    reg_labels bit for bit.  Returns the number of points with an in-band decision"""
    cls, reg = np.asarray(cls), np.asarray(reg)
    possible, certain, last, rows = label_replay(pts, boxes, count=count, delaunay=delaunay)
    ok = possible[np.arange(len(cls)), cls + 1]
    assert ok.all(), "%s: labels %s at points %s are outside the band" % (where, cls[~ok][:8], np.nonzero(~ok)[0][:8])
    want = reg_labels(pts, rows, last)
    same = ((reg.view(np.uint32) == want.view(np.uint32)) | (np.isnan(reg) & np.isnan(want))).all(1)     # any NaN payload
    bad = np.nonzero(certain & ~same)[0]
    assert len(bad) == 0, "%s: regression targets differ at points %s with certain decisions" % (where, bad[:8])
    return int((~certain).sum())


# ------------------------------------------------------------------------------------------------ families
def _cars(rng, m, off=0.0):
    b = np.empty((m, 7))
    b[:, 0] = rng.uniform(-30, 30, m) + off
    b[:, 1] = rng.uniform(1.4, 1.9, m)
    b[:, 2] = rng.uniform(5, 65, m) + off
    b[:, 3] = rng.uniform(1.4, 1.8, m)
    b[:, 4] = rng.uniform(1.5, 1.9, m)
    b[:, 5] = rng.uniform(3.4, 4.6, m)
    b[:, 6] = rng.uniform(-np.pi, np.pi, m)
    return b


def _offsets(rng, n, scale):
    """signed offsets of k ulp of `scale`: |k| in 0..8 and powers of two up to 2^14, half outward, half inward"""
    k = np.where(rng.random(n) < 0.6, rng.integers(0, 9, n), 2.0 ** rng.integers(4, 15, n))
    return rng.choice([-1.0, 1.0], n) * k * ulp(scale)


def _to_world(box, loc):
    """box-frame coordinates (u along l, v along h from the box centre, t along w) -> float64 world points"""
    c, s = np.cos(box[:, 6]), np.sin(box[:, 6])
    u, v, t = loc[:, 0], loc[:, 1], loc[:, 2]
    return np.stack([box[:, 0] + u * c + t * s, box[:, 1] - box[:, 3] / 2 + v, box[:, 2] - u * s + t * c], 1)


def _near_faces(rng, box, nfix):
    """points of `box` rows with nfix of their three box-frame coordinates at a face +- k ulp, the rest inside"""
    n = len(box)
    half = np.abs(box[:, [5, 3, 4]]) / 2
    loc = rng.uniform(-0.9, 0.9, (n, 3)) * half
    order = np.argsort(rng.random((n, 3)), 1)[:, :nfix]
    scale = np.maximum(np.abs(box[:, [0, 2]]).max(1), np.abs(box[:, 1]))
    for j in range(nfix):
        a = order[:, j]
        sgn = rng.choice([-1.0, 1.0], n)
        loc[np.arange(n), a] = sgn * (half[np.arange(n), a] + _offsets(rng, n, np.maximum(scale, 1.0)))
    return _to_world(box, loc)


def _around(rng, boxes, per, spread):
    which = np.repeat(np.arange(len(boxes)), per)
    b = boxes[which]
    loc = rng.uniform(-spread, spread, (len(b), 3)) * np.abs(b[:, [5, 3, 4]]) / 2
    return _to_world(b, loc)


def family(name, seed, m=24, per=48):
    """one scene of family `name`: (N,3) fp32 points, (m,7) fp32 boxes; N about m * per, points shuffled"""
    rng = np.random.default_rng([seed, FAMILIES.index(name)])
    boxes = _cars(rng, m)
    n = m * per
    which = np.repeat(np.arange(m), per)
    if name == "random":
        scope = rng.uniform([-40, -1, 0], [40, 3, 70.4], (n // 2, 3))
        pts = np.concatenate([scope, _around(rng, boxes, per - per // 2, 1.6)], 0)
    elif name in ("faces", "edges", "corners"):
        pts = _near_faces(rng, boxes[which], ("faces", "edges", "corners").index(name) + 1)
    elif name == "headings":
        base = rng.choice([0.0, 0.5, 1.0, 1.5, -0.5, -1.0, 2.0], m) * np.pi
        step = rng.integers(-3, 4, m) * ulp(np.maximum(np.abs(base), 1e-30))
        boxes[:, 6] = np.where(rng.random(m) < 0.75, f32(base) + step, rng.choice([-1, 1], m) * rng.uniform(990, 1010, m))
        boxes[: m // 4, 4] = boxes[: m // 4, 5]                       # squares: a turn by pi/2 maps the box onto itself
        half = per // 2
        pts = np.concatenate([_near_faces(rng, boxes[np.repeat(np.arange(m), half)], 1), _around(rng, boxes, per - half, 1.3)], 0)
    elif name == "cap":
        boxes[:, 5] = rng.uniform(20, 40, m)
        boxes[:, 4] = rng.uniform(2, 25, m)
        boxes[: m // 3, 6] = rng.choice([0.0, np.pi / 4, -np.pi / 4, np.pi / 2], m // 3)
        b = boxes[which]
        half = per // 2
        # |dx| or |dz| = 10 m +- k ulp, the other coordinate anywhere within the cap, y inside
        d = rng.choice([-1.0, 1.0], len(b)) * (CAP + _offsets(rng, len(b), 10.0))
        o = rng.uniform(-10, 10, len(b))
        onx = rng.random(len(b)) < 0.5
        y = b[:, 1] - b[:, 3] * rng.uniform(0.1, 0.9, len(b))
        edge = np.stack([b[:, 0] + np.where(onx, d, o), y, b[:, 2] + np.where(onx, o, d)], 1)
        loose = np.stack([b[:, 0] + rng.uniform(-15, 15, len(b)), y, b[:, 2] + rng.uniform(-15, 15, len(b))], 1)
        pts = np.where((np.arange(len(b)) % per < half)[:, None], edge, loose)
    elif name == "degenerate":
        pts = _around(rng, boxes, per, 1.4)
        k = np.arange(m) % 8
        for j, col in enumerate((3, 4, 5)):                           # zero and negative sizes
            boxes[k == j, col] = 0.0
            boxes[k == j + 3, col] = -boxes[k == j + 3, col]
        bad = np.array([np.nan, np.inf, -np.inf])
        boxes[k == 6, rng.integers(0, 7)] = bad[rng.integers(0, 3)]    # one non-finite field per box
        boxes[np.nonzero(k == 7)[0], rng.integers(0, 7, (k == 7).sum())] = bad[rng.integers(0, 3, (k == 7).sum())]
        hit = rng.random(len(pts)) < 0.06                              # non-finite coordinates
        pts[hit, rng.integers(0, 3, hit.sum())] = bad[rng.integers(0, 3, hit.sum())]
        dup = rng.integers(0, len(pts), len(pts) // 8)                 # duplicate points
        pts[rng.integers(0, len(pts), len(dup))] = pts[dup]
    elif name == "far":
        boxes = _cars(rng, m, off=3.0e4)
        half = per // 2
        pts = np.concatenate([_near_faces(rng, boxes[np.repeat(np.arange(m), half)], rng.integers(1, 4)),
                              _around(rng, boxes, per - half, 1.4)], 0)
    elif name == "overlap":
        g = m // 4                                                     # groups of four boxes around one spot
        lead = np.repeat(np.arange(g), 4)
        boxes[: 4 * g, [0, 1, 2]] = boxes[lead, :][:, [0, 1, 2]] + rng.uniform(-0.8, 0.8, (4 * g, 3)) * [1, 0.2, 1]
        pts = _around(rng, boxes, per, 1.6)
    else:
        raise KeyError(name)
    pts = f32(pts)[rng.permutation(len(pts))]
    return pts, f32(boxes)

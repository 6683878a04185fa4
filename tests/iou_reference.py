"""A float64 reference of the rotated BEV overlap (csrc/iou3d_dev.cuh) with an error bound, a conditioning measure, and a
generator of seeded box-pair families where the reference's algorithm is known to be fragile.

The overlap kernel is the reference's algorithm (corners rotated about the centre, 4 x 4 edge crossings, corners of one
box inside the other with a fixed MARGIN of 1e-5, bubble sort by polar angle, fan area) and must stay bit-identical to
it.  That algorithm is only right on well-conditioned pairs:

  exact        the intersection of the two rectangles the fp32 box describes: corners [x1,y1],[x2,y1],[x2,y2],[x1,y2]
               rotated about the fp32 centre ((x1 + x2) / 2, (y1 + y2) / 2) exactly as rot_center rotates them, with
               cos / sin of the fp32 heading, all in float64, clipped by a float64 Sutherland-Hodgman
  conditioning a pair is ill-conditioned when a corner of one box lies within MARGIN + CORNER_ULPS ulp(R) of the other
               box's boundary (the inside test can go either way, or count it twice with an edge crossing), when two
               edges whose bounding boxes come within EDGE_GAP meet at |sin| < MIN_SIN (the crossing is badly placed or
               missed, or a sliver is counted), or
               when a field is not finite or an extent is <= 0
  the bound    |got - exact| <= K_BOUND * U * R * (P_a + P_b) on well-conditioned pairs, R the largest corner coordinate
               (at least 1 m), P a perimeter.  K_BOUND is chosen from 1.31e6 well-conditioned pairs of the oracle
               (oracle/pointops_oracle.c; generic, nested, pedestrian and 20 m families, near, far and at 1000 m): the
               largest |got - exact| / (U R (P_a + P_b)) was 0.51, 0.227 of K_BOUND, so a correct kernel sits below a
               quarter of the bound.  `python tests/iou_reference.py` repeats that run

On ill-conditioned pairs there is no truth claim: an identical box can overlap itself by half its area, or 0, at KITTI
far range, as in the reference.  Tests pin those values against the reference kernel and across consumers instead.
"""
import numpy as np

U = 2.0 ** -24                # unit roundoff of one fp32 round-to-nearest
MARGIN = 1e-5                 # in_box2d's margin
CORNER_ULPS = 16              # rounding of the rotate-and-unrotate round trip of a corner, in ulps of R
MIN_SIN = 0.02                # edges closer to parallel than this are ill-conditioned ...
EDGE_GAP = 0.02               # ... when their bounding boxes come closer than this (m)
K_BOUND = 2.25                # see the module docstring


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def to_bev(b7):
    """box7_to_bev: [x,y,z,h,w,l,ry] -> [x - l/2, z - w/2, x + l/2, z + w/2, ry], every op one fp32 rounding"""
    b = f32(b7)
    hl, hw = b[:, 5] * np.float32(0.5), b[:, 4] * np.float32(0.5)
    return np.stack([b[:, 0] - hl, b[:, 2] - hw, b[:, 0] + hl, b[:, 2] + hw, b[:, 6]], 1).astype(np.float32)


def corners(bev):
    """(n,5) fp32 BEV boxes -> (n,4,2) float64 corners in the order the kernel builds them"""
    b = f32(bev)
    cx = ((b[:, 0] + b[:, 2]) / np.float32(2)).astype(np.float64)
    cy = ((b[:, 1] + b[:, 3]) / np.float32(2)).astype(np.float64)
    x1, y1, x2, y2, ang = (b[:, k].astype(np.float64) for k in range(5))
    c, s = np.cos(ang), np.sin(ang)
    px = np.stack([x1, x2, x2, x1], 1) - cx[:, None]
    py = np.stack([y1, y1, y2, y2], 1) - cy[:, None]
    return np.stack([px * c[:, None] + py * s[:, None] + cx[:, None], -px * s[:, None] + py * c[:, None] + cy[:, None]], 2)


def _shoelace(p, n):
    """signed area of the first n[r] vertices of each padded polygon p (r, W, 2)"""
    W = p.shape[1]
    j = np.arange(W)[None, :]
    nxt = np.where(j + 1 < n[:, None], j + 1, 0)
    q = np.take_along_axis(p, nxt[..., None], 1)
    t = p[..., 0] * q[..., 1] - p[..., 1] * q[..., 0]
    return 0.5 * np.where(j < n[:, None], t, 0.0).sum(1)


def clip_area(P, Q):
    """(n,4,2), (n,4,2) float64 convex quadrilaterals -> (n,) area of their intersection: Sutherland-Hodgman of P against
    the four edges of Q, vectorised over pairs (padded polygons of up to 16 vertices)"""
    n = P.shape[0]
    W = 16
    Q = np.where((_shoelace(Q, np.full(n, 4)) < 0)[:, None, None], Q[:, ::-1], Q)         # counter-clockwise clip edges
    poly = np.zeros((n, W, 2))
    poly[:, :4] = P
    cnt = np.full(n, 4)
    j = np.arange(W)[None, :]
    rows = np.arange(n)[:, None]
    for e in range(4):
        p0, p1 = Q[:, e], Q[:, (e + 1) % 4]
        ex, ey = (p1 - p0)[:, 0:1], (p1 - p0)[:, 1:2]
        side = ex * (poly[..., 1] - p0[:, 1:2]) - ey * (poly[..., 0] - p0[:, 0:1])
        valid = j < cnt[:, None]
        prev = np.where(j == 0, np.maximum(cnt[:, None] - 1, 0), j - 1)
        sp = np.take_along_axis(side, prev, 1)
        pp = np.take_along_axis(poly, prev[..., None], 1)
        cur_in, prev_in = side >= 0, sp >= 0
        emit_x = valid & (cur_in != prev_in)
        emit_c = valid & cur_in
        with np.errstate(invalid="ignore", divide="ignore"):
            t = np.where(emit_x, sp / (sp - side), 0.0)
        inter = pp + (poly - pp) * t[..., None]
        k = emit_x.astype(np.int64) + emit_c
        start = np.cumsum(k, 1) - k
        cnt = k.sum(1)
        assert cnt.max(initial=0) <= W
        out = np.zeros_like(poly)
        r, c = np.nonzero(emit_x)
        out[r, start[r, c]] = inter[r, c]
        r, c = np.nonzero(emit_c)
        out[r, start[r, c] + emit_x[r, c]] = poly[r, c]
        poly = out
    return np.where(cnt >= 3, np.abs(_shoelace(poly, cnt)), 0.0)


def finite_rows(*boxes):
    ok = np.ones(len(boxes[0]), bool)
    for b in boxes:
        ok &= np.isfinite(b).all(1)
    return ok


def exact_overlap(a_bev, b_bev):
    """(n,5), (n,5) fp32 BEV boxes, aligned pairs -> float64 overlap area; NaN for a pair with a non-finite field"""
    a, b = f32(a_bev), f32(b_bev)
    ok = finite_rows(a, b)
    out = np.full(len(a), np.nan)
    if ok.any():
        out[ok] = clip_area(corners(a[ok]), corners(b[ok]))
    return out


def bev_area(bev):
    b = f32(bev).astype(np.float64)
    return (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])


# ------------------------------------------------------------------------------------------------------ conditioning
def ulp(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


def _corner_distance(C, bev):
    """distance of corners C (n,4,2) to the boundary of the boxes bev (n,5), in the box's frame (in_box2d's rotation)"""
    b = f32(bev)
    cx = ((b[:, 0] + b[:, 2]) / np.float32(2)).astype(np.float64)[:, None]
    cy = ((b[:, 1] + b[:, 3]) / np.float32(2)).astype(np.float64)[:, None]
    ang = b[:, 4].astype(np.float64)[:, None]
    dx, dy = C[..., 0] - cx, C[..., 1] - cy
    u = dx * np.cos(ang) - dy * np.sin(ang)
    v = dx * np.sin(ang) + dy * np.cos(ang)
    lx1, lx2 = b[:, 0:1].astype(np.float64) - cx, b[:, 2:3].astype(np.float64) - cx
    ly1, ly2 = b[:, 1:2].astype(np.float64) - cy, b[:, 3:4].astype(np.float64) - cy
    gx = np.maximum(np.maximum(lx1 - u, u - lx2), 0.0)
    gy = np.maximum(np.maximum(ly1 - v, v - ly2), 0.0)
    inside = np.minimum(np.minimum(u - lx1, lx2 - u), np.minimum(v - ly1, ly2 - v))
    return np.where((gx > 0) | (gy > 0), np.hypot(gx, gy), inside).min(1)


def _edge_min_sin(A, B, tol):
    """smallest |sin| between an edge of A and an edge of B whose bounding boxes (grown by tol) overlap; 1 when none do"""
    ea0, ea1 = A, np.roll(A, -1, 1)
    eb0, eb1 = B, np.roll(B, -1, 1)
    da, db = ea1 - ea0, eb1 - eb0
    lo_a, hi_a = np.minimum(ea0, ea1)[:, :, None], np.maximum(ea0, ea1)[:, :, None]
    lo_b, hi_b = np.minimum(eb0, eb1)[:, None], np.maximum(eb0, eb1)[:, None]
    t = tol[:, None, None, None]
    meet = ((lo_a <= hi_b + t) & (lo_b <= hi_a + t)).all(-1)
    cr = da[:, :, None, 0] * db[:, None, :, 1] - da[:, :, None, 1] * db[:, None, :, 0]
    na, nb = np.hypot(da[..., 0], da[..., 1])[:, :, None], np.hypot(db[..., 0], db[..., 1])[:, None, :]
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.abs(cr) / (na * nb)
    s = np.where(np.isfinite(s), s, 0.0)
    return np.where(meet, s, 1.0).reshape(len(A), -1).min(1)


def conditioning(a_bev, b_bev):
    """per aligned pair: dict(R, corner (smallest corner-to-boundary distance), sin (smallest edge |sin|), degenerate
    (a field not finite or an extent <= 0), ill (bool))"""
    a, b = f32(a_bev), f32(b_bev)
    n = len(a)
    ok = finite_rows(a, b)
    ok &= (a[:, 2] > a[:, 0]) & (a[:, 3] > a[:, 1]) & (b[:, 2] > b[:, 0]) & (b[:, 3] > b[:, 1])
    R = np.full(n, np.inf)
    corner = np.zeros(n)
    sin = np.zeros(n)
    if ok.any():
        A, B = corners(a[ok]), corners(b[ok])
        R[ok] = np.maximum(np.abs(np.concatenate([A, B], 1)).reshape(ok.sum(), -1).max(1), 1.0)
        corner[ok] = np.minimum(_corner_distance(A, b[ok]), _corner_distance(B, a[ok]))
        sin[ok] = _edge_min_sin(A, B, np.full(ok.sum(), EDGE_GAP))
    tol = MARGIN + CORNER_ULPS * ulp(np.where(ok, R, 1.0))
    ill = ~ok | (corner < tol) | (sin < MIN_SIN)
    return dict(R=R, corner=corner, sin=sin, degenerate=~ok, ill=ill)


def bound(a_bev, b_bev, R):
    """the overlap error bound of a well-conditioned pair"""
    a, b = f32(a_bev).astype(np.float64), f32(b_bev).astype(np.float64)
    per = 2 * ((a[:, 2] - a[:, 0]) + (a[:, 3] - a[:, 1]) + (b[:, 2] - b[:, 0]) + (b[:, 3] - b[:, 1]))
    return K_BOUND * U * R * per


def check(got, exact, bnd):
    """-> (ok, max err/bound, number outside)"""
    err = np.abs(np.asarray(got, np.float64) - exact)
    ratio = err / bnd
    return bool((ratio <= 1).all()), float(ratio.max(initial=0.0)), int((ratio > 1).sum())


# ------------------------------------------------------------------------------------------------------ pair families
PLACES = ("near", "far")
# families whose every pair must be classified ill-conditioned
ILL = ("identical", "shifted", "rotated", "flipped", "square90", "shared_edge", "corner", "zero", "nonfinite")
FAMILIES = ("generic", "nested", "pedestrian", "big") + ILL


def _cars(rng, n, place, size=1.0):
    b = np.empty((n, 7))
    if place == "near":
        b[:, 0], b[:, 2] = rng.uniform(-5, 5, n), rng.uniform(0, 10, n)
    elif place == "far":
        b[:, 0], b[:, 2] = rng.uniform(-40, 40, n), rng.uniform(60, 80, n)
    else:                                                   # a 1000 m offset
        b[:, 0], b[:, 2] = rng.uniform(-40, 40, n) + 1000.0, rng.uniform(0, 80, n)
    b[:, 1] = rng.uniform(1.5, 1.9, n)
    b[:, 3] = rng.uniform(1.4, 1.7, n)
    b[:, 4] = rng.uniform(1.5, 1.8, n) * size
    b[:, 5] = rng.uniform(3.5, 4.5, n) * size
    b[:, 6] = rng.uniform(-np.pi, np.pi, n)
    return b


def _q64(x):
    return np.round(np.asarray(x) * 64) / 64                # exact in fp32 at these ranges


def family(name, place, n, seed):
    """n aligned pairs (a, b) of [x,y,z,h,w,l,ry] fp32 boxes of one family at one placement ("near": |x| <= 5 m, z 0-10 m;
    "far": |x| <= 40 m, z 60-80 m; "off1000": x + 1000 m)"""
    rng = np.random.default_rng([seed, FAMILIES.index(name), (PLACES + ("off1000",)).index(place)])
    a = _cars(rng, n, place)
    if name == "generic":
        b = _cars(rng, n, place)
        b[:, 0], b[:, 2] = a[:, 0] + rng.uniform(-3, 3, n), a[:, 2] + rng.uniform(-3, 3, n)
        b[:, 1] = a[:, 1] + rng.uniform(-1, 1, n)
    elif name == "pedestrian":
        a[:, 4], a[:, 5] = rng.uniform(0.25, 0.35, n), rng.uniform(0.25, 0.35, n)
        b = a.copy()
        b[:, 4], b[:, 5] = rng.uniform(0.25, 0.35, n), rng.uniform(0.25, 0.35, n)
        b[:, 0], b[:, 2] = a[:, 0] + rng.uniform(-0.3, 0.3, n), a[:, 2] + rng.uniform(-0.3, 0.3, n)
        b[:, 6] = rng.uniform(-np.pi, np.pi, n)
    elif name == "big":
        a[:, 5], a[:, 4] = 20.0, rng.uniform(2, 4, n)
        b = _cars(rng, n, place, size=1.0)
        b[:, 5], b[:, 4] = rng.choice([20.0, 4.0], n), rng.uniform(2, 4, n)
        b[:, 0], b[:, 2] = a[:, 0] + rng.uniform(-12, 12, n), a[:, 2] + rng.uniform(-4, 4, n)
    elif name == "nested":
        b = a.copy()
        b[:, 4:6] *= rng.uniform(0.3, 0.6, (n, 1))
        b[:, 6] = a[:, 6] + rng.uniform(-0.3, 0.3, n)
    elif name == "identical":
        b = a.copy()
    elif name == "shifted":
        b = a.copy()
        d, phi = 10.0 ** rng.uniform(-7, -2, n), rng.uniform(0, 2 * np.pi, n)
        b[:, 0] += d * np.cos(phi)
        b[:, 2] += d * np.sin(phi)
    elif name == "rotated":
        b = a.copy()
        b[:, 6] += rng.choice([-1, 1], n) * 10.0 ** rng.uniform(-7, -2, n)
    elif name == "flipped":
        b = a.copy()
        b[:, 6] = a[:, 6] + rng.choice([-np.pi, np.pi], n)
    elif name == "square90":
        a[:, 4] = a[:, 5]
        b = a.copy()
        b[:, 6] = a[:, 6] + rng.choice([-np.pi / 2, np.pi / 2], n)
    elif name in ("shared_edge", "corner"):
        a[:, [0, 2, 4, 5]] = _q64(a[:, [0, 2, 4, 5]])
        a[: n // 2, 6] = rng.choice([0.0, np.pi / 2, -np.pi, np.pi], n // 2)
        b = a.copy()
        b[:, 4:6] = _q64(rng.uniform(1.5, 4.5, (n, 2)))
        sx = rng.choice([-1, 1], n) * (a[:, 5] + b[:, 5]) / 2
        sz = rng.choice([-1, 1], n) * (a[:, 4] + b[:, 4]) / 2
        if name == "shared_edge":
            side = rng.random(n) < 0.5                       # along x (the b box slides along the edge) or along z
            sx = np.where(side, sx, _q64(rng.uniform(-1, 1, n)))
            sz = np.where(side, _q64(rng.uniform(-0.5, 0.5, n)), sz)
        c, s = np.cos(a[:, 6]), np.sin(a[:, 6])
        rot = a[:, 6] != 0                                   # a shifted frame: exact only for ry = 0
        b[:, 0] = a[:, 0] + np.where(rot, sx * c + sz * s, sx)
        b[:, 2] = a[:, 2] + np.where(rot, -sx * s + sz * c, sz)
    elif name == "zero":
        b = a.copy()
        b[:, 0] += rng.uniform(-1, 1, n)
        which = rng.integers(0, 4, n)                        # a.w, a.l, b.w, b.l
        for k, (box, col) in enumerate([(a, 4), (a, 5), (b, 4), (b, 5)]):
            box[which == k, col] = 0.0
    elif name == "nonfinite":
        b = a.copy()
        b[:, 0] += rng.uniform(-1, 1, n)
        field = np.arange(n) % 7
        val = np.array([np.nan, np.inf, -np.inf])[(np.arange(n) // 7) % 3]
        on_b = (np.arange(n) // 21) % 2 == 1
        for k in range(n):
            (b if on_b[k] else a)[k, field[k]] = val[k]
    else:
        raise KeyError(name)
    return f32(a), f32(b)


if __name__ == "__main__":
    # the run K_BOUND is chosen from: the oracle on 150000 pairs of each generic family and placement
    import sys
    sys.path.insert(0, __import__("os").path.join(__import__("os").path.dirname(__file__), ".."))
    from oracle import oracle as O
    worst, nwell = 0.0, 0
    for f, p in [(f, p) for f in ("generic", "nested", "pedestrian", "big") for p in PLACES] + [("generic", "off1000")]:
        a, b = (to_bev(x) for x in family(f, p, 150000, 12345))
        got, _ = O.box_overlap_pairs(a, b)
        c = conditioning(a, b)
        w = ~c["ill"]
        k = np.abs(got[w] - exact_overlap(a, b)[w]) / (bound(a[w], b[w], c["R"][w]) / K_BOUND)
        nwell, worst = nwell + int(w.sum()), max(worst, float(k.max()))
        print("%-10s %-8s %7d well-conditioned pairs, largest err / (U R P) %.4f" % (f, p, w.sum(), k.max()))
    print("%d pairs: largest %.4f = %.3f of K_BOUND" % (nwell, worst, worst / K_BOUND))

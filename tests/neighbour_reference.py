"""Adversarial point clouds for the index kernels (FPS, ball query, 3-NN) and float64 checks of their selections.

Every generator is seeded and returns float32 arrays.  A family is built to land on one kind of decision the
kernels prune or dispatch on:
  lidar      a ray-cast 64-beam scan (ground plane, boxes, a wall): dense near field, planes, regular rings
  shell      points at fl(d2) == fl(r*r), and at the fp32 neighbours of that value, for every network radius
  cell_edge  centres and points on the hash-grid cell boundaries k*h and one fp32 ulp either side
  caps       clusters sized to the grid's dispatch limits (bitonic / ranking switch, candidate cap, walk cap, nsample)
  ties       integer lattices, a sphere of equal distances around point 0, duplicate stacks
  far/flat   clouds offset by 3e4 or 1e6, a zero-extent axis, collinear points
  nonfinite  a few NaN / inf coordinates among points (and centres)
Boundary placements are certified with the oracle's own distance (oracle.dist2, the reference's FMA order): numpy has
no fused multiply-add, so it cannot say on which side of r an fp32 distance lands.
"""
import numpy as np

from oracle import oracle as O

RPN_RADII = ((0.1, 0.5), (0.5, 1.0), (1.0, 2.0), (2.0, 4.0))
RPN_NSAMPLE = (16, 32)
RPN_NPOINTS = (4096, 1024, 256, 64)
RCNN_RADII = (0.2, 0.4)
RCNN_NSAMPLE = 64
ALL_RADII = (0.1, 0.2, 0.4, 0.5, 1.0, 2.0, 4.0)
SCOPE_LO = np.array([-40.0, -1.0, 0.0])
SCOPE_HI = np.array([40.0, 3.0, 70.4])
F32 = np.float32


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def ulp_steps(v, k):
    """v moved by k fp32 ulps (k may be negative), elementwise, for finite v"""
    i = _f32(v).view(np.int32).astype(np.int64)
    key = np.where(i >= 0, i, -(i & 0x7fffffff)) + np.asarray(k, dtype=np.int64)
    return np.where(key >= 0, key, (-key) | 0x80000000).astype(np.uint32).view(np.float32)


def bq_cell(rmax):
    """cell edge of the ball-query grid, computed as the host computes it"""
    return float(np.float32(rmax)) * 1.0001


def nn_cell(known, factor=1.6):
    """cell edge of the 3-NN grid of one scene (n, 3): factor * cbrt(volume / n) over the finite bounding box"""
    k = np.asarray(known, dtype=np.float32)
    fin = np.isfinite(k)
    ext = []
    for a in range(3):
        v = k[fin[:, a], a]
        ext.append(float(v.max()) - float(v.min()) if v.size else 0.0)
    emax = max(ext)
    if not emax > 0:
        emax = 1.0
    vol = 1.0
    for e in ext:
        vol *= max(e, emax * 0.02)
    return max(factor * np.cbrt(vol / max(len(k), 1)), emax * 1e-4)


# ------------------------------------------------------------------------------------------------ lidar
def _ray_boxes(o, d, boxes):
    """nearest positive hit parameter of rays (o + t d) with axis-aligned boxes (lo, hi); inf where none"""
    best = np.full(d.shape[0], np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        for lo, hi in boxes:
            t1 = (np.asarray(lo)[None] - o) / d
            t2 = (np.asarray(hi)[None] - o) / d
            tn = np.nanmax(np.minimum(t1, t2), axis=1)
            tf = np.nanmin(np.maximum(t1, t2), axis=1)
            hit = (tf >= tn) & (tf > 0)
            t = np.where(tn > 0, tn, tf)
            best = np.where(hit & (t < best), t, best)
    return best


def lidar_scan(seed, height=1.7):
    """all returns of one scan of a 64-beam scanner at `height` above the ground, in rect coordinates (x right, y down,
    z forward), inside PC_AREA_SCOPE and the camera's 90 degree field of view"""
    rng = np.random.default_rng(seed)
    el = np.deg2rad(np.linspace(2.0, -24.8, 64))
    az = np.deg2rad(np.arange(-45.0, 45.0, 0.08) + rng.uniform(0, 0.08))
    E, A = np.meshgrid(el, az, indexing="ij")
    d = np.stack([np.cos(E) * np.sin(A), -np.sin(E), np.cos(E) * np.cos(A)], axis=-1).reshape(-1, 3)
    o = np.zeros(3)
    t = np.full(d.shape[0], np.inf)
    with np.errstate(divide="ignore"):
        tg = np.where(d[:, 1] > 0, height / d[:, 1], np.inf)                 # ground plane y = +height
    t = np.minimum(t, tg)
    boxes = []
    for _ in range(rng.integers(5, 9)):                                       # cars / vans standing on the ground
        cx, cz = rng.uniform(-20, 20), rng.uniform(4, 50)
        w, l, h = rng.uniform(1.5, 2.2), rng.uniform(3.5, 6.0), rng.uniform(1.4, 2.6)
        boxes.append(((cx - w / 2, height - h, cz - l / 2), (cx + w / 2, height, cz + l / 2)))
    wx = rng.uniform(8, 15) * rng.choice([-1, 1])                              # a wall along the road
    boxes.append(((wx, height - 4.0, 0.0), (wx + 0.3 * np.sign(wx), height, 80.0)))
    t = np.minimum(t, _ray_boxes(o, d, boxes))
    ok = np.isfinite(t)
    r = t[ok] * (1.0 + rng.normal(0, 2e-4, ok.sum()))                         # range noise
    pts = d[ok] * r[:, None]
    keep = np.all((pts >= SCOPE_LO) & (pts <= SCOPE_HI), axis=1)
    return pts[keep]


def lidar(n, seed):
    """(n, 3) float32: a scan subsampled as the dataset does it (every point at depth >= 40 m, then random near ones)"""
    rng = np.random.default_rng(seed + 1)
    pts = lidar_scan(seed)
    depth = pts[:, 2]
    far, near = np.where(depth >= 40.0)[0], np.where(depth < 40.0)[0]
    if n <= len(pts):
        take = np.concatenate([far, rng.choice(near, n - len(far), replace=False)]) if len(far) < n else rng.choice(far, n, replace=False)
    else:
        take = np.concatenate([np.arange(len(pts)), rng.choice(len(pts), n - len(pts), replace=True)])
    rng.shuffle(take)
    return _f32(pts[take])


def _assemble(special, n, seed, avoid=None, reach=0.0):
    """special points (k, 3) + scan points up to n, shuffled so that index order is unrelated to placement; scan points
    within `reach` of any `avoid` point are dropped (the gaps are refilled far below the scene).  Returns the cloud and
    where each special point went"""
    rng = np.random.default_rng(seed + 99)
    special = _f32(special)
    k = len(special)
    assert k <= n, (k, n)
    fill = lidar(n, seed)
    if avoid is not None:
        dmin = np.min(np.linalg.norm(fill[:, None, :].astype(np.float64) - np.asarray(avoid, np.float64)[None], axis=2), axis=1)
        fill = fill[dmin > reach]
        pad = n - len(fill)
        fill = np.concatenate([fill, _f32(np.array([0.0, -60.0, 0.0]) + rng.uniform(-40, 40, (pad, 3)))])
    cloud = np.concatenate([special, fill[: n - k]])
    perm = rng.permutation(n)
    out = np.empty_like(cloud)
    out[perm] = cloud
    return _f32(out), perm[:k]


# ------------------------------------------------------------------------------------------------ shell
def place_at(centre, dirs, target):
    """points p = centre + dir * s with O.dist2(centre, p) == target exactly, searched over fp32 ulp steps of the
    component with the finest fp32 spacing; returns (points, ok mask).  Exact hits need one fine component: a centre
    coordinate near zero on an axis the direction uses"""
    centre = _f32(centre)
    dirs = np.asarray(dirs, dtype=np.float64)
    dirs = dirs / np.linalg.norm(dirs, axis=1, keepdims=True)
    base = _f32(centre[None].astype(np.float64) + dirs * np.sqrt(float(target)))
    steps = np.arange(-64, 65)
    cand = np.repeat(base[:, None, :], len(steps), axis=1).copy()
    ax = np.argmin(np.where(np.abs(dirs) > 1e-3, np.abs(base), np.inf), axis=1)
    for i in range(len(base)):
        cand[i, :, ax[i]] = ulp_steps(np.full(len(steps), base[i, ax[i]]), steps)
    d = O.dist2(np.broadcast_to(centre, cand.shape), cand)
    hit = d == F32(target)
    ok = hit.any(axis=1)
    first = np.argmax(hit, axis=1)
    return _f32(cand[np.arange(len(base)), first]), ok


def _shell_dirs(rng, n2, n3):
    one = np.concatenate([np.eye(3)[:2], -np.eye(3)[:2]])            # x and y: the fine axes at the centre
    two = np.zeros((n2, 3))
    for i in range(n2):
        a, b = (0, 1) if i % 2 == 0 else (int(rng.integers(0, 2)), 2)
        two[i, a], two[i, b] = rng.uniform(0.3, 1.0) * rng.choice([-1, 1]), rng.uniform(0.3, 1.0) * rng.choice([-1, 1])
    three = rng.uniform(0.3, 1.0, (n3, 3)) * rng.choice([-1, 1], (n3, 3))
    return np.concatenate([one, two, three])


def shell(n, seed, radii=ALL_RADII, n2=4, n3=4):
    """one centre per radius, far from the filler; around it points at fl(d2) == prev(r2), r2 and next(r2), along one,
    two and three axes.  Returns (cloud (n,3), centres (len(radii),3), placements) where placements is a list of
    (point index, centre row, radius, level in {-1, 0, +1}, axes)"""
    rng = np.random.default_rng(seed)
    special, meta, centres = [], [], []
    for ci, r in enumerate(radii):
        c = _f32([0.0, 0.0, 6.0 + 10.0 * ci + rng.uniform(0, 0.5)])  # x = y = 0: fine fp32 spacing around the centre
        centres.append(c)
        r2 = F32(r) * F32(r)
        dirs = _shell_dirs(rng, n2, n3)
        axes = np.count_nonzero(dirs, axis=1)
        for level in (-1, 0, 1):
            target = ulp_steps(np.array([r2]), level)[0]
            pts, ok = place_at(c, dirs, target)
            for p, a in zip(pts[ok], axes[ok]):
                special.append(p)
                meta.append((ci, float(r), level, int(a)))
        for a in (0, 1):                                         # one axis: the fp32 neighbours of r itself
            for s in (-1.0, 1.0):
                for k in (-1, 1):
                    p = c.copy()
                    p[a] = F32(s) * ulp_steps(np.array([F32(r)]), k)[0]
                    d = O.dist2(c, p)
                    special.append(p)
                    meta.append((ci, float(r), int(np.sign(d - r2)), 1))
    cloud, where = _assemble(np.array(special), n, seed, avoid=centres, reach=4.5)
    placements = [(int(w),) + m for w, m in zip(where, meta)]
    return cloud, _f32(centres), placements


# ------------------------------------------------------------------------------------------------ cell edges
def cell_edge(n, seed, rmax=0.5, radii=None):
    """centres on ball-query cell boundaries k*h (h = rmax * 1.0001 as the host computes it) and one fp32 ulp either side,
    each with points just inside its radius along every axis and points on the neighbouring cell boundaries"""
    rng = np.random.default_rng(seed)
    h = bq_cell(rmax)
    r = F32(min(radii) if radii else rmax)
    special, centres = [], []
    for i in range(24):
        k = np.array([rng.integers(-30, 30), rng.integers(20, 40), rng.integers(5, 60)]) * (int(np.ceil(3 / h)) + 1)
        base = _f32(k * h)
        off = _f32([(i % 3) - 1, ((i // 3) % 3) - 1, 0])
        c = ulp_steps(base, off.astype(int))
        centres.append(c)
        for a in range(3):
            for s in (-1, 1):
                for rad in ((F32(rmax), r) if radii else (F32(rmax),)):
                    for back in (1, 2, 3):                        # just inside the radius: largest fp32 offsets below it
                        p = c.copy()
                        p[a] = ulp_steps(np.array([c[a] + s * rad]), -s * back)[0]
                        special.append(p)
                p = c.copy()
                for j in (1, 2):                                  # on the next cell boundaries, one ulp either side
                    e = F32(c[a] + s * j * h)
                    for u in (-1, 0, 1):
                        q = c.copy()
                        q[a] = ulp_steps(np.array([e]), u)[0]
                        special.append(q)
    cloud, _ = _assemble(np.array(special), n, seed, avoid=centres, reach=max(rmax, 1.0) * 3.5)
    return cloud, _f32(centres)


def nn_cell_edge(n, m, seed):
    """(unknown (n,3), known (m,3)) for the 3-NN grid: queries on the cell boundaries of the grid the known cloud
    defines, and pockets where the third neighbour sits at the certification radius (0.9999 h) +- fp32 ulps"""
    rng = np.random.default_rng(seed)
    known = _f32(SCOPE_LO + (SCOPE_HI - SCOPE_LO) * rng.random((m, 3)))
    known[0], known[1] = SCOPE_LO, SCOPE_HI                      # pin the bounding box, so h is known here
    h = nn_cell(known)
    hb = F32(F32(h) * F32(0.9999))
    cert = F32(hb * hb)
    pockets = []
    for i in range(6):                                           # x = y = 0: fine fp32 spacing for the placements
        pockets.append(_f32([0.0, 0.0, 10.0 + 10.0 * i]))
    pockets = _f32(pockets)
    far_from = np.min(np.linalg.norm(known[:, None, :].astype(np.float64) - pockets[None], axis=2), axis=1) > 2.5 * h
    far_from[:2] = True
    known = known[far_from]
    probe = []
    for i, c in enumerate(pockets):
        dirs = np.array([[1.0, 0, 0], [0, 1.0, 0], [-1.0, 0, 0], [0, -1.0, 0], [1.0, 1.0, 0], [-1.0, 0.5, 1.0]])
        lv, way = (i % 3) - 1, 1 if i % 3 == 2 else -1
        for level in (lv, lv + way, lv + 2 * way, lv + 3 * way):  # the nearest reachable fp32 value on that side
            pts, ok = place_at(c, dirs, ulp_steps(np.array([cert]), level)[0])
            if ok.sum() >= 3:
                break
        probe.append(pts[ok][:3])
        out = c.copy()
        out[0] = F32(c[0] - 1.0001 * h)                          # just beyond the block on the low side
        probe.append(out[None])
    probe = np.concatenate(probe)
    known = np.concatenate([known[:2], probe, known[2:]])
    extra = m - len(known)
    filler = _f32(SCOPE_LO + (SCOPE_HI - SCOPE_LO) * rng.random((4 * extra + 16, 3)))
    ok = np.min(np.linalg.norm(filler[:, None, :].astype(np.float64) - pockets[None], axis=2), axis=1) > 2.5 * h
    known = _f32(np.concatenate([known, filler[ok][:extra]]))[:m]
    assert len(known) == m
    q = []
    for c in pockets:
        q.append(c)
    for i in range(256):                                          # queries on cell boundaries
        kc = np.floor(known[rng.integers(2, m)].astype(np.float64) / h)
        base = _f32(kc * h)
        q.append(ulp_steps(base, rng.integers(-1, 2, 3)))
    q = _f32(q)
    unknown = np.concatenate([q, _f32(SCOPE_LO + (SCOPE_HI - SCOPE_LO) * rng.random((n - len(q), 3)))])
    return _f32(unknown), known, len(pockets)


def nn_stack(n, m, seed, stack=2100, k=8):
    """(unknown (n,3), known (m,3), k) for the 3-NN grid's walk cap: the known bounding box pinned to the scope, so h is
    known here, and `stack` known points in the middle of one cell, more than the 2048 nodes a query walks before it
    leaves itself to the exhaustive scan; the first k queries sit in that cell"""
    rng = np.random.default_rng(seed)
    known = _f32(SCOPE_LO + (SCOPE_HI - SCOPE_LO) * rng.random((m, 3)))
    known[0], known[1] = SCOPE_LO, SCOPE_HI
    h = nn_cell(known)
    centre = (np.floor(np.array([1.0, 1.0, 30.0]) / h) + 0.5) * h
    known[2:2 + stack] = _f32(centre + rng.uniform(-0.3, 0.3, (stack, 3)) * h)
    known = known[np.concatenate([[0, 1], 2 + rng.permutation(m - 2)])]
    q = _f32(centre + rng.uniform(-0.3, 0.3, (k, 3)) * h)
    unknown = np.concatenate([q, _f32(SCOPE_LO + (SCOPE_HI - SCOPE_LO) * rng.random((n - k, 3)))])
    return _f32(unknown), _f32(known), k


# ------------------------------------------------------------------------------------------------ caps
CAP_SIZES = (15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200)


def caps(n, seed, radii=(0.1, 0.5)):
    """one centre per cluster size: `size` points strictly inside the smaller radius (so inside both), nothing else in
    reach; plus a centre with a 600-point stack in a corner cell of its 3x3x3 block (outside the radius) that overflows
    the list walk's cap of 512 nodes.  Returns (cloud, centres, sizes) with size -1 for the stack centre"""
    rng = np.random.default_rng(seed)
    r0, rmax = min(radii), max(radii)
    h = bq_cell(rmax)
    special, centres, sizes = [], [], []
    sp = 3.0 * rmax + 4 * h + 1.0
    for i, size in enumerate(CAP_SIZES + (-1,)):
        c = _f32([-35.0 + sp * (i % 8), 25.0 + sp * (i // 8), 30.0])
        centres.append(c)
        sizes.append(size)
        if size > 0:
            u = rng.normal(size=(size, 3))
            u /= np.linalg.norm(u, axis=1, keepdims=True)
            special.append(_f32(c + u * (0.8 * r0) * rng.random((size, 1)) ** (1 / 3)))
        else:
            corner = (np.floor(c.astype(np.float64) / h) + 1.5) * h
            special.append(_f32(corner + rng.uniform(-0.3, 0.3, (600, 3)) * h))
    cloud, _ = _assemble(np.concatenate(special), n, seed, avoid=centres, reach=3 * h + rmax)
    return cloud, _f32(centres), sizes


# ------------------------------------------------------------------------------------------------ ties
def ties(n, seed, spacing=1.0):
    """point 0 at the origin, an integer lattice (every distance an exact small integer), a sphere of points at the same
    fp32 distance 5 from point 0 (integer triples with x^2+y^2+z^2 = 25) and stacks of duplicates"""
    rng = np.random.default_rng(seed)
    k = int(np.ceil((0.8 * n) ** (1 / 3)))
    g = np.arange(k) - k // 2
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.float64) * spacing
    lat = lat[np.any(lat != 0, axis=1)]
    trip = [(x, y, z) for x in range(-5, 6) for y in range(-5, 6) for z in range(-5, 6) if x * x + y * y + z * z == 25]
    sphere = np.array(trip, dtype=np.float64) * spacing + np.array([0.5, 0.5, 0.5]) * spacing * k
    rest = n - 1 - len(sphere)
    nl = min(len(lat), int(rest * 0.85))
    lat = lat[rng.permutation(len(lat))[:nl]]
    dups = lat[rng.integers(0, nl, rest - nl)]
    body = np.concatenate([lat, dups, sphere])
    body = body[rng.permutation(len(body))]
    return _f32(np.concatenate([np.zeros((1, 3)), body]))


def sphere_around_zero(n, seed):
    """point 0 and every other point at one fp32 distance from it: the first pick after point 0 is a tie of n - 1"""
    trip = np.array([(x, y, z) for x in range(-13, 14) for y in range(-13, 14) for z in range(-13, 14)
                     if x * x + y * y + z * z == 169], dtype=np.float64)
    rng = np.random.default_rng(seed)
    pts = trip[rng.integers(0, len(trip), n - 1)]
    return _f32(np.concatenate([np.zeros((1, 3)), pts]))


# ------------------------------------------------------------------------------------------------ conditioning
def far(n, seed, offset):
    return _f32(lidar(n, seed).astype(np.float64) + offset)


def flat(n, seed):
    """the scan with every y on one value: one axis of zero extent"""
    p = lidar(n, seed)
    p[:, 1] = F32(1.7)
    return p


def collinear(n, seed):
    rng = np.random.default_rng(seed)
    t = _f32(rng.uniform(0, 60, n))
    return _f32(np.stack([t * F32(0.5) - F32(15), np.full(n, F32(1.0)), t], axis=1))


def nonfinite(n, seed, count=12):
    """the scan with a few NaN / +-inf coordinates; point 0 stays finite"""
    rng = np.random.default_rng(seed)
    p = lidar(n, seed)
    where = rng.choice(np.arange(1, n), 3 * count, replace=False)
    p[where[:count], rng.integers(0, 3, count)] = np.nan
    p[where[count:2 * count], rng.integers(0, 3, count)] = np.inf
    p[where[2 * count:], :] = -np.inf
    return p


# ------------------------------------------------------------------------------------------------ float64 checks
def _d64(c, p):
    return np.sum((np.asarray(p, np.float64) - np.asarray(c, np.float64)) ** 2, axis=-1)


REL_BAND = 2.0 ** -19      # a few fp32 ulps: the FMA distance of fp32 differences is within ~5 * 2^-24 of the true one


def ball_query_f64_violations(xyz, centres, r, ns, idx):
    """number of centres whose oracle selection `idx` (m, ns) disagrees with float64 distances outside the band: a listed
    hit that is surely out, a skipped point (before the last listed hit, or anywhere when fewer than ns were found) that
    is surely in, hits not in index order"""
    r2 = float(F32(r) * F32(r))
    bad = 0
    for j in range(len(centres)):
        d = _d64(centres[j], xyz)
        with np.errstate(invalid="ignore"):
            sure_in = d < r2 * (1 - REL_BAND)
            sure_out = ~(d <= r2 * (1 + REL_BAND))
        row = idx[j]
        hits = [int(row[0])]
        for v in row[1:]:
            if v <= hits[-1]:
                break
            hits.append(int(v))
        if not np.any(~sure_out[hits]) and not sure_in.any() and len(set(row.tolist())) == 1 and row[0] == 0:
            continue                                              # no hit at all: the row stays zero
        if sure_out[hits].any():
            bad += 1
            continue
        end = hits[-1] + 1 if len(hits) == ns else len(xyz)
        missing = np.where(sure_in[:end])[0]
        if not set(missing.tolist()) <= set(hits):
            bad += 1
    return bad


def three_nn_f64_violations(unknown, known, idx):
    """number of queries whose three listed neighbours are not the three nearest in float64 outside the band, or are
    not listed in ascending distance"""
    bad = 0
    for j in range(len(unknown)):
        if not np.all(np.isfinite(unknown[j])):
            continue
        d = _d64(unknown[j], known)
        d = np.where(np.isfinite(d), d, np.inf)
        sel = d[idx[j]]
        rest = np.delete(d, idx[j])
        tol = REL_BAND * max(sel.max(), 1e-30)
        if rest.size and sel.max() > rest.min() + tol:
            bad += 1
        elif sel[0] > sel[1] + tol or sel[1] > sel[2] + tol:
            bad += 1
    return bad


# ------------------------------------------------------------------------------------------------ restatements
def fps_replay(xyz, m, larger_rank_wins=False):
    """FPS of one scene with the oracle's distance, ties settled by the reference rank rule (smaller rank wins), or by
    the opposite rule.  Returns (idx, ties) where ties[j] = number of points at the maximum in round j"""
    xyz = _f32(xyz)
    n = len(xyz)
    S = O.opt_n_threads(n)
    logS = S.bit_length() - 1
    Q = -(-n // S)
    k = np.arange(n)
    t = k & (S - 1)
    rev = np.array([int(format(v, "0%db" % logS)[::-1], 2) if logS else 0 for v in range(S)])
    rank = rev[t] * Q + (k >> logS)
    temp = np.full(n, F32(1e10), dtype=np.float32)
    idx, nties = [0], [1]
    old = 0
    for _ in range(1, m):
        d = O.dist2(xyz, np.broadcast_to(xyz[old], xyz.shape))
        temp = np.fmin(temp, d)
        mx = temp.max()
        at = np.where(temp == mx)[0]
        old = int(at[np.argmax(rank[at])] if larger_rank_wins else at[np.argmin(rank[at])])
        idx.append(old)
        nties.append(len(at))
    return np.array(idx, dtype=np.int32), np.array(nties)


def ball_query_np(xyz, centres, r, ns, strict=True, fused=True):
    """brute-force ball query of one scene: `strict` False uses <=, `fused` False the unfused dx*dx + dy*dy + dz*dz"""
    xyz, centres = _f32(xyz), _f32(centres)
    r2 = F32(r) * F32(r)
    out = np.zeros((len(centres), ns), dtype=np.int32)
    for j, c in enumerate(centres):
        if fused:
            d = O.dist2(np.broadcast_to(c, xyz.shape), xyz)
        else:
            e = (c[None] - xyz).astype(np.float32)
            d = ((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]).astype(np.float32) + e[:, 2] * e[:, 2]).astype(np.float32)
        with np.errstate(invalid="ignore"):
            hit = np.where(d < r2 if strict else d <= r2)[0][:ns]
        if len(hit):
            out[j, :] = hit[0]
            out[j, : len(hit)] = hit
    return out


def _cells(p, h):
    with np.errstate(invalid="ignore"):
        c = np.floor(np.asarray(p, np.float64) * (1.0 / h))
    return np.where(np.isfinite(c), c, 0).astype(np.int64)


def ball_query_grid_np(xyz, centres, r, ns, h):
    """ball query restricted to the 3x3x3 block of cells of edge h around each centre (the grid kernels' candidates)"""
    xyz, centres = _f32(xyz), _f32(centres)
    r2 = F32(r) * F32(r)
    pc, cc = _cells(xyz, h), _cells(centres, h)
    out = np.zeros((len(centres), ns), dtype=np.int32)
    for j, c in enumerate(centres):
        near = np.all(np.abs(pc - cc[j]) <= 1, axis=1)
        d = O.dist2(np.broadcast_to(c, xyz.shape), xyz)
        with np.errstate(invalid="ignore"):
            hit = np.where(near & (d < r2))[0][:ns]
        if len(hit):
            out[j, :] = hit[0]
            out[j, : len(hit)] = hit
    return out


def three_nn_grid_np(unknown, known, cert=0.9999, factor=1.6):
    """3-NN through the grid of the kernels: the lexicographic top 3 of the 3x3x3 block, accepted when the third distance
    is below (cert * h)^2 in fp32, else the exhaustive answer.  Returns (dist2, idx, certified mask)"""
    unknown, known = _f32(unknown), _f32(known)
    h = nn_cell(known, factor)
    hb = F32(F32(h) * F32(cert))
    lim = F32(hb * hb)
    kc, qc = _cells(known, h), _cells(unknown, h)
    d_all, i_all = O.three_nn(unknown[None], known[None])
    d_out, i_out = d_all[0].copy(), i_all[0].copy()
    certified = np.zeros(len(unknown), bool)
    for j, q in enumerate(unknown):
        near = np.where(np.all(np.abs(kc - qc[j]) <= 1, axis=1))[0]
        if len(near) < 3:
            continue
        d = O.dist2(np.broadcast_to(q, (len(near), 3)), known[near])
        order = np.lexsort((near, d))[:3]
        b3 = d[order[2]]
        if b3 < lim:
            certified[j] = True
            d_out[j], i_out[j] = d[order], near[order]
    return d_out, i_out, certified

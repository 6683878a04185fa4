"""oracle/kitti_eval.py -- CPU restatement (numpy) of the KITTI AP evaluation, tools/kitti_object_eval_python/eval.py.
TEST INFRASTRUCTURE ONLY: imported by tests/ and scripts/, never by pointrcnn_b200/.

Follows (reference eval.py:line), restated rather than transcribed: the matching loops are vectorised over images,
thresholds and detections, with the GT loop kept sequential.
  overlaps        calculate_iou_partly :335-409 (image_box_overlap :85-111, rotate_iou_gpu_eval, d3_box_overlap :120-152); the
                  rotated BEV intersection is oracle/gt_paste.py::clip_area's exact float64 clip of the fp32 boxes
  clean           clean_data :28-81
  statistics      compute_statistics_jit :156-273 (pass 1 without, pass 2 with compute_fp), fused_compute_statistics :285-332
  thresholds      get_thresholds :8-25
  evaluate        eval_class :443-548, do_eval :567-587, get_official_eval_result :608-678
Pinned by tests/golden/kitti_eval.npz, which the reference's own evaluator produced (oracle/make_golden_kitti_eval.py).
Unlike the reference it evaluates any number of images (the reference needs at least 50).
"""
import numpy as np

from oracle.gt_paste import clip_area

CLASS_TO_NAME = {0: "Car", 1: "Pedestrian", 2: "Cyclist", 3: "Van", 4: "Person_sitting"}
MIN_OVERLAPS = np.array([[[0.7, 0.5, 0.5, 0.7, 0.5]] * 3,
                         [[0.7, 0.5, 0.5, 0.7, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25], [0.5, 0.25, 0.25, 0.5, 0.25]]])
MIN_HEIGHT, MAX_OCCLUSION, MAX_TRUNCATION = (40, 25, 25), (0, 1, 2), (0.15, 0.3, 0.5)
NEIGHBOUR = {0: "van", 1: "person_sitting"}
N_PTS = 41


# ------------------------------------------------------------------------------------------------ overlaps
def image_iou(a, b, union=True):
    """(n,4), (k,4) float64 -> (n,k): intersection over union, or over a's area (union=False)"""
    iw = np.minimum(a[:, None, 2], b[None, :, 2]) - np.maximum(a[:, None, 0], b[None, :, 0])
    ih = np.minimum(a[:, None, 3], b[None, :, 3]) - np.maximum(a[:, None, 1], b[None, :, 1])
    area_a = ((a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1]))[:, None]
    area_b = ((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1]))[None, :]
    inter = iw * ih
    with np.errstate(divide="ignore", invalid="ignore"):
        r = inter / ((area_a + area_b - inter) if union else area_a + 0 * area_b)
    return np.where((iw > 0) & (ih > 0), r, 0.0)


def bev_corners(x, z, l, w, ry):
    """corners of (x, z, l, w, ry) boxes (float64 of the fp32 values), rotated as rotate_iou's rbbox_to_corners"""
    dx = np.stack([-l, -l, l, l], 1) / 2
    dy = np.stack([-w, w, w, -w], 1) / 2
    c, s = np.cos(ry)[:, None], np.sin(ry)[:, None]
    return np.stack([c * dx + s * dy + x[:, None], -s * dx + c * dy + z[:, None]], 2)


def overlaps(dt, gt):
    """-> (3, nd, ng) float64: image-box IoU (double), BEV IoU (fp32), 3D IoU (fp32) of one image"""
    nd, ng = len(dt["name"]), len(gt["name"])
    out = np.zeros((3, nd, ng))
    if nd == 0 or ng == 0:
        return out
    out[0] = image_iou(np.asarray(dt["bbox"], np.float64), np.asarray(gt["bbox"], np.float64))

    def bev(a):
        f = lambda v: np.asarray(v, np.float32).astype(np.float64)
        loc, dim = np.asarray(a["location"]), np.asarray(a["dimensions"])
        x, z, l, w, ry = f(loc[:, 0]), f(loc[:, 2]), f(dim[:, 0]), f(dim[:, 2]), f(a["rotation_y"])
        return bev_corners(x, z, l, w, ry), np.float32(l) * np.float32(w), np.stack([x, z], 1), np.hypot(l, w) / 2
    cd, area_d, cen_d, rad_d = bev(dt)
    cg, area_g, cen_g, rad_g = bev(gt)
    near = np.linalg.norm(cen_d[:, None] - cen_g[None], axis=2) < (rad_d[:, None] + rad_g[None]) * 1.001 + 1e-6
    yd, hd = np.asarray(dt["location"], np.float64)[:, 1], np.asarray(dt["dimensions"], np.float64)[:, 1]
    yg, hg = np.asarray(gt["location"], np.float64)[:, 1], np.asarray(gt["dimensions"], np.float64)[:, 1]
    vol = lambda a: np.asarray(a["dimensions"], np.float64).prod(1)
    vd, vg = vol(dt), vol(gt)
    for j, i in zip(*np.nonzero(near)):
        inter = np.float32(clip_area(cd[j], cg[i]))
        if inter <= 0:
            continue
        out[1, j, i] = inter / (area_g[i] + area_d[j] - inter)
        iw = min(yd[j], yg[i]) - max(yd[j] - hd[j], yg[i] - hg[i])
        if iw > 0:
            inc = iw * np.float64(inter)
            out[2, j, i] = np.float32(inc / (vd[j] + vg[i] - inc))
    return out


# ------------------------------------------------------------------------------------------------ clean
def clean(gt, dt, cls, diff):
    """-> ignored_gt (ng) in {0, 1, -1}, ignored_dt (nd) in {0, 1, -1}, DontCare boxes (n,4), valid GT count"""
    name = CLASS_TO_NAME[cls].lower()
    gname = np.array([str(n).lower() for n in gt["name"]], dtype=object)
    gbox = np.asarray(gt["bbox"], np.float64).reshape(-1, 4)
    hard = (np.asarray(gt["occluded"], np.float64) > MAX_OCCLUSION[diff]) | (np.asarray(gt["truncated"], np.float64) > MAX_TRUNCATION[diff]) | \
        (gbox[:, 3] - gbox[:, 1] <= MIN_HEIGHT[diff])
    same = gname == name
    neighbour = gname == NEIGHBOUR.get(cls, "")
    ig_gt = np.where(same & ~hard, 0, np.where(neighbour | same, 1, -1)).astype(np.int64)
    dc = gbox[np.array([n == "DontCare" for n in gt["name"]], bool)] if len(gbox) else np.zeros((0, 4))
    dbox = np.asarray(dt["bbox"], np.float64).reshape(-1, 4)
    dsame = np.array([str(n).lower() == name for n in dt["name"]], bool)
    ig_dt = np.where(np.abs(dbox[:, 3] - dbox[:, 1]) < MIN_HEIGHT[diff], 1, np.where(dsame, 0, -1)).astype(np.int64)
    return ig_gt, ig_dt, dc, int((ig_gt == 0).sum())


# ------------------------------------------------------------------------------------------------ statistics
def _pad(rows, width, fill, dtype):
    out = np.full((len(rows), width), fill, dtype)
    for k, r in enumerate(rows):
        out[k, :len(r)] = r
    return out


class _Split:
    """one (class, difficulty) of the whole split, padded to (images, max dt, max gt)"""

    def __init__(self, gt_annos, dt_annos, ovs, cls, diff):
        cl = [clean(g, d, cls, diff) for g, d in zip(gt_annos, dt_annos)]
        self.nvalid = sum(c[3] for c in cl)
        nd = max([len(d["name"]) for d in dt_annos] + [1])
        ng = max([len(g["name"]) for g in gt_annos] + [1])
        self.ig_gt = _pad([c[0] for c in cl], ng, -1, np.int64)
        self.ig_dt = _pad([c[1] for c in cl], nd, -1, np.int64)
        self.score = _pad([np.asarray(d["score"], np.float64) for d in dt_annos], nd, 0.0, np.float64)
        self.dt_alpha = _pad([np.asarray(d["alpha"], np.float64) for d in dt_annos], nd, 0.0, np.float64)
        self.gt_alpha = _pad([np.asarray(g["alpha"], np.float64) for g in gt_annos], ng, 0.0, np.float64)
        self.ov = np.zeros((3, len(gt_annos), nd, ng))
        for k, o in enumerate(ovs):
            self.ov[:, k, :o.shape[1], :o.shape[2]] = o
        # per detection: intersection over its own area with each DontCare box (criterion 0), the max over the boxes
        self.dc_ov = np.zeros((len(gt_annos), nd))
        for k, (d, c) in enumerate(zip(dt_annos, cl)):
            if len(c[2]) and len(d["name"]):
                self.dc_ov[k, :len(d["name"])] = image_iou(np.asarray(d["bbox"], np.float64), c[2], union=False).max(1)

    def tp_scores(self, metric, mo):
        """pass 1: per GT in order, the highest-scoring unassigned candidate (overlap > mo) wins, the first on ties"""
        n_img, nd = self.ig_dt.shape
        assigned = np.zeros((n_img, nd), bool)
        rows = np.arange(n_img)
        out = []
        for i in range(self.ig_gt.shape[1]):
            ig = self.ig_gt[:, i]
            cand = (self.ig_dt != -1) & ~assigned & (self.ov[metric, :, :, i] > mo) & (ig != -1)[:, None]
            s = np.where(cand, self.score, -np.inf)
            j = np.argmax(s, 1)
            hit = s[rows, j] > -10000000
            tp = hit & (ig == 0) & (self.ig_dt[rows, j] == 0)
            out.append(self.score[rows, j][tp])
            assigned[rows[hit], j[hit]] = True
        return np.concatenate(out) if out else np.zeros(0)

    def statistics(self, metric, mo, thresholds, aos):
        """pass 2 at every threshold -> pr (T, 4): tp, fp, fn, similarity"""
        T = len(thresholds)
        n_img, nd = self.ig_dt.shape
        usable = (self.ig_dt != -1)[:, None, :] & ~(self.score[:, None, :] < np.asarray(thresholds)[None, :, None])
        assigned = np.zeros((n_img, T, nd), bool)
        tp = np.zeros((n_img, T), np.int64)
        fn = np.zeros((n_img, T), np.int64)
        sim = np.zeros((n_img, T))
        cols = np.arange(nd)
        ig0, ig1 = (self.ig_dt == 0)[:, None, :], (self.ig_dt == 1)[:, None, :]
        for i in range(self.ig_gt.shape[1]):
            ig = self.ig_gt[:, i][:, None]
            o = self.ov[metric, :, :, i][:, None, :]
            cand = usable & ~assigned & (o > mo) & (ig != -1)[:, :, None]
            c0, c1 = cand & ig0, cand & ig1
            has0, has1 = c0.any(2), c1.any(2)
            det = np.where(has0, np.argmax(np.where(c0, o, -np.inf), 2), np.argmax(c1, 2))
            found = has0 | has1
            fn += ~found & (ig == 0)
            hit = has0 & (ig == 0)
            tp += hit
            if aos:
                delta = self.gt_alpha[:, i][:, None] - np.take_along_axis(self.dt_alpha, det, 1)
                sim = sim + np.where(hit, (1.0 + np.cos(delta)) / 2.0, 0.0)
            assigned |= found[:, :, None] & (cols[None, None, :] == det[:, :, None])
        left = usable & ~assigned & ig0
        fp = left.sum(2)
        if metric == 0:
            fp = fp - (left & (self.dc_ov > mo)[:, None, :]).sum(2)
        sim = np.where((tp > 0) | (fp > 0), sim, 0.0)
        pr = np.zeros((T, 4))
        pr[:, 0], pr[:, 1], pr[:, 2] = tp.sum(0), fp.sum(0), fn.sum(0)
        acc = np.zeros(T)
        for k in range(n_img):          # images in order
            acc = acc + sim[k]
        pr[:, 3] = acc
        return pr


def get_thresholds(scores, num_gt, n=N_PTS):
    """the recall-sampled thresholds: walking the scores in descending order, a score is taken when its recall is at least
    as close to the next sample point as the following score's, and the last one always"""
    s = np.sort(np.asarray(scores, np.float64))[::-1]
    cur, out = 0.0, []
    for i in range(len(s)):
        left = (i + 1) / num_gt
        right = (i + 2) / num_gt if i + 1 < len(s) else left
        if i + 1 < len(s) and (right - cur) < (cur - left):
            continue
        out.append(s[i])
        cur += 1 / (n - 1.0)
    return np.array(out)


def evaluate(gt_annos, dt_annos, current_classes, ovs=None):
    """ovs: per image (3, nd, ng) overlap matrices to use instead of computing them -> dict: overlaps (per image (3, nd, ng)), thresholds / pr per config {(metric, j, diff, k)}, precision / recall /
    orientation (3, C, 3, 2, 41), mAP_R11 / mAP_R40 (3, C, 3, 2), mAP_aos, compute_aos, result_str, ret_dict"""
    assert len(gt_annos) == len(dt_annos)
    classes = current_classes if isinstance(current_classes, (list, tuple)) else [current_classes]
    classes = [{v: k for k, v in CLASS_TO_NAME.items()}[c] if isinstance(c, str) else c for c in classes]
    mo_all = MIN_OVERLAPS[:, :, classes]
    first = next((d for d in dt_annos if len(d["alpha"])), None)
    compute_aos = first is not None and first["alpha"][0] != -10
    if ovs is None:
        ovs = [overlaps(d, g) for g, d in zip(gt_annos, dt_annos)]
    shape = (3, len(classes), 3, 2, N_PTS)
    prec, rec, orient = np.zeros(shape), np.zeros(shape), np.zeros(shape)
    thresholds, prs = {}, {}
    for j, c in enumerate(classes):
        for diff in range(3):
            sp = _Split(gt_annos, dt_annos, ovs, c, diff)
            for metric in range(3):
                for k in range(2):
                    mo = mo_all[k, metric, j]
                    thr = get_thresholds(sp.tp_scores(metric, mo), sp.nvalid)
                    pr = sp.statistics(metric, mo, thr, aos=compute_aos and metric == 0)
                    thresholds[(metric, j, diff, k)], prs[(metric, j, diff, k)] = thr, pr
                    T = len(thr)
                    with np.errstate(divide="ignore", invalid="ignore"):
                        r = np.zeros(N_PTS); p = np.zeros(N_PTS); a = np.zeros(N_PTS)
                        r[:T] = pr[:, 0] / (pr[:, 0] + pr[:, 2])
                        p[:T] = pr[:, 0] / (pr[:, 0] + pr[:, 1])
                        if compute_aos and metric == 0:
                            a[:T] = pr[:, 3] / (pr[:, 0] + pr[:, 1])
                    for arr, dst in ((r, rec), (p, prec), (a, orient)):
                        # suffix maxima; np.maximum.accumulate would skip NaN differently from np.max, so use np.max
                        dst[metric, j, diff, k] = arr
                        for t in range(T):
                            dst[metric, j, diff, k, t] = np.max(arr[t:])
    m11 = lambda x: sum_points(x, range(0, N_PTS, 4)) / 11 * 100
    m40 = lambda x: sum_points(x, range(1, N_PTS)) / 40 * 100
    mAP = m11(prec)
    mAP_aos = m11(orient[0]) if compute_aos else None
    res = dict(overlaps=ovs, thresholds=thresholds, pr=prs, precision=prec, recall=rec, orientation=orient, mAP_R11=mAP, mAP_R40=m40(prec),
               mAP_aos=mAP_aos, compute_aos=compute_aos)
    res["result_str"], res["ret_dict"] = report(classes, mo_all, mAP, mAP_aos)
    return res


def sum_points(x, idx):
    s = 0
    for i in idx:
        s = s + x[..., i]
    return s


def report(classes, mo, mAP, mAP_aos):
    bbox, bev, d3 = mAP
    text = ""
    for j, c in enumerate(classes):
        for i in range(mo.shape[0]):
            text += "%s AP@%s:\n" % (CLASS_TO_NAME[c], ", ".join("%.2f" % v for v in mo[i, :, j]))
            for tag, m in (("bbox", bbox), ("bev ", bev), ("3d  ", d3)):
                text += "%s AP:%s\n" % (tag, ", ".join("%.4f" % m[j, d, i] for d in range(3)))
            if mAP_aos is not None:
                text += "aos  AP:%s\n" % ", ".join("%.2f" % mAP_aos[j, d, i] for d in range(3))
    ret = {}
    for tag, m in (("3d", d3), ("bev", bev), ("image", bbox)):
        for d, name in enumerate(("easy", "moderate", "hard")):
            ret["Car_%s_%s" % (tag, name)] = m[0, d, 0]
    return text, ret


# ------------------------------------------------------------------------------------------------ synthetic splits
def synth_split(seed, n_img, n_gt, n_dt, classes=("Car", "Pedestrian", "Cyclist", "Van", "Person_sitting", "DontCare"), jitter=0.12):
    """random annotation lists (gt, dt) in the reference's dict layout: GT spread over the camera's field of view with
    every truncation / occlusion band and heights on both sides of the limits; detections are jittered copies of GT boxes
    (some duplicated) and free boxes, with scores rounded to 4 decimals so that ties occur"""
    rng = np.random.default_rng(seed)
    gts, dts = [], []
    for _ in range(n_img):
        g = _random_objects(rng, int(rng.integers(0, n_gt + 1)) if n_gt else 0, classes)
        g["score"] = np.zeros(len(g["name"]))
        gts.append(g)
        nd = int(rng.integers(0, n_dt + 1)) if n_dt else 0
        src = rng.integers(0, max(len(g["name"]), 1), nd)
        d = _random_objects(rng, nd, ("Car", "Pedestrian", "Cyclist"))
        from_gt = (rng.random(nd) < 0.7) & (len(g["name"]) > 0)
        for key in ("bbox", "dimensions", "location", "rotation_y", "alpha"):
            if len(g["name"]):
                d[key][from_gt] = g[key][src[from_gt]]
        d["name"][from_gt] = np.array([n if n in ("Car", "Pedestrian", "Cyclist") else "Car" for n in g["name"][src[from_gt]]])
        k = int(from_gt.sum())
        d["bbox"][from_gt] += rng.normal(0, 6 * jitter, (k, 4))
        d["location"][from_gt] += rng.normal(0, jitter, (k, 3)) * [1, 0.2, 1]
        d["dimensions"][from_gt] *= 1 + rng.normal(0, jitter / 4, (k, 3))
        d["rotation_y"][from_gt] += rng.normal(0, jitter, k)
        d["alpha"][from_gt] += rng.normal(0, jitter, k)
        d["bbox"] = np.round(d["bbox"], 4)
        d["score"] = np.round(np.where(from_gt, 0.3 + 0.7 * rng.random(nd), 0.6 * rng.random(nd)), 2 if rng.random() < 0.5 else 4)
        d["truncated"][:] = -1
        d["occluded"][:] = -1
        dts.append(d)
    return gts, dts


def _random_objects(rng, n, classes):
    name = np.array([classes[k] for k in rng.integers(0, len(classes), n)]) if n else np.array([])
    x1 = rng.uniform(0, 1100, n)
    y1 = rng.integers(100, 250, n).astype(np.float64)      # integral: heights of exactly 40 or 25 stay exact
    h = np.where(rng.random(n) < 0.2, np.where(rng.random(n) < 0.5, 40.0, 25.0), rng.uniform(10, 120, n))
    bbox = np.stack([x1, y1, x1 + rng.uniform(20, 200, n), y1 + h], 1) if n else np.zeros((0, 4))
    dims = np.stack([rng.uniform(0.5, 4.5, n), rng.uniform(1.4, 1.9, n), rng.uniform(0.5, 1.9, n)], 1) if n else np.zeros((0, 3))
    loc = np.stack([rng.uniform(-20, 20, n), rng.uniform(1.4, 2.0, n), rng.uniform(5, 60, n)], 1) if n else np.zeros((0, 3))
    return dict(name=name, truncated=rng.choice([0.0, 0.1, 0.15, 0.2, 0.3, 0.4, 0.5, 0.6], n).astype(np.float64),
                occluded=rng.integers(0, 4, n), alpha=rng.uniform(-np.pi, np.pi, n), bbox=bbox, dimensions=dims, location=loc,
                rotation_y=rng.uniform(-np.pi, np.pi, n))

"""oracle/make_golden_kitti_eval.py -- golden vectors for the KITTI AP evaluation.

Runs the reference's OWN tools/kitti_object_eval_python (eval.py and kitti_common.get_label_anno, imported unchanged from
/root/reference) on a synthetic split written as KITTI label and result files, and writes tests/golden/kitti_eval.npz.
TEST INFRASTRUCTURE ONLY.
    python oracle/make_golden_kitti_eval.py

Stand-ins for what the reference's module-level imports need and this environment lacks:
  - skimage (imported by kitti_common for image reading, unused here) is an empty module in sys.modules;
  - eval.py is imported directly: evaluate.py only adds the file reading (restated by read_label_annos) and imports fire;
  - NUMBA_ENABLE_CUDASIM=1 runs rotate_iou_gpu_eval's numba.cuda kernel on the CPU.
The simulator evaluates in Python, so its BEV / 3D IoU can differ from a GPU run in the last fp32 bits: detections whose
BEV or 3D IoU with a GT lies within 1e-4 of 0.25, 0.5 or 0.7 are moved until none does (measured with the oracle's exact
clip).  For small or nearly parallel boxes the reference's fp32 clipper is itself off by up to ~2e-4 from the exact
area, and any other fp32 clipper by a different amount: detections with a BEV IoU more than 1.5e-6 from the exact clip are
turned until none is, and so are those whose corners, rounded to fp32 the way the iou3d overlap builds them, move the
exact IoU by more than 1.5e-6; so the fixture pins the convention and not the rounding noise of one clipper.

The split (120 images; the reference needs at least 50) has Car, Van, Pedestrian, Person_sitting, Cyclist and DontCare
labels, truncation / occlusion in every difficulty band and at the band limits, GT and detections with heights at and
around the minimum heights, duplicated detections, tied scores, and images without GT, without detections or with only
DontCare.  Besides the texts and the reference's parsed annotations it stores the three overlap matrices, each config's
thresholds and pr counts (captured around get_thresholds / fused_compute_statistics), the precision / recall / orientation
arrays, the mAPs, the result string and ret_dict.
"""
import os
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
N_IMG, N_GT, N_DT, SEED = 120, 10, 12, 77
CLASSES = [0, 1, 2]
KEYS = ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score")


def gt_line(a, k):
    x1, y1, x2, y2 = a["bbox"][k]
    l, h, w = a["dimensions"][k]
    x, y, z = a["location"][k]
    return "%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
        a["name"][k], a["truncated"][k], a["occluded"][k], a["alpha"][k], x1, y1, x2, y2, h, w, l, x, y, z, a["rotation_y"][k])


def dt_line(a, k):
    x1, y1, x2, y2 = a["bbox"][k]
    l, h, w = a["dimensions"][k]
    x, y, z = a["location"][k]
    return "%s -1 -1 %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f" % (
        a["name"][k], a["alpha"][k], x1, y1, x2, y2, h, w, l, x, y, z, a["rotation_y"][k], a["score"][k])


def split():
    from oracle import kitti_eval as OK
    gts, dts = OK.synth_split(SEED, N_IMG, N_GT, N_DT)
    empty = lambda a: {k: (v[:0] if k != "name" else np.array([])) for k, v in a.items()}
    gts[3] = empty(gts[3])                       # no GT
    dts[5] = empty(dts[5])                       # no detections
    dts[6] = empty(dts[6])
    g = gts[7]                                   # only DontCare
    g["name"] = np.array(["DontCare"] * len(g["name"]))
    return gts, dts


def fp32_box_iou(d, g):
    """BEV IoU of the exact clip of corners built in fp32 the way the iou3d overlap builds them from
    [x - l/2, z - w/2, x + l/2, z + w/2, ry] (extent rounded to fp32, rotated about the rounded centre)"""
    from oracle.gt_paste import clip_area
    f = np.float32

    def corners(a):
        x, z = a["location"][:, 0].astype(f), a["location"][:, 2].astype(f)
        l, w, ry = a["dimensions"][:, 0].astype(f), a["dimensions"][:, 2].astype(f), a["rotation_y"].astype(f)
        x1, y1, x2, y2 = x - l * f(0.5), z - w * f(0.5), x + l * f(0.5), z + w * f(0.5)
        cx, cy, c, s = (x1 + x2) / f(2), (y1 + y2) / f(2), np.cos(ry), np.sin(ry)
        px, py = np.stack([x1, x2, x2, x1], 1), np.stack([y1, y1, y2, y2], 1)
        dx, dy = px - cx[:, None], py - cy[:, None]
        return np.stack([dx * c[:, None] + dy * s[:, None] + cx[:, None], -dx * s[:, None] + dy * c[:, None] + cy[:, None]], 2), l * w
    cd, ad = corners(d)
    cg, ag = corners(g)
    out = np.zeros((len(cd), len(cg)))
    for j in range(len(cd)):
        for i in range(len(cg)):
            inter = clip_area(cd[j], cg[i])
            out[j, i] = inter / (float(ad[j]) + float(ag[i]) - inter)
    return out


def settle(gts, dts, E, rng):
    """move detections until no BEV / 3D IoU lies within 1e-4 of a threshold, and turn the ones whose BEV IoU in the
    reference's fp32 clipper is more than 1.5e-6 from the exact clip a little (after 20 tries: far away).
    The values are rounded as the result text rounds them."""
    from oracle import kitti_eval as OK
    marks = np.array([0.25, 0.5, 0.7])
    moved = turned = 0
    for g, d in zip(gts, dts):
        for attempt in range(30):
            o = OK.overlaps(d, g)
            bad = (np.abs(o[1:, :, :, None] - marks).min(-1) < 1e-4).any(0).any(1)
            if len(d["name"]) and len(g["name"]):
                box = lambda a: np.concatenate([a["location"][:, [0, 2]], a["dimensions"][:, [0, 2]], a["rotation_y"][:, None]], 1)
                ill = ((np.abs(E.bev_box_overlap(box(d), box(g)).astype(np.float64) - o[1]) > 1.5e-6) |
                       (np.abs(fp32_box_iou(d, g) - o[1]) > 1.5e-6)).any(1)
            else:
                ill = np.zeros(len(d["name"]), bool)
            if not (bad | ill).any():
                break
            d["location"][bad, 0] = np.round(d["location"][bad, 0] + rng.uniform(0.01, 0.03, int(bad.sum())), 4)
            d["rotation_y"][ill] = np.round(d["rotation_y"][ill] + rng.uniform(0.05, 0.15, int(ill.sum())), 4)
            if attempt >= 20:                    # still ill-conditioned: a free detection far from every GT
                d["location"][ill, 0] += 200.0
            moved += int(bad.sum())
            turned += int(ill.sum())
        else:
            raise RuntimeError("could not settle a detection")
    return moved, turned


def main():
    os.environ["NUMBA_ENABLE_CUDASIM"] = "1"
    sys.modules.setdefault("skimage", types.ModuleType("skimage")).io = None
    sys.path.insert(0, ROOT)
    sys.path.insert(0, REF)
    import tools.kitti_object_eval_python.eval as E
    import tools.kitti_object_eval_python.kitti_common as KC

    gts, dts = split()
    tmp = tempfile.mkdtemp()
    lab, res = os.path.join(tmp, "label"), os.path.join(tmp, "result")
    os.makedirs(lab)
    os.makedirs(res)

    def write(gts, dts):
        gt_text, dt_text = [], []
        for k, (g, d) in enumerate(zip(gts, dts)):
            gt_text.append("".join(gt_line(g, i) + "\n" for i in range(len(g["name"]))))
            dt_text.append("".join(dt_line(d, i) + "\n" for i in range(len(d["name"]))))
            open(os.path.join(lab, "%06d.txt" % k), "w").write(gt_text[-1])
            open(os.path.join(res, "%06d.txt" % k), "w").write(dt_text[-1])
        return gt_text, dt_text

    # round-trip through the texts before checking the thresholds: the reference reads the rounded values
    write(gts, dts)
    gts = KC.get_label_annos(lab, list(range(N_IMG)))
    dts = KC.get_label_annos(res)
    moved, turned = settle(gts, dts, E, np.random.default_rng(SEED))
    gt_text, dt_text = write(gts, dts)
    gt_annos = KC.get_label_annos(lab, list(range(N_IMG)))
    dt_annos = KC.get_label_annos(res)

    # capture each config's thresholds and pr counts, and each metric's eval_class arrays
    thr_log, pr_log, cls_log = [], {}, []
    get_thresholds, fused, eval_class = E.get_thresholds, E.fused_compute_statistics, E.eval_class

    def get_thresholds_logged(scores, num_gt, *a):
        t = get_thresholds(scores, num_gt, *a)
        thr_log.append(np.array(t, np.float64))
        return t

    def fused_logged(overlaps, pr, *a, **k):
        fused(overlaps, pr, *a, **k)
        pr_log[len(thr_log) - 1] = pr.copy()

    def eval_class_logged(*a, **k):
        r = eval_class(*a, **k)
        cls_log.append(r)
        return r

    E.get_thresholds, E.fused_compute_statistics, E.eval_class = get_thresholds_logged, fused_logged, eval_class_logged
    t0 = time.time()
    result_str, ret_dict = E.get_official_eval_result(gt_annos, dt_annos, CLASSES)
    print("reference evaluation: %.1f s" % (time.time() - t0))
    E.get_thresholds, E.fused_compute_statistics, E.eval_class = get_thresholds, fused, eval_class

    nc = len(CLASSES)
    shape = (3, nc, 3, 2)
    thresholds, nthr, pr = np.zeros(shape + (41,)), np.zeros(shape, np.int64), np.zeros(shape + (41, 4))
    for n, idx in enumerate(np.ndindex(*shape)):         # eval_class order: metric, class, difficulty, overlap set
        t = thr_log[n]
        thresholds[idx][:len(t)], nthr[idx] = t, len(t)
        if len(t):
            pr[idx][:len(t)] = pr_log[n]
    out = dict(gt_text=np.array(gt_text), dt_text=np.array(dt_text), classes=np.array(CLASSES), moved=np.array([moved, turned]),
               thresholds=thresholds, nthr=nthr, pr=pr,
               precision=np.stack([r["precision"] for r in cls_log]), recall=np.stack([r["recall"] for r in cls_log]),
               orientation=np.stack([r["orientation"] for r in cls_log]),
               result_str=np.array(result_str), ret_keys=np.array(list(ret_dict)), ret_values=np.array(list(ret_dict.values())))
    for metric in range(3):
        ov, _, _, _ = E.calculate_iou_partly(dt_annos, gt_annos, metric, 50)
        out["overlaps%d" % metric] = np.concatenate([o.reshape(-1) for o in ov])
    for tag, annos in (("gt", gt_annos), ("dt", dt_annos)):
        out[tag + "_counts"] = np.array([len(a["name"]) for a in annos])
        for key in KEYS:
            vals = [a[key] for a in annos if len(a["name"])]
            out["%s_%s" % (tag, key)] = np.concatenate(vals)
    path = os.path.join(ROOT, "tests", "golden", "kitti_eval.npz")
    np.savez_compressed(path, **out)
    print(result_str)
    print("moved %d detections off the thresholds, turned %d; %d GT, %d detections" % (moved, turned, out["gt_counts"].sum(), out["dt_counts"].sum()))
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

"""oracle/make_golden_kitti_eval_coco.py -- golden vectors for the COCO-style KITTI AP and the score filter.

Runs the reference's OWN tools/kitti_object_eval_python (eval.get_coco_eval_result, kitti_common.get_label_anno and
filter_annos_low_score, imported unchanged from /root/reference) on the synthetic split of make_golden_kitti_eval.py and
writes tests/golden/kitti_eval_coco.npz.  TEST INFRASTRUCTURE ONLY.
    python oracle/make_golden_kitti_eval_coco.py

The stand-ins are make_golden_kitti_eval.py's (skimage an empty module, NUMBA_ENABLE_CUDASIM=1), plus one:
do_coco_style_eval calls np.linspace(*overlap_ranges[:, i, j]), which passes the sample count as the float 10.0, and
numpy >= 1.18 refuses a float count.  eval's `np` is replaced by a copy of the numpy module whose linspace takes int(num);
nothing else changes.  The split is that script's, settled by its rule (settle below; the clipper check is that
script's fp32_box_iou) except that the marks a BEV / 3D IoU keeps 1e-4 away from are every COCO threshold (0.25 .. 0.7
and 0.5 .. 0.95 in steps of 0.05) instead of 0.25, 0.5 and 0.7.

Stored: the texts and the reference's parsed annotations (as in kitti_eval.npz); each config's thresholds and pr counts
and the per-set precision / recall / orientation arrays (metric, class, difficulty, set, 41) of the COCO evaluation of
classes [0, 1, 2], captured around do_eval; its result string; the string for "Pedestrian" alone; the reference's
filter_annos_low_score output at SCORE_THRESH and the [0, 1, 2] string of the filtered detections.
"""
import os
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
SCORE_THRESH = 0.5
CLASSES = [0, 1, 2]
MARKS = np.round(np.arange(0.25, 0.951, 0.05), 2)


def settle(gts, dts, E, rng, marks):
    """make_golden_kitti_eval.settle with the marks as an argument: move detections until no BEV / 3D IoU lies within
    1e-4 of a mark, and turn the ones whose BEV IoU in the reference's fp32 clipper (or from fp32-rounded corners) is more
    than 1.5e-6 from the exact clip a little (after 20 tries: far away).  The values are rounded as the result text
    rounds them."""
    from oracle import kitti_eval as OK
    from oracle.make_golden_kitti_eval import fp32_box_iou
    marks = np.asarray(marks, np.float64)
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
            if attempt >= 20:
                d["location"][ill, 0] += 200.0
            moved += int(bad.sum())
            turned += int(ill.sum())
        else:
            raise RuntimeError("could not settle a detection")
    return moved, turned


def pack(out, tag, annos, keys):
    out[tag + "_counts"] = np.array([len(a["name"]) for a in annos])
    for key in keys:
        vals = [a[key] for a in annos if len(a["name"])]
        out["%s_%s" % (tag, key)] = np.concatenate(vals)


def main():
    os.environ["NUMBA_ENABLE_CUDASIM"] = "1"
    sys.modules.setdefault("skimage", types.ModuleType("skimage")).io = None
    sys.path.insert(0, ROOT)
    sys.path.insert(0, REF)
    import tools.kitti_object_eval_python.eval as E
    import tools.kitti_object_eval_python.kitti_common as KC
    from oracle import make_golden_kitti_eval as G

    # the only patch: linspace with an integral sample count, in eval's namespace
    np_int = types.ModuleType("numpy")
    np_int.__dict__.update(np.__dict__)
    np_int.linspace = lambda start, stop, num=50, *a, **k: np.linspace(start, stop, int(num), *a, **k)
    E.np = np_int

    gts, dts = G.split()
    tmp = tempfile.mkdtemp()
    lab, res = os.path.join(tmp, "label"), os.path.join(tmp, "result")
    os.makedirs(lab)
    os.makedirs(res)

    def write(gts, dts):
        gt_text, dt_text = [], []
        for k, (g, d) in enumerate(zip(gts, dts)):
            gt_text.append("".join(G.gt_line(g, i) + "\n" for i in range(len(g["name"]))))
            dt_text.append("".join(G.dt_line(d, i) + "\n" for i in range(len(d["name"]))))
            open(os.path.join(lab, "%06d.txt" % k), "w").write(gt_text[-1])
            open(os.path.join(res, "%06d.txt" % k), "w").write(dt_text[-1])
        return gt_text, dt_text

    write(gts, dts)
    gts = KC.get_label_annos(lab, list(range(G.N_IMG)))
    dts = KC.get_label_annos(res)
    moved, turned = settle(gts, dts, E, np.random.default_rng(G.SEED), MARKS)
    gt_text, dt_text = write(gts, dts)
    gt_annos = KC.get_label_annos(lab, list(range(G.N_IMG)))
    dt_annos = KC.get_label_annos(res)

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
    coco_str = E.get_coco_eval_result(gt_annos, dt_annos, CLASSES)
    print("reference COCO evaluation: %.1f s" % (time.time() - t0))
    E.get_thresholds, E.fused_compute_statistics, E.eval_class = get_thresholds, fused, eval_class
    coco_ped = E.get_coco_eval_result(gt_annos, dt_annos, "Pedestrian")
    filtered = KC.filter_annos_low_score(dt_annos, SCORE_THRESH)
    coco_thresh = E.get_coco_eval_result(gt_annos, filtered, CLASSES)

    nc, ns = len(CLASSES), 10
    shape = (3, nc, 3, ns)
    assert len(thr_log) == int(np.prod(shape)) and len(cls_log) == 3
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
               coco_str=np.array(coco_str), coco_str_pedestrian=np.array(coco_ped), score_thresh=np.array(SCORE_THRESH),
               coco_str_score_thresh=np.array(coco_thresh))
    pack(out, "gt", gt_annos, G.KEYS)
    pack(out, "dt", dt_annos, G.KEYS)
    pack(out, "dtf", filtered, G.KEYS)
    path = os.path.join(ROOT, "tests", "golden", "kitti_eval_coco.npz")
    np.savez_compressed(path, **out)
    print(coco_str + coco_ped + coco_thresh)
    print("moved %d detections off the thresholds, turned %d; %d GT, %d detections, %d above %g" % (
        moved, turned, out["gt_counts"].sum(), out["dt_counts"].sum(), out["dtf_counts"].sum(), SCORE_THRESH))
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

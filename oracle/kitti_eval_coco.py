"""oracle/kitti_eval_coco.py -- CPU restatement (numpy) of the KITTI AP evaluation over any number of overlap sets, and
of the COCO-style report, tools/kitti_object_eval_python/eval.py.
TEST INFRASTRUCTURE ONLY: imported by tests/ and scripts/, never by pointrcnn_b200/.

Built on oracle/kitti_eval.py (overlaps, clean_data, both statistics passes, get_thresholds), which evaluates the official
two sets; here the sets are an argument:
  evaluate_sets   eval_class :443-548 and do_eval :567-587 for K sets (K, 3, C)
  coco            do_coco_style_eval :590-605, get_coco_eval_result :681-740 (ten sets per class, averaged)
Pinned by tests/golden/kitti_eval_coco.npz, which the reference's own evaluator produced
(oracle/make_golden_kitti_eval_coco.py).
"""
import numpy as np

from oracle import kitti_eval as OK

CLASS_TO_RANGE = {0: [0.5, 0.95, 10], 1: [0.25, 0.7, 10], 2: [0.25, 0.7, 10], 3: [0.5, 0.95, 10], 4: [0.25, 0.7, 10]}


def _classes(current_classes):
    classes = current_classes if isinstance(current_classes, (list, tuple)) else [current_classes]
    return [{v: k for k, v in OK.CLASS_TO_NAME.items()}[c] if isinstance(c, str) else c for c in classes]


def evaluate_sets(gt_annos, dt_annos, current_classes, min_overlaps, ovs=None):
    """min_overlaps (K, 3, C); ovs: per image (3, nd, ng) overlap matrices to use instead of computing them -> dict:
    overlaps, thresholds / pr per config {(metric, j, diff, k)}, precision / recall / orientation (3, C, 3, K, 41),
    mAP_R11 (3, C, 3, K), mAP_aos (C, 3, K) or None, compute_aos"""
    assert len(gt_annos) == len(dt_annos)
    classes = _classes(current_classes)
    mo_all = np.asarray(min_overlaps, np.float64)
    K = mo_all.shape[0]
    first = next((d for d in dt_annos if len(d["alpha"])), None)
    compute_aos = first is not None and first["alpha"][0] != -10
    if ovs is None:
        ovs = [OK.overlaps(d, g) for g, d in zip(gt_annos, dt_annos)]
    shape = (3, len(classes), 3, K, OK.N_PTS)
    prec, rec, orient = np.zeros(shape), np.zeros(shape), np.zeros(shape)
    thresholds, prs = {}, {}
    for j, c in enumerate(classes):
        for diff in range(3):
            sp = OK._Split(gt_annos, dt_annos, ovs, c, diff)
            for metric in range(3):
                for k in range(K):
                    mo = mo_all[k, metric, j]
                    thr = OK.get_thresholds(sp.tp_scores(metric, mo), sp.nvalid)
                    pr = sp.statistics(metric, mo, thr, aos=compute_aos and metric == 0)
                    thresholds[(metric, j, diff, k)], prs[(metric, j, diff, k)] = thr, pr
                    T = len(thr)
                    with np.errstate(divide="ignore", invalid="ignore"):
                        r = np.zeros(OK.N_PTS); p = np.zeros(OK.N_PTS); a = np.zeros(OK.N_PTS)
                        r[:T] = pr[:, 0] / (pr[:, 0] + pr[:, 2])
                        p[:T] = pr[:, 0] / (pr[:, 0] + pr[:, 1])
                        if compute_aos and metric == 0:
                            a[:T] = pr[:, 3] / (pr[:, 0] + pr[:, 1])
                    for arr, dst in ((r, rec), (p, prec), (a, orient)):
                        # suffix maxima with np.max's NaN rule, as oracle/kitti_eval.py
                        dst[metric, j, diff, k] = arr
                        for t in range(T):
                            dst[metric, j, diff, k, t] = np.max(arr[t:])
    m11 = lambda x: OK.sum_points(x, range(0, OK.N_PTS, 4)) / 11 * 100
    return dict(overlaps=ovs, thresholds=thresholds, pr=prs, precision=prec, recall=rec, orientation=orient, mAP_R11=m11(prec),
                mAP_aos=m11(orient[0]) if compute_aos else None, compute_aos=compute_aos)


def coco_min_overlaps(classes):
    """do_coco_style_eval's ten sets (10, 3, C): np.linspace over each class's range, with the sample count as an int
    (the reference passes the float 10.0, which numpy >= 1.18 refuses)"""
    out = np.zeros([10, 3, len(classes)])
    for j, c in enumerate(classes):
        start, stop, num = CLASS_TO_RANGE[c]
        out[:, :, j] = np.linspace(start, stop, int(num))[:, None]
    return out


def coco_evaluate(gt_annos, dt_annos, current_classes, ovs=None):
    """get_coco_eval_result: evaluate_sets() over the ten sets -> its dict, plus mAP_coco (3, C, 3) and mAP_aos_coco
    (C, 3), the R11 mAPs averaged over the sets, and coco_str, the reference's string"""
    classes = _classes(current_classes)
    res = evaluate_sets(gt_annos, dt_annos, classes, coco_min_overlaps(classes), ovs=ovs)
    res["mAP_coco"] = np.stack([np.ascontiguousarray(m).mean(-1) for m in res["mAP_R11"]])
    res["mAP_aos_coco"] = np.ascontiguousarray(res["mAP_aos"]).mean(-1) if res["compute_aos"] else None
    res["coco_str"] = coco_report(classes, res["mAP_coco"], res["mAP_aos_coco"])
    return res


def coco_report(classes, mAP, mAP_aos):
    text = ""
    for j, c in enumerate(classes):
        start, stop, num = CLASS_TO_RANGE[c]
        text += "%s coco AP@%.2f:%.2f:%.2f:\n" % (OK.CLASS_TO_NAME[c], start, (stop - start) / (num - 1), stop)
        for tag, m in zip(("bbox", "bev ", "3d  "), mAP):
            text += "%s AP:%s\n" % (tag, ", ".join("%.2f" % m[j, d] for d in range(3)))
        if mAP_aos is not None:
            text += "aos  AP:%s\n" % ", ".join("%.2f" % mAP_aos[j, d] for d in range(3))
    return text

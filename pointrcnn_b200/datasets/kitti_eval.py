"""The KITTI AP metric on the device: tools/kitti_object_eval_python (eval.py:608-678 get_official_eval_result,
evaluate.py:14-28 evaluate, kitti_common.py:293-346 get_label_annos) with the statistics in CUDA (`prb_kitti_eval`).

Two ways in:
  - from annotations or files: `get_official_eval_result(gt_annos, dt_annos, current_classes)` and
    `evaluate(label_path, result_path, label_split_file, current_class)` return the reference's (result_str, ret_dict);
    `evaluate_annos` returns a KittiEvalResult with the full precision / recall / orientation arrays and mAP_R40 as well;
  - in memory: `KittiEvaluator` takes `detections_device` output batch by batch without synchronising, and `result()`
    evaluates with one device-to-host copy.  With text_rounding=True its AP equals, bit for bit, the AP of the result
    files `write_kitti_batch` writes for the same batches.

Differences from the reference: any number of images works (the reference needs at least 50); BEV and 3D IoU come from the
iou3d overlap in fp32 (a few 1e-6 from numba's clipper, so a pair right at a threshold may be decided differently); the
orientation similarity is summed in another order (differences ~1e-12).
"""
import ctypes
import pathlib
import re

import numpy as np
import torch

from .. import _cabi as C

CLASS_TO_NAME = {0: "Car", 1: "Pedestrian", 2: "Cyclist", 3: "Van", 4: "Person_sitting"}
NAME_TO_CLASS = {v: k for k, v in CLASS_TO_NAME.items()}
# eval.py:609-615: [overlap set, metric (bbox, bev, 3d), class]
MIN_OVERLAPS = np.array([[[0.7, 0.5, 0.5, 0.7, 0.5]] * 3,
                         [[0.7, 0.5, 0.5, 0.7, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25], [0.5, 0.25, 0.25, 0.5, 0.25]]])
N_SAMPLE_PTS = 41
MAX_DET_PER_IMAGE = 1024
# row of the device tables (include/pointrcnn_b200.h)
COLS = 16
_CODES = {"car": 0, "pedestrian": 1, "cyclist": 2, "van": 3, "person_sitting": 4}
_DONTCARE = 5


# ------------------------------------------------------------------------------------------------ host: labels
def read_label_anno(path):
    """one KITTI label / result file -> the reference's annotation dict (float64 fields, dimensions reordered hwl -> lhw,
    the score column when a line has 16 fields, else zeros)"""
    with open(path, "r") as f:
        rows = [line.strip().split(" ") for line in f.readlines()]

    def cols(a, b):
        return np.array([[float(v) for v in r[a:b]] for r in rows])

    anno = {
        "name": np.array([r[0] for r in rows]),
        "truncated": np.array([float(r[1]) for r in rows]),
        "occluded": np.array([int(r[2]) for r in rows]),
        "alpha": np.array([float(r[3]) for r in rows]),
        "bbox": cols(4, 8).reshape(-1, 4),
        "dimensions": cols(8, 11).reshape(-1, 3)[:, [2, 0, 1]],
        "location": cols(11, 14).reshape(-1, 3),
        "rotation_y": np.array([float(r[14]) for r in rows]).reshape(-1),
    }
    has_score = len(rows) != 0 and len(rows[0]) == 16
    anno["score"] = np.array([float(r[15]) for r in rows]) if has_score else np.zeros([len(anno["bbox"])])
    return anno


def read_label_annos(label_dir, image_ids=None):
    """get_label_annos: image_ids None -> every <6 digits>.txt of the directory in id order; an int n -> 0..n-1"""
    label_dir = pathlib.Path(label_dir)
    if image_ids is None:
        pat = re.compile(r"^\d{6}.txt$")
        image_ids = sorted(int(p.stem) for p in label_dir.glob("*.txt") if pat.match(p.name))
    elif not isinstance(image_ids, list):
        image_ids = list(range(image_ids))
    return [read_label_anno(label_dir / ("%06d.txt" % i)) for i in image_ids]


def class_code(name):
    """class names compare case-insensitively, except DontCare, which clean_data matches exactly"""
    return _DONTCARE if name == "DontCare" else _CODES.get(str(name).lower(), -1)


def pack_annos(annos):
    """list of annotation dicts -> (table (rows, 16) float64 in the device layout, per-image row counts int64)"""
    counts = np.array([len(a["name"]) for a in annos], np.int64)
    t = np.zeros((int(counts.sum()), COLS))
    if len(t):
        def cat(key, width):
            return np.concatenate([np.asarray(a[key], np.float64).reshape(len(a["name"]), width) for a in annos])
        t[:, 0:4] = cat("bbox", 4)
        t[:, 4] = cat("alpha", 1)[:, 0]
        t[:, 5] = cat("truncated", 1)[:, 0]
        t[:, 6] = cat("occluded", 1)[:, 0]
        t[:, 7:10] = cat("dimensions", 3)
        t[:, 10:13] = cat("location", 3)
        t[:, 13] = cat("rotation_y", 1)[:, 0]
        t[:, 14] = np.concatenate([np.asarray(a.get("score", np.zeros(len(a["name"]))), np.float64).reshape(-1) for a in annos])
        t[:, 15] = [class_code(n) for a in annos for n in a["name"]]
    return t, counts


def class_list(current_classes):
    """get_official_eval_result's normalisation: one class or a list, names or indices; only 0..2 can be evaluated"""
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    out = [NAME_TO_CLASS[c] if isinstance(c, str) else int(c) for c in current_classes]
    for c in out:
        if c not in (0, 1, 2):
            raise ValueError("kitti_eval: class %r cannot be evaluated (clean_data knows Car, Pedestrian and Cyclist)" % (c,))
    if not 1 <= len(out) <= 8:
        raise ValueError("kitti_eval: 1 to 8 classes, got %d" % len(out))
    return out


def _offsets(counts):
    off = np.zeros(len(counts) + 1, np.int64)
    np.cumsum(counts, out=off[1:])
    return off


# ------------------------------------------------------------------------------------------------ device
def _launch(classes, gt, gt_off, gt_counts, dt, dt_off, dt_count, dt_caps, device):
    """prb_kitti_eval on the current stream -> (out, overlaps) device tensors; nothing waits for the GPU.
    gt_counts / dt_caps are host arrays (row counts, rows owned per image)."""
    lib = C.lib()
    n_img = len(gt_counts)
    if n_img < 1:
        raise ValueError("kitti_eval: no images")
    max_det = int(dt_caps.max())
    if max_det > MAX_DET_PER_IMAGE:
        raise ValueError("kitti_eval: %d detections in one image > %d" % (max_det, MAX_DET_PER_IMAGE))
    n_gt, n_dt, nc = int(gt_counts.sum()), int(dt_caps.sum()), len(classes)
    pair_off = _offsets(gt_counts * dt_caps)
    n_pairs = int(pair_off[-1])
    cls = np.ascontiguousarray(classes, np.int32)
    mo = np.ascontiguousarray(MIN_OVERLAPS[:, :, classes], np.float64)
    nconf = 18 * nc
    ws_bytes = lib.prb_kitti_eval_workspace_bytes(n_img, n_gt, n_dt, nc)
    with torch.cuda.device(device):
        pair_dev = torch.from_numpy(pair_off).to(device, non_blocking=True)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        ov = torch.empty(max(3 * n_pairs, 1), dtype=torch.float64, device=device)
        out = torch.empty(nconf * N_SAMPLE_PTS * 8 + 1 + nconf, dtype=torch.float64, device=device)
        P = ctypes.c_void_p
        C.check(lib.prb_kitti_eval(n_img, nc, P(cls.ctypes.data), P(mo.ctypes.data), C.ptr(gt), C.ptr(gt_off), n_gt, C.ptr(dt), C.ptr(dt_off),
                                   C.ptr(dt_count), n_dt, max_det, C.ptr(pair_dev), ctypes.c_longlong(n_pairs), C.ptr(ov), C.ptr(out), C.ptr(ws),
                                   ctypes.c_size_t(ws_bytes), C.stream()), "kitti_eval")
    return out, ov[:3 * n_pairs].view(3, n_pairs)


class KittiEvalResult:
    """precision / recall / orientation: (metric (bbox, bev, 3d), class, difficulty, overlap set, 41) float64, each metric's
    array as the reference's eval_class returns it (orientation only for bbox, zero without AOS); mAP_R11 / mAP_R40:
    (metric, class, difficulty, overlap set); mAP_aos (class, difficulty, overlap set) or None; counts: (..., 41, 4)
    tp, fp, fn, similarity; thresholds (..., 41) and num_thresholds (...)"""

    def __init__(self, classes, out):
        nc = len(classes)
        nconf = 18 * nc
        body = out[:nconf * N_SAMPLE_PTS * 8].reshape(3, nc, 3, 2, N_SAMPLE_PTS, 8)
        self.classes = list(classes)
        self.min_overlaps = MIN_OVERLAPS[:, :, self.classes]
        self.compute_aos = bool(out[nconf * N_SAMPLE_PTS * 8] != 0)
        self.num_thresholds = out[nconf * N_SAMPLE_PTS * 8 + 1:].reshape(3, nc, 3, 2).astype(np.int64)
        self.counts = body[..., 0:4].copy()
        self.thresholds = body[..., 7].copy()
        self.recall = body[..., 4].copy()
        self.precision = body[..., 5].copy()
        self.orientation = np.zeros_like(self.precision)
        if self.compute_aos:
            self.orientation[0] = body[0, ..., 6]
        self.mAP_R11 = _map_r11(self.precision)
        self.mAP_R40 = _map_r40(self.precision)
        self.mAP_aos = _map_r11(self.orientation[0]) if self.compute_aos else None
        self.result_str, self.ret_dict = self._report()

    def _report(self):
        bbox, bev, d3 = self.mAP_R11
        lines = []
        for j, c in enumerate(self.classes):
            for i in range(self.min_overlaps.shape[0]):
                lines.append("{} AP@{:.2f}, {:.2f}, {:.2f}:".format(CLASS_TO_NAME[c], *self.min_overlaps[i, :, j]))
                for tag, m in (("bbox AP", bbox), ("bev  AP", bev), ("3d   AP", d3)):
                    lines.append(f"{tag}:{m[j, 0, i]:.4f}, {m[j, 1, i]:.4f}, {m[j, 2, i]:.4f}")
                if self.compute_aos:
                    a = self.mAP_aos
                    lines.append(f"aos  AP:{a[j, 0, i]:.2f}, {a[j, 1, i]:.2f}, {a[j, 2, i]:.2f}")
        ret = {}
        # the reference files the first requested class under the Car_* keys, whatever it is
        for tag, m in (("3d", d3), ("bev", bev), ("image", bbox)):
            for d, diff in enumerate(("easy", "moderate", "hard")):
                ret["Car_%s_%s" % (tag, diff)] = m[0, d, 0]
        return "".join(s + "\n" for s in lines), ret


def _map_r11(prec):
    """get_mAP: the 11 recall points 0, 4, ..., 40, summed in that order"""
    sums = 0
    for i in range(0, prec.shape[-1], 4):
        sums = sums + prec[..., i]
    return sums / 11 * 100


def _map_r40(prec):
    """the 40 recall points 1..40 of the current KITTI benchmark, summed in that order"""
    sums = 0
    for i in range(1, prec.shape[-1]):
        sums = sums + prec[..., i]
    return sums / 40 * 100


def _device(device):
    return torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())


def evaluate_annos(gt_annos, dt_annos, current_classes, device=None, return_overlaps=False):
    """the whole evaluation of two annotation lists on the device -> KittiEvalResult (and the (3, pairs) overlap matrices,
    (dt x gt) row-major per image, when asked)"""
    assert len(gt_annos) == len(dt_annos)
    classes = class_list(current_classes)
    dev = _device(device)
    gt, gt_counts = pack_annos(gt_annos)
    dt, dt_counts = pack_annos(dt_annos)
    up = lambda a, dt_=torch.float64: torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dt_)
    dt_count = up(dt_counts, torch.int32)
    out, ov = _launch(classes, up(gt), up(_offsets(gt_counts), torch.int32), gt_counts, up(dt), up(_offsets(dt_counts), torch.int32), dt_count,
                      dt_counts, dev)
    res = KittiEvalResult(classes, out.cpu().numpy())
    return (res, ov.cpu().numpy()) if return_overlaps else res


def get_official_eval_result(gt_annos, dt_annos, current_classes):
    """eval.py:608-678 -> (result_str, ret_dict), the same string and keys"""
    r = evaluate_annos(gt_annos, dt_annos, current_classes)
    return r.result_str, r.ret_dict


def evaluate(label_path, result_path, label_split_file, current_class=0):
    """evaluate.py:14-28: every result file of result_path against the labels of the split's image ids"""
    dt_annos = read_label_annos(result_path)
    with open(label_split_file, "r") as f:
        ids = [int(line) for line in f.readlines()]
    gt_annos = read_label_annos(label_path, ids)
    return get_official_eval_result(gt_annos, dt_annos, current_class)


# ------------------------------------------------------------------------------------------------ in memory
class KittiEvaluator:
    """Accumulates detections on the device and evaluates them against ground truth uploaded once.

        ev = KittiEvaluator(gt_annos, [0], "cuda")
        for batch: ev.add_batch(image_index, boxes3d, scores, select, P2, img_hw)     # no host synchronisation
        result_str, ret_dict = ev.result().result_str, ev.result().ret_dict

    Image k of the evaluation is gt_annos[k]; an image that receives no batch has no detections, and a second batch for
    the same image replaces the first."""

    def __init__(self, gt_annos, current_classes, device=None):
        self.classes = class_list(current_classes)
        self.device = _device(device)
        gt, self._gt_counts = pack_annos(gt_annos)
        self.n_img = len(gt_annos)
        self._gt = torch.from_numpy(gt).to(self.device)
        self._gt_off = torch.from_numpy(_offsets(self._gt_counts)).to(self.device, torch.int32)
        self._cap = 0
        self._dt = torch.zeros((self.n_img, 0, COLS), dtype=torch.float64, device=self.device)
        self._dt_off = torch.zeros(self.n_img + 1, dtype=torch.int32, device=self.device)
        self._dt_count = torch.zeros(self.n_img, dtype=torch.int32, device=self.device)

    def _reserve(self, m):
        if m <= self._cap:
            return
        if m > MAX_DET_PER_IMAGE:
            raise ValueError("KittiEvaluator: %d detection rows per scene > %d" % (m, MAX_DET_PER_IMAGE))
        grown = torch.zeros((self.n_img, m, COLS), dtype=torch.float64, device=self.device)
        grown[:, :self._cap] = self._dt
        self._dt, self._cap = grown, m
        self._dt_off = (torch.arange(self.n_img + 1, device=self.device, dtype=torch.int32) * m).contiguous()

    def add_batch(self, image_index, boxes3d, scores, select, P2, img_hw, text_rounding=True, classes="Car"):
        """boxes3d (B,M,7), scores (B,M) and select (B,M) as detections_device returns them; image_index: B image
        positions; P2 (B,3,4) and img_hw (B,2) [height, width], host arrays or tensors.  Keeps the rows save_kitti_format
        writes (selected, and narrower / lower than 0.8 of the image), named `classes`."""
        C.require_cuda(boxes3d, scores, select)
        B, M = int(boxes3d.shape[0]), int(boxes3d.shape[1])
        if len(image_index) != B:
            raise ValueError("KittiEvaluator.add_batch: %d image indices for %d scenes" % (len(image_index), B))
        idx = np.asarray(image_index, np.int64).reshape(-1)
        if B and (idx.min() < 0 or idx.max() >= self.n_img):
            raise IndexError("KittiEvaluator.add_batch: image index outside 0..%d" % (self.n_img - 1))
        self._reserve(M)
        dev = self.device
        up = lambda a: (a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a, np.float32))).to(
            dev, torch.float32, non_blocking=True).reshape(B, -1).contiguous()
        p2, hw = up(P2), up(img_hw)
        b = boxes3d.to(dev, torch.float32).contiguous()
        sc = scores.to(dev, torch.float32).contiguous()
        sel = select.to(dev, torch.int32).contiguous()
        slot = torch.from_numpy(idx.astype(np.int32)).to(dev, non_blocking=True)
        img_boxes = torch.empty((B, M, 4), dtype=torch.float32, device=dev)
        alpha = torch.empty((B, M), dtype=torch.float32, device=dev)
        valid = torch.empty((B, M), dtype=torch.int32, device=dev)
        lib = C.lib()
        with torch.cuda.device(dev):
            C.check(lib.prb_kitti_image_boxes_batch(B, M, C.ptr(b), C.ptr(p2), C.ptr(hw), C.ptr(img_boxes), C.ptr(alpha), C.ptr(valid), C.stream()),
                    "kitti_image_boxes_batch")
            C.check(lib.prb_kitti_eval_add_detections(B, M, C.ptr(b), C.ptr(sc), C.ptr(img_boxes), C.ptr(alpha), C.ptr(valid), C.ptr(sel),
                                                      C.ptr(slot), 1 if text_rounding else 0, class_code(classes), C.ptr(self._dt),
                                                      C.ptr(self._dt_off), C.ptr(self._dt_count), C.stream()), "kitti_eval_add_detections")

    def result(self, return_overlaps=False):
        """evaluate everything added so far: the device stages and ONE device-to-host copy -> KittiEvalResult"""
        caps = np.full(self.n_img, self._cap, np.int64)
        out, ov = _launch(self.classes, self._gt, self._gt_off, self._gt_counts, self._dt.view(-1, COLS), self._dt_off, self._dt_count,
                          caps, self.device)
        res = KittiEvalResult(self.classes, out.cpu().numpy())
        return (res, ov) if return_overlaps else res

"""Offline RCNN training samples on the device: the ROI_SAMPLE_JIT=False recipe (`--train_mode rcnn_offline`) of
lib/datasets/kitti_rcnn_dataset.py:876-1077 (get_rcnn_training_sample_batch), with the RPN features and proposals that
tools/eval_rcnn.py --save_rpn_feature saved.

The reference builds ONE scene per `__getitem__` in numpy: a shapely IoU matrix, a jitter loop of up to 10 shapely IoUs per
foreground RoI, roipool3d_cpu, a per-RoI data_augmentation call and a canonical transform.  Here a batch goes through
prb_boxes_iou3d, csrc/rcnn_sample.cu's sample stage, the roipool3d passes and the targets stage without a host
synchronisation:

    sampler = RCNNOfflineSampler()
    batch = sampler.prepare_batch(scenes, seed=step)        # dict of CUDA tensors, RoI axis flattened to B * ROI_PER_IMAGE
    loss, terms = trainer.step_offline(batch)

File IO: `read_rpn_features` / `read_rois` read what the reference reads; `write_rpn_features_batch` writes what
save_rpn_features writes, for a whole batch.  Differences from the reference (INTEGRATION.md): hashed draws, fp32 IoU,
the flat RoI layout, the fg-only branch, a status instead of pdb, roipool3d_kernel.cu's inside test.
"""
import os
import types

import numpy as np
import torch

from .. import _cabi as C
from .kitti_eval import read_label_anno

# tools/cfgs/default.yaml:6-9, :60-122
DEFAULT_CFG = dict(AUG_DATA=True, AUG_METHOD_LIST=["rotation", "scaling", "flip"], AUG_METHOD_PROB=[1.0, 1.0, 0.5], AUG_ROT_RANGE=18,
                   RCNN=dict(USE_INTENSITY=False, USE_DEPTH=True, USE_SEG_SCORE=False, POOL_EXTRA_WIDTH=1.0, NUM_POINTS=512,
                             REG_AUG_METHOD="multiple", CLS_FG_THRESH=0.6, CLS_BG_THRESH=0.45, CLS_BG_THRESH_LO=0.05,
                             REG_FG_THRESH=0.55, FG_RATIO=0.5, ROI_PER_IMAGE=64, HARD_BG_RATIO=0.8))
AUG_METHODS = {"single": 0, "multiple": 1, "normal": 2}
# aug_roi_by_noise_batch is called with aug_times=10 for the foreground rows (kitti_rcnn_dataset.py:942), not ROI_FG_AUG_TIMES
FG_AUG_TIMES = 10
# coordinate of padding points: outside every box (the inside test rejects |dx| > 10), and ignored by the bounds of
# roipool3d's point grid, which only finite coordinates set
FAR = float("inf")


def _boxes7(b):
    """(n, 7 or more) boxes, or a flat empty array -> (n, 7) [x, y, z, h, w, l, ry]"""
    return (b.reshape(-1, b.shape[-1]) if b.ndim == 2 else b.reshape(-1, 7))[:, :7]


def _pad(ts, n, value):
    """list of (n_k, c) tensors -> (len, n, c), rows n_k.. filled with value"""
    out = torch.nn.utils.rnn.pad_sequence(ts, batch_first=True, padding_value=value)
    return out if out.shape[1] == n else torch.nn.functional.pad(out, (0, 0, 0, n - out.shape[1]), value=value)


def _ns(d):
    return types.SimpleNamespace(**{k: (_ns(v) if isinstance(v, dict) else v) for k, v in d.items()})


# ------------------------------------------------------------------------------------------------ files
def read_rpn_features(feature_dir, sample_id, use_seg_score=False):
    """get_rpn_features (kitti_rcnn_dataset.py:139-150) -> rpn_xyz (N,3), rpn_features (N,C), rpn_intensity (N,), seg (N,):
    the saved segmentation mask, or sigmoid of the raw scores with use_seg_score"""
    f = lambda suffix: os.path.join(feature_dir, "%06d%s.npy" % (sample_id, suffix))
    if use_seg_score:
        seg = torch.sigmoid(torch.from_numpy(np.load(f("_rawscore")).reshape(-1))).numpy()
    else:
        seg = np.load(f("_seg")).reshape(-1)
    return np.load(f("_xyz")), np.load(f("")), np.load(f("_intensity")).reshape(-1), seg


def read_rois(roi_dir, sample_id, with_scores=False):
    """the proposals of one scene from a KITTI result file -> (M,7) float32 [x, y, z, h, w, l, ry] (objs_to_boxes3d);
    with_scores: also the (M,) float32 score column, as get_proposal_from_file reads it (kitti_rcnn_dataset.py:800-803)"""
    a = read_label_anno(os.path.join(roi_dir, "%06d.txt" % sample_id))
    out = np.zeros((len(a["name"]), 7), np.float32)
    if len(out):
        out[:, 0:3] = a["location"]
        out[:, 3:6] = a["dimensions"][:, [1, 2, 0]]      # the parser stores l, h, w
        out[:, 6] = a["rotation_y"]
    if with_scores:
        return out, np.asarray(a["score"], np.float32).reshape(-1)
    return out


def write_rpn_features_batch(feature_dir, sample_ids, seg, rawscore, intensity, xyz, features):
    """save_rpn_features (tools/eval_rcnn.py:97-110) for a batch: seg (B,N), rawscore (B,N), intensity (B,N), xyz (B,N,3),
    features (B,C,N) as the backbone returns them -> per scene %06d.npy (N,C), _xyz, _seg, _intensity, _rawscore, float32.
    One device-to-host copy for CUDA tensors; CPU tensors and numpy arrays are written as they are."""
    B = len(sample_ids)
    parts = [torch.as_tensor(t).float().reshape(B, -1) for t in (seg, rawscore, intensity, xyz, features)]
    sizes = [p.shape[1] for p in parts]
    host = torch.cat(parts, 1).cpu().numpy() if parts[0].is_cuda else torch.cat(parts, 1).numpy()
    n = sizes[0]
    c = sizes[4] // n
    offs = np.cumsum([0] + sizes)
    os.makedirs(feature_dir, exist_ok=True)
    for k, sid in enumerate(sample_ids):
        row = host[k]
        s, raw, inten, x, feat = (row[offs[j]:offs[j + 1]] for j in range(5))
        p = lambda suffix: os.path.join(feature_dir, "%06d%s.npy" % (sid, suffix))
        np.save(p(""), feat.reshape(c, n).T)          # the transposed (C, N) view: a Fortran-order file, as the reference writes
        np.save(p("_xyz"), x.reshape(n, 3))
        np.save(p("_seg"), s)
        np.save(p("_intensity"), inten)
        np.save(p("_rawscore"), raw)


# ------------------------------------------------------------------------------------------------ sampler
class RCNNOfflineSampler:
    """get_rcnn_training_sample_batch for a batch of scenes on the device.  cfg: the reference's global cfg (or any object
    with its AUG_* and RCNN.* keys); None -> lib.config.cfg inside the reference tree, else tools/cfgs/default.yaml."""

    def __init__(self, cfg=None, device=None):
        if cfg is None:
            try:
                from lib.config import cfg as ref_cfg
                cfg = ref_cfg
            except ImportError:
                cfg = _ns(DEFAULT_CFG)
        self.cfg = cfg
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type != "cuda":
            raise RuntimeError("pointrcnn_b200: the offline RCNN sampler runs on a CUDA device (there is no CPU path)")
        r = cfg.RCNN
        if r.REG_AUG_METHOD not in AUG_METHODS:
            raise NotImplementedError(r.REG_AUG_METHOD)
        self.num_extra = int(r.USE_INTENSITY) + 1 + int(r.USE_DEPTH)

    def _pack_host(self, scenes, B, N, M, G, E, Cf):
        """numpy scenes -> one float32 host buffer [xyz | features | rois | gt | counts (int32 bits)], uploaded once"""
        r = self.cfg.RCNN
        sizes = [B * N * 3, B * N * (E + Cf), B * M * 7, B * G * 7, 2 * B]
        offs = np.cumsum([0] + sizes)
        buf = np.zeros(int(offs[-1]), np.float32)
        xyz = buf[offs[0]:offs[1]].reshape(B, N, 3)
        feat = buf[offs[1]:offs[2]].reshape(B, N, E + Cf)
        rois = buf[offs[2]:offs[3]].reshape(B, M, 7)
        gt = buf[offs[3]:offs[4]].reshape(B, G, 7)
        counts = buf[offs[4]:offs[5]].view(np.int32).reshape(2, B)
        xyz[:] = FAR
        for k, s in enumerate(scenes):
            p = np.asarray(s["rpn_xyz"], np.float32)
            n = len(p)
            xyz[k, :n] = p
            col = 0
            if r.USE_INTENSITY:
                feat[k, :n, col] = np.asarray(s["rpn_intensity"], np.float32).reshape(-1)
                col += 1
            feat[k, :n, col] = np.asarray(s["seg_mask"], np.float32).reshape(-1)
            col += 1
            if r.USE_DEPTH:
                feat[k, :n, col] = np.linalg.norm(p, ord=2, axis=1) / 70.0 - 0.5
            feat[k, :n, E:] = np.asarray(s["rpn_features"], np.float32)
            rb, gb = _boxes7(np.asarray(s["roi_boxes3d"], np.float32)), _boxes7(np.asarray(s["gt_boxes3d"], np.float32))
            rois[k, :len(rb)] = rb
            gt[k, :len(gb)] = gb
            counts[0, k], counts[1, k] = len(rb), len(gb)
        dev = torch.from_numpy(buf).to(self.device)
        return (dev[offs[0]:offs[1]].view(B, N, 3), dev[offs[1]:offs[2]].view(B, N, E + Cf), dev[offs[2]:offs[3]].view(B, M, 7),
                dev[offs[3]:offs[4]].view(B, G, 7), dev[offs[4]:offs[5]].view(torch.int32).view(2, B))

    def _pack_device(self, scenes, B, N, M, G, E, Cf):
        """CUDA scenes -> padded batch tensors with batch-wide torch ops on the current stream (no host round trip)"""
        r = self.cfg.RCNN
        dev = self.device
        t = lambda v: torch.as_tensor(v, device=dev).float()
        ps = [t(s["rpn_xyz"]).reshape(-1, 3) for s in scenes]
        xyz = _pad(ps, N, FAR)
        cols = [_pad([t(s["rpn_intensity"]).reshape(-1, 1) for s in scenes], N, 0.0)] if r.USE_INTENSITY else []
        cols.append(_pad([t(s["seg_mask"]).reshape(-1, 1) for s in scenes], N, 0.0))
        if r.USE_DEPTH:      # padding rows get an infinite depth; no box contains them, so it is never pooled
            cols.append(torch.linalg.vector_norm(xyz, ord=2, dim=2, keepdim=True) / 70.0 - 0.5)
        feat = torch.cat(cols + [_pad([t(s["rpn_features"]) for s in scenes], N, 0.0)], dim=2)
        rb = [_boxes7(t(s["roi_boxes3d"])) for s in scenes]
        gb = [_boxes7(t(s["gt_boxes3d"])) for s in scenes]
        counts = np.array([[b.shape[0] for b in rb], [b.shape[0] for b in gb]], np.int32)
        return xyz, feat, _pad(rb, M, 0.0), _pad(gb, G, 0.0), torch.from_numpy(counts).to(dev, non_blocking=True)

    def _dims(self, scenes, what):
        """-> B, N, M, G, C of a batch (M, G at least 1) and the packer for where its arrays live"""
        B = len(scenes)
        if B == 0:
            raise ValueError("%s: empty batch" % what)
        on_device = all(torch.is_tensor(s["rpn_xyz"]) and s["rpn_xyz"].is_cuda for s in scenes)
        shape = lambda v: tuple(v.shape)
        N = max(shape(s["rpn_xyz"])[0] for s in scenes)
        Cf = shape(scenes[0]["rpn_features"])[1]
        rows = lambda v: shape(v)[0] if len(shape(v)) == 2 else int(np.prod(shape(v))) // 7
        M = max(max(rows(s["roi_boxes3d"]) for s in scenes), 1)
        G = max(max(rows(s["gt_boxes3d"]) for s in scenes), 1)
        for s in scenes:
            if shape(s["rpn_features"])[1] != Cf or shape(s["rpn_features"])[0] != shape(s["rpn_xyz"])[0]:
                raise ValueError("%s: rpn_features must be (N, C) with one C for the batch" % what)
        return B, N, M, G, Cf, (self._pack_device if on_device else self._pack_host)

    def prepare_eval_batch(self, scenes):
        """get_proposal_from_file (kitti_rcnn_dataset.py:790-874) for a batch, no sampling and no augmentation: every
        proposal is pooled on its enlarged box with the canonical transform (RCNNStage.pool, rcnn_net.py:127-152, the
        reference's default ROI_SAMPLE_JIT eval), and gt_iou is each proposal's max 3D IoU over the scene's GT (0 without GT).
        scenes: dicts rpn_xyz (N,3), rpn_features (N,C), rpn_intensity (N,), seg_mask (N,), roi_boxes3d (M,7), roi_scores
        (M,) (optional), gt_boxes3d (G,7), numpy or CUDA.  -> dict of CUDA tensors: rows (B*M, NUM_POINTS, 3 + extra + C),
        roi_boxes3d (B,M,7), roi_scores (B,M), roi_count (B) int32, gt_boxes3d (B,G,7), gt_count (B) int32, gt_iou (B,M),
        pooled_empty_flag (B,M) int32.  Padding RoIs (rows past roi_count) are zero boxes with gt_iou 0."""
        from ..roipool3d import roipool3d_utils
        r = self.cfg.RCNN
        B, N, M, G, Cf, pack = self._dims(scenes, "prepare_eval_batch")
        dev = self.device
        with torch.cuda.device(dev):
            xyz, feat, rois, gt, counts = pack(scenes, B, N, M, G, self.num_extra, Cf)
            if pack == self._pack_device:
                score = lambda s: s["roi_scores"] if s.get("roi_scores") is not None else torch.zeros(s["roi_boxes3d"].shape[0], device=dev)
                scores = _pad([torch.as_tensor(score(s), device=dev).float().reshape(-1, 1) for s in scenes], M, 0.0)
                scores = scores.view(B, M)
            else:
                host = np.zeros((B, M), np.float32)
                for k, s in enumerate(scenes):
                    if s.get("roi_scores") is not None:
                        v = np.asarray(s["roi_scores"], np.float32).reshape(-1)
                        host[k, :len(v)] = v
                scores = torch.from_numpy(host).to(dev)
            pooled, empty = roipool3d_utils.roipool3d_gpu(xyz, feat, rois, r.POOL_EXTRA_WIDTH, sampled_pt_num=int(r.NUM_POINTS),
                                                          canonical_rois=rois)
            gt_iou = torch.empty((B, M), dtype=torch.float32, device=dev)
            C.check(C.lib().prb_eval_box_recall(B, M, C.ptr(rois), C.ptr(counts[0]), G, C.ptr(gt), C.ptr(counts[1]), 0, None, None, None,
                                                C.ptr(gt_iou), C.stream()), "eval_box_recall")
        return {"rows": pooled.view(B * M, pooled.shape[2], pooled.shape[3]), "roi_boxes3d": rois, "roi_scores": scores,
                "roi_count": counts[0], "gt_boxes3d": gt, "gt_count": counts[1], "gt_iou": gt_iou, "pooled_empty_flag": empty}

    def prepare_batch(self, scenes, seed=0, mode="TRAIN"):
        """scenes: list of dicts rpn_xyz (N,3), rpn_features (N,C), rpn_intensity (N,), seg_mask (N,), roi_boxes3d (M,7),
        gt_boxes3d (G,7), numpy or CUDA.  -> dict of CUDA tensors over the flat RoI axis K = B * ROI_PER_IMAGE:
        rows (K, NUM_POINTS, 3 + extra + C) the pooled buffer; pts_input / pts_features its [xyz | extra] / feature views;
        cls_label (K) int32, reg_valid_mask (K) int32, gt_boxes3d_ct (K,7), roi_boxes3d (K,7), roi_size (K,3), gt_boxes3d
        (K,7), gt_iou (K), sample_status (B) int32, sample_index (K,3) int32 [source RoI, GT, jitter tries]."""
        cfg, r = self.cfg, self.cfg.RCNN
        B, N, M, G, Cf, pack = self._dims(scenes, "prepare_batch")
        dev = self.device
        E, R, S = self.num_extra, int(r.ROI_PER_IMAGE), int(r.NUM_POINTS)
        with torch.cuda.device(dev):
            xyz, feat, rois, gt, counts = pack(scenes, B, N, M, G, E, Cf)
            L, st = C.lib(), C.stream()
            iou = torch.empty((B, M, G), dtype=torch.float32, device=dev)
            C.check(L.prb_boxes_iou3d(B, M, C.ptr(rois), G, C.ptr(gt), C.ptr(iou), st), "boxes_iou3d")
            f = lambda *shp: torch.empty(shp, dtype=torch.float32, device=dev)
            rois_out, gt_out, iou_out, pool_boxes = f(B, R, 7), f(B, R, 7), f(B, R), f(B, R, 7)
            sel = torch.empty((B, R, 3), dtype=torch.int32, device=dev)
            status = torch.empty(B, dtype=torch.int32, device=dev)
            fg_quota = int(np.round(r.FG_RATIO * R))
            C.check(L.prb_rcnn_sample_rois(B, M, G, C.ptr(iou), C.ptr(rois), C.ptr(counts[0]), C.ptr(gt), C.ptr(counts[1]), R, fg_quota,
                                           r.REG_FG_THRESH, r.CLS_FG_THRESH, r.CLS_BG_THRESH, r.CLS_BG_THRESH_LO, r.HARD_BG_RATIO,
                                           AUG_METHODS[r.REG_AUG_METHOD], FG_AUG_TIMES, r.POOL_EXTRA_WIDTH, seed & 0xffffffff,
                                           C.ptr(rois_out), C.ptr(gt_out), C.ptr(iou_out), C.ptr(pool_boxes), C.ptr(sel), C.ptr(status),
                                           st), "rcnn_sample_rois")
            W = 3 + E + Cf
            pooled = f(B, R, S, W)
            empty = torch.zeros((B, R), dtype=torch.int32, device=dev)
            wsb = L.prb_roipool3d_workspace_bytes(B, N, R, S)
            ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
            C.check(L.prb_roipool3d_ws(B, N, R, E + Cf, S, C.ptr(xyz), C.ptr(pool_boxes), C.ptr(feat), C.ptr(pooled), C.ptr(empty),
                                       None, 1, C.ptr(ws), C.c_size_t(wsb), st), "roipool3d")
            aug = bool(cfg.AUG_DATA) and mode == "TRAIN"
            methods = list(cfg.AUG_METHOD_LIST)
            gt_ct = f(B * R, 7)
            cls = torch.empty(B * R, dtype=torch.int32, device=dev)
            reg = torch.empty(B * R, dtype=torch.int32, device=dev)
            C.check(L.prb_rcnn_roi_targets(B, R, S, W, C.ptr(pooled), C.ptr(rois_out), C.ptr(gt_out), C.ptr(iou_out), C.ptr(empty),
                                           int(aug), int("rotation" in methods), int("scaling" in methods), int("flip" in methods),
                                           float(cfg.AUG_ROT_RANGE), float(cfg.AUG_METHOD_PROB[2]), r.REG_FG_THRESH, r.CLS_FG_THRESH,
                                           r.CLS_BG_THRESH, seed & 0xffffffff, C.ptr(gt_ct), C.ptr(cls), C.ptr(reg), st), "rcnn_roi_targets")
        rows = pooled.view(B * R, S, W)
        rois_flat = rois_out.view(B * R, 7)
        return {"rows": rows, "pts_input": rows[..., :3 + E], "pts_features": rows[..., 3 + E:], "cls_label": cls,
                "reg_valid_mask": reg, "gt_boxes3d_ct": gt_ct, "roi_boxes3d": rois_flat, "roi_size": rois_flat[:, 3:6],
                "gt_boxes3d": gt_out.view(B * R, 7), "gt_iou": iou_out.view(B * R), "sample_status": status,
                "sample_index": sel.view(B * R, 3), "pooled_empty_flag": empty.view(B * R)}

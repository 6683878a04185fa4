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

The in-network recipe (ROI_SAMPLE_JIT=True, the shipped default.yaml) reads the same files through
get_rcnn_sample_jit + collate_batch and samples inside the network; here:

    batch = sampler.prepare_jit_batch(scenes)               # padded input dict of CUDA tensors
    loss, terms = trainer.step_jit(batch)                   # ProposalTargetLayer inside RCNNStage.forward_train

File IO: `read_rpn_features` / `read_rois` read what the reference reads; `write_rpn_features_batch` writes what
save_rpn_features writes, for a whole batch.  Differences from the reference (INTEGRATION.md): hashed draws, fp32 IoU,
the flat RoI layout, the fg-only branch, a status instead of pdb, roipool3d_kernel.cu's inside test.
"""
import os

import numpy as np
import torch

from .. import _cabi as C
from ..rcnn import targets
from ..rcnn.targets import AUG_METHODS, DEFAULT_CFG, ns as _ns  # the names this module has always exported
from .kitti_eval import read_label_anno

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


# ------------------------------------------------------------------------------------------------ in-network recipe
def pack_jit_scenes(scenes):
    """get_rcnn_sample_jit (kitti_rcnn_dataset.py:1079-1102) + collate_batch (:1104-1137) for numpy scenes, into ONE float32
    host buffer.  scenes: dicts rpn_xyz (N,3), rpn_features (N,C), rpn_intensity (N,), seg_mask (N,), roi_boxes3d (M,7),
    gt_boxes3d (G,7).  -> (buffer, dict of views of it): rpn_xyz (B,N,3), rpn_features (B,N,C), rpn_intensity (B,N),
    seg_mask (B,N), pts_depth (B,N) = ||xyz|| (np.linalg.norm in float32, as get_rcnn_sample_jit), roi_boxes3d (B,M,7) and
    gt_boxes3d (B,G,7) zero-padded to the batch's longest list (M or G is 0 when every list is empty), roi_count /
    gt_count (B) int32 (the int32 bits of float32 slots).  collate_batch stacks the point arrays and so needs one N for
    the batch; a shorter scene is padded here with points at infinity (depth inf), which no box contains."""
    B = len(scenes)
    if B == 0:
        raise ValueError("pack_jit_scenes: empty batch")
    N = max(len(s["rpn_xyz"]) for s in scenes)
    Cf = np.shape(scenes[0]["rpn_features"])[1]
    rb = [_boxes7(np.asarray(s["roi_boxes3d"], np.float32)) for s in scenes]
    gb = [_boxes7(np.asarray(s["gt_boxes3d"], np.float32)) for s in scenes]
    M, G = max(len(b) for b in rb), max(len(b) for b in gb)
    layout = _jit_layout(B, N, Cf, M, G)
    buf = np.zeros(sum(int(np.prod(shape)) for _, shape in layout), np.float32)
    v = _jit_views(buf, layout, lambda a: a.view(np.int32))
    v["rpn_xyz"][:] = FAR
    v["pts_depth"][:] = FAR
    for k, s in enumerate(scenes):
        p = np.asarray(s["rpn_xyz"], np.float32).reshape(-1, 3)
        n = len(p)
        if np.shape(s["rpn_features"]) != (n, Cf):
            raise ValueError("pack_jit_scenes: rpn_features must be (N, C) with one C for the batch")
        v["rpn_xyz"][k, :n] = p
        v["rpn_features"][k, :n] = s["rpn_features"]
        v["rpn_intensity"][k, :n] = np.asarray(s["rpn_intensity"], np.float32).reshape(-1)
        v["seg_mask"][k, :n] = np.asarray(s["seg_mask"], np.float32).reshape(-1)
        v["pts_depth"][k, :n] = np.linalg.norm(p, ord=2, axis=1)
        v["roi_boxes3d"][k, :len(rb[k])] = rb[k]
        v["gt_boxes3d"][k, :len(gb[k])] = gb[k]
        v["roi_count"][k], v["gt_count"][k] = len(rb[k]), len(gb[k])
    return buf, v


def _jit_layout(B, N, Cf, M, G):
    return [("rpn_xyz", (B, N, 3)), ("rpn_features", (B, N, Cf)), ("rpn_intensity", (B, N)), ("seg_mask", (B, N)), ("pts_depth", (B, N)),
            ("roi_boxes3d", (B, M, 7)), ("gt_boxes3d", (B, G, 7)), ("roi_count", (B,)), ("gt_count", (B,))]


def _jit_views(flat, layout, as_int32):
    """views of a flat float32 array (numpy or torch) in the order of layout; the counts as int32 bits"""
    out, o = {}, 0
    for k, shape in layout:
        n = int(np.prod(shape))
        a = flat[o:o + n]
        out[k] = (as_int32(a) if k.endswith("_count") else a).reshape(shape)
        o += n
    return out


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

    def prepare_jit_batch(self, scenes):
        """get_rcnn_sample_jit + collate_batch for a batch (pack_jit_scenes): the input dict of the in-network recipe, for
        RCNNTrainer.step_jit (or the reference's rcnn_net under dropin.activate()), whose ProposalTargetLayer samples the
        RoIs: every row of roi_boxes3d is a candidate there, zero padding included (IoU 0: easy background, as in the
        reference).  numpy scenes go up in one copy; CUDA scenes are padded with batch-wide torch ops.  -> dict of CUDA
        tensors rpn_xyz (B,N,3), rpn_features (B,N,C), rpn_intensity (B,N), seg_mask (B,N), pts_depth (B,N), roi_boxes3d
        (B,M,7), gt_boxes3d (B,G,7), roi_count (B) int32, gt_count (B) int32."""
        if len(scenes) == 0:
            raise ValueError("prepare_jit_batch: empty batch")
        dev = self.device
        if not all(torch.is_tensor(s["rpn_xyz"]) and s["rpn_xyz"].is_cuda for s in scenes):
            buf, host = pack_jit_scenes(scenes)
            layout = [(k, a.shape) for k, a in host.items()]
            return _jit_views(torch.from_numpy(buf).to(dev), layout, lambda a: a.view(torch.int32))
        t = lambda v: torch.as_tensor(v, device=dev).float()
        N = max(s["rpn_xyz"].shape[0] for s in scenes)
        xyz = _pad([t(s["rpn_xyz"]).reshape(-1, 3) for s in scenes], N, FAR)
        col = lambda key: _pad([t(s[key]).reshape(-1, 1) for s in scenes], N, 0.0).squeeze(2)
        rb = [_boxes7(t(s["roi_boxes3d"])) for s in scenes]
        gb = [_boxes7(t(s["gt_boxes3d"])) for s in scenes]
        M, G = max(b.shape[0] for b in rb), max(b.shape[0] for b in gb)
        counts = torch.from_numpy(np.array([[b.shape[0] for b in rb], [b.shape[0] for b in gb]], np.int32)).to(dev, non_blocking=True)
        return {"rpn_xyz": xyz, "rpn_features": _pad([t(s["rpn_features"]) for s in scenes], N, 0.0), "rpn_intensity": col("rpn_intensity"),
                "seg_mask": col("seg_mask"), "pts_depth": torch.linalg.vector_norm(xyz, ord=2, dim=2), "roi_boxes3d": _pad(rb, M, 0.0),
                "gt_boxes3d": _pad(gb, G, 0.0), "roi_count": counts[0], "gt_count": counts[1]}

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
        B, N, M, G, Cf, pack = self._dims(scenes, "prepare_batch")
        recipe = targets.loader_recipe(self.cfg, mode)
        E, R = self.num_extra, recipe.roi_per_image
        with torch.cuda.device(self.device):
            xyz, feat, rois, gt, counts = pack(scenes, B, N, M, G, E, Cf)
            o = targets.run(recipe, xyz, feat, rois, gt, counts, seed)
        rows = o["pooled"].view(B * R, recipe.num_points, 3 + E + Cf)
        rois_flat = o["rois"].view(B * R, 7)
        return {"rows": rows, "pts_input": rows[..., :3 + E], "pts_features": rows[..., 3 + E:], "cls_label": o["cls"],
                "reg_valid_mask": o["reg"], "gt_boxes3d_ct": o["gt_ct"], "roi_boxes3d": rois_flat, "roi_size": rois_flat[:, 3:6],
                "gt_boxes3d": o["gts"].view(B * R, 7), "gt_iou": o["iou"].view(B * R), "sample_status": o["status"],
                "sample_index": o["sel"].view(B * R, 3), "pooled_empty_flag": o["empty"].view(B * R)}

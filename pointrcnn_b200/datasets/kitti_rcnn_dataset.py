"""RPN input pipeline on the device: mirror of lib/datasets/kitti_rcnn_dataset.py:246-394 (get_rpn_sample,
generate_rpn_training_labels), :198-219 (get_valid_flag), :513-570 (data_augmentation, stage 1) and :1104-1137
(collate_batch) -- SURVEY.md 8(f) rank 4.

The reference prepares ONE scene per `__getitem__` in numpy (calibration products, a boolean-mask compaction, np.random
draws, two Delaunay triangulations per GT box for the labels) and stacks scenes in `collate_batch`.  Here a whole batch
of raw scans goes through four launches (csrc/kitti_io.cu) and comes out as the tensors the network and the loss read:

    pipe = RPNInputPipeline(npoints=16384, mode="TRAIN")
    batch = pipe.prepare_batch(scans, seed=step)          # dict of CUDA tensors, same keys as collate_batch

File IO (KITTI .bin / calib / label / plane readers, the GT-paste database pickle) stays with the caller: a scan is
`dict(lidar=(n,4) float32 numpy array or (pinned) torch tensor, calib=Calibration|dict, img_shape=(H,W[,3]),
gt_boxes3d=(g,7), gt_alpha=(g,))`, plus for GT-paste (TRAIN with `gt_database=GTDatabase...`) `road_plane=(4,)` as
get_road_plane returns it and optionally `all_gt_boxes3d=(m,7)`, the collision list (default: gt_boxes3d).  GT-paste adds
two launches (csrc/gt_paste.cu) between the validity flags and the npoints draw.

Two ways to draw the npoints sample:
  draw="device" (default)  counter-based hashes on the device, no host round trip; same distribution as the reference
  draw="numpy"             the reference's own np.random calls in the reference's order (needs the valid flags on the
                           host): bit-for-bit the reference's sample for a given np.random state -- used by the parity tests
There is no CPU path: the kernels are required (RuntimeError without the library / a CUDA device).
"""
import ctypes

import numpy as np
import torch

from .. import _cabi as C

PC_AREA_SCOPE = ((-40.0, 40.0), (-1.0, 3.0), (0.0, 70.4))      # tools/cfgs/default.yaml:18


class Calibration(object):
    """lib/utils/calibration.py:24-41 for an in-memory dict {'P2','R0','Tr_velo2cam'} (fp32 like get_calib_from_file)"""

    def __init__(self, calib):
        if isinstance(calib, Calibration):
            calib = dict(P2=calib.P2, R0=calib.R0, Tr_velo2cam=calib.V2C)
        self.P2 = np.asarray(calib["P2"], dtype=np.float32).reshape(3, 4)
        self.R0 = np.asarray(calib["R0"], dtype=np.float32).reshape(3, 3)
        self.V2C = np.asarray(calib["Tr_velo2cam"], dtype=np.float32).reshape(3, 4)

    def lidar_to_rect_matrix(self):
        """(4,3) fp32: rect = [x y z 1] . M  (calibration.py:57: np.dot(self.V2C.T, self.R0.T))"""
        return np.dot(self.V2C.T, self.R0.T).astype(np.float32)

    def pack(self, img_shape, scope=None):
        row = np.zeros(32, dtype=np.float32)
        row[0:12] = self.lidar_to_rect_matrix().reshape(-1)
        row[12:24] = self.P2.reshape(-1)
        row[24], row[25] = float(img_shape[0]), float(img_shape[1])
        if scope is not None:
            row[26:32] = np.asarray(scope, dtype=np.float32).reshape(-1)
        return row


def _dev(device):
    device = torch.device(device if device is not None else "cuda")
    if device.type != "cuda":
        raise RuntimeError("pointrcnn_b200: the input pipeline runs on a CUDA device (there is no CPU path)")
    return device


def _i32(t):
    return t if t.dtype == torch.int32 else t.to(torch.int32)


def generate_rpn_training_labels(pts_rect, gt_boxes3d, extra_width=0.2, gt_count=None):
    """kitti_rcnn_dataset.py:355-391.  numpy (N,3),(G,7) -> numpy (N,) int32, (N,7) float32 like the reference's static
    method; CUDA tensors (B,N,3),(B,G,7) -> CUDA tensors (B,N) int32, (B,N,7) (batched, zero rows of a padded batch skipped
    unless gt_count (B,) says how many rows are real)."""
    as_numpy = isinstance(pts_rect, np.ndarray)
    if as_numpy:
        dev = _dev(None)
        p = torch.from_numpy(np.ascontiguousarray(pts_rect, dtype=np.float32)).to(dev).unsqueeze(0)
        g = torch.from_numpy(np.ascontiguousarray(gt_boxes3d, dtype=np.float32).reshape(-1, 7)).to(dev).unsqueeze(0)
        gt_count = torch.tensor([g.size(1)], dtype=torch.int32, device=dev)
    else:
        p, g = pts_rect.contiguous(), gt_boxes3d.contiguous()
        C.require_cuda(p, g)
        if p.dtype != torch.float32 or g.dtype != torch.float32:
            raise RuntimeError("generate_rpn_training_labels: float32 tensors expected")
    B, N, _ = p.shape
    G = g.size(1)
    cls = torch.empty((B, N), dtype=torch.int32, device=p.device)
    reg = torch.empty((B, N, 7), dtype=torch.float32, device=p.device)
    if gt_count is not None:
        gt_count = _i32(gt_count.to(p.device)).contiguous()
    with torch.cuda.device(p.device):
        C.check(C.lib().prb_rpn_training_labels(B, N, G, C.ptr(p), C.ptr(g) if G else None, C.ptr(gt_count),
                                                ctypes.c_float(extra_width), C.ptr(cls), C.ptr(reg), C.stream()), "rpn_training_labels")
    if as_numpy:
        return cls[0].cpu().numpy(), reg[0].cpu().numpy()
    return cls, reg


def draw_augmentation(rng=np.random, aug_list=("rotation", "scaling", "flip"),
                      aug_prob=(0.5, 0.5, 0.5), rot_range=18, mustaug=False):
    """the random draws of data_augmentation (kitti_rcnn_dataset.py:520-568) in the reference's order:
    -> (angle or None, scale or None, flip bool, aug_method list)"""
    aug_enable = 1 - rng.rand(3)
    if mustaug:
        aug_enable[0] = aug_enable[1] = -1
    angle = scale = None
    flip = False
    method = []
    if "rotation" in aug_list and aug_enable[0] < aug_prob[0]:
        angle = rng.uniform(-np.pi / rot_range, np.pi / rot_range)
        method.append(["rotation", angle])
    if "scaling" in aug_list and aug_enable[1] < aug_prob[1]:
        scale = rng.uniform(0.95, 1.05)
        method.append(["scaling", scale])
    if "flip" in aug_list and aug_enable[2] < aug_prob[2]:
        flip = True
        method.append("flip")
    return angle, scale, flip, method


def augment_gt_boxes3d(gt_boxes3d, gt_alpha, angle, scale, flip):
    """the GT-box half of data_augmentation (stage 1): a handful of boxes per scene, host numpy with the reference's
    float64 intermediates (kitti_rcnn_dataset.py:528-560, kitti_utils.py:32-42)"""
    b = np.array(gt_boxes3d, dtype=np.float32, copy=True)
    if angle is not None and b.shape[0]:
        c, s = np.cos(angle), np.sin(angle)
        x, z = b[:, 0].astype(np.float64), b[:, 2].astype(np.float64)
        b[:, 0], b[:, 2] = x * c - z * s, x * s + z * c
        beta = np.arctan2(b[:, 2], b[:, 0])
        b[:, 6] = np.sign(beta) * np.pi / 2 + gt_alpha - beta
    if scale is not None:
        b[:, 0:6] = b[:, 0:6] * scale
    if flip:
        b[:, 0] = -b[:, 0]
        b[:, 6] = np.sign(b[:, 6]) * np.pi - b[:, 6]
    return b


def draw_choice_numpy(pts_depth, npoints, rng=np.random):
    """the npoints draw of kitti_rcnn_dataset.py:285-303 with the reference's np.random calls in its order;
    pts_depth = rect z of the VALID points; returns indices into the valid points"""
    n = len(pts_depth)
    if npoints < n:
        near = pts_depth < 40.0
        far_idxs = np.where(near == 0)[0]
        near_idxs = np.where(near == 1)[0]
        picked = rng.choice(near_idxs, npoints - len(far_idxs), replace=False)
        choice = np.concatenate((picked, far_idxs), axis=0) if len(far_idxs) > 0 else picked
        rng.shuffle(choice)
    else:
        choice = np.arange(0, n, dtype=np.int32)
        if npoints > n:
            extra = rng.choice(choice, npoints - n, replace=False)
            choice = np.concatenate((choice, extra), axis=0)
        rng.shuffle(choice)
    return choice


class GTDatabase(object):
    """the GT-paste database (tools/generate_gt_database.py:72-84, loaded at kitti_rcnn_dataset.py:64-80), device resident:
    points (P,4) [rect x, y, z, intensity] of all entries back to back, offsets (E+1), boxes (E,7), alpha (E,), and the
    easy (> 100 points) / hard (<= 100 points) entry lists the reference splits the database into when
    GT_AUG_HARD_RATIO > 0.  The boxes, counts and alpha stay on the host for the candidate draw; the points are uploaded
    once, by upload() (RPNInputPipeline calls it)."""

    def __init__(self, boxes, points, counts, alpha):
        self.boxes = np.ascontiguousarray(boxes, dtype=np.float32).reshape(-1, 7)
        self.counts = np.asarray(counts, dtype=np.int64).reshape(-1)
        self.alpha = np.ascontiguousarray(alpha, dtype=np.float32).reshape(-1)
        pts = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 4)
        E = len(self.boxes)
        if len(self.counts) != E or len(self.alpha) != E or int(self.counts.sum()) != len(pts):
            raise ValueError("GTDatabase: boxes, counts, alpha and points disagree")
        self.offsets = np.zeros(E + 1, dtype=np.int64)
        self.offsets[1:] = np.cumsum(self.counts)
        if self.offsets[-1] >= 2 ** 31:
            raise ValueError("GTDatabase: more than 2^31 points")
        self.easy = np.nonzero(self.counts > 100)[0]
        self.hard = np.nonzero(self.counts <= 100)[0]
        self.host_points = pts
        self.points = None
        self._eligible = {}

    def upload(self, device=None):
        """the points to the device, once"""
        dev = _dev(device)
        if self.points is None or self.points.device != dev:
            pts = self.host_points if len(self.host_points) else np.zeros((1, 4), np.float32)
            self.points = torch.from_numpy(pts).to(dev)
        return self

    def __len__(self):
        return len(self.boxes)

    @classmethod
    def from_arrays(cls, boxes, points, alpha):
        """boxes (E,7), points: a list of E (n_e,4) arrays [rect x, y, z, intensity], alpha (E,)"""
        counts = [len(p) for p in points]
        packed = np.concatenate([np.asarray(p, np.float32).reshape(-1, 4) for p in points], 0) if len(points) else np.zeros((0, 4), np.float32)
        return cls(boxes, packed, counts, alpha)

    @classmethod
    def from_reference(cls, db):
        """the reference's list of dicts {gt_box3d (7,), points (n,3), intensity (n,), obj, ...}; alpha from obj.alpha"""
        boxes = np.array([d["gt_box3d"] for d in db], dtype=np.float32).reshape(-1, 7)
        points = [np.concatenate([np.asarray(d["points"], np.float32).reshape(-1, 3),
                                  np.asarray(d["intensity"], np.float32).reshape(-1, 1)], 1) for d in db]
        alpha = np.array([d["obj"].alpha for d in db], dtype=np.float32)
        return cls.from_arrays(boxes, points, alpha)

    def eligible(self, scope):
        """(E,) bool: entries a try may take -- centre inside the range box (checked before the move; scope None: no
        check) and at least 5 points (kitti_rcnn_dataset.py:459-464)"""
        key = None if scope is None else tuple(np.asarray(scope, dtype=np.float64).reshape(-1))
        if key not in self._eligible:
            ok = self.counts >= 5
            if scope is not None:
                sc = np.asarray(scope, dtype=np.float64).reshape(3, 2)      # cfg.PC_AREA_SCOPE is a float64 array
                for k in range(3):
                    ok &= (sc[k, 0] <= self.boxes[:, k].astype(np.float64)) & (self.boxes[:, k].astype(np.float64) <= sc[k, 1])
            self._eligible[key] = ok
        return self._eligible[key]

    def require_lists(self, hard_ratio):
        """the reference's randint(0, len(list)) raises on an empty list: refuse such a database up front"""
        if hard_ratio > 0 and (len(self.easy) == 0 or len(self.hard) == 0):
            raise ValueError("GTDatabase: hard_ratio > 0 needs both easy (> 100 points) and hard (<= 100 points) entries "
                             "(easy %d, hard %d)" % (len(self.easy), len(self.hard)))
        if hard_ratio <= 0 and len(self) == 0:
            raise ValueError("GTDatabase: empty database")


def draw_gt_paste_candidates(db, road_plane, rng=np.random, apply_prob=1.0, extra_num=15, rand_num=True, hard_ratio=0.6,
                             scope=PC_AREA_SCOPE, reduce_by_range=True, max_tries=100):
    """the random half of GT-paste (kitti_rcnn_dataset.py:279, 415-477) with the reference's draws in its order: the apply
    draw, the number of extra objects, then per try the easy / hard draw and the entry draw.  Every draw comes before the
    collision test and the reference counts a candidate before testing it, so the candidates that reach the test follow
    from the random stream alone.  road_plane: (a, b, c, d), normal facing up (get_road_plane).
    -> dict(applied, entries (k,) int64, boxes (k,7) float32 moved onto the road plane, moves (k,) float64)"""
    entries = []
    applied = rng.rand() < apply_prob
    if applied:
        extra = rng.randint(10, extra_num) if rand_num else extra_num
        ok = db.eligible(scope if reduce_by_range else None)
        cnt = 0
        for _ in range(max_tries):
            if cnt > extra:
                break
            if hard_ratio > 0:
                pool = db.easy if rng.rand() > hard_ratio else db.hard
                e = pool[rng.randint(0, len(pool))]
            else:
                e = rng.randint(0, len(db))
            if ok[e]:
                entries.append(e)
                cnt += 1
    entries = np.array(entries, dtype=np.int64)
    boxes = db.boxes[entries].copy()
    # onto the road plane: float64 arithmetic on float32 values, float32 stores (numpy's promotion rules), elementwise
    # the reference's scalar expressions
    a, b, c, d = np.asarray(road_plane, dtype=np.float64).reshape(4)
    cur_height = (-d - a * boxes[:, 0].astype(np.float64) - c * boxes[:, 2].astype(np.float64)) / b
    moves = boxes[:, 1].astype(np.float64) - cur_height
    boxes[:, 1] = boxes[:, 1].astype(np.float64) - moves
    return dict(applied=bool(applied), entries=entries, boxes=boxes, moves=moves)


def collate_batch(batch):
    """kitti_rcnn_dataset.py:1104-1137 (RPN mode): gt_boxes3d zero-padded to the longest list, arrays stacked,
    ints / floats to arrays, everything else listed"""
    out = {}
    bs = len(batch)
    for key in batch[0].keys():
        if key == "gt_boxes3d":
            mg = max(len(batch[k][key]) for k in range(bs))
            g = np.zeros((bs, mg, 7), dtype=np.float32)
            for i in range(bs):
                g[i, :len(batch[i][key]), :] = batch[i][key]
            out[key] = g
        elif isinstance(batch[0][key], np.ndarray):
            out[key] = np.stack([batch[k][key] for k in range(bs)], axis=0)
        else:
            vals = [batch[k][key] for k in range(bs)]
            if isinstance(batch[0][key], int):
                vals = np.array(vals, dtype=np.int32)
            elif isinstance(batch[0][key], float):
                vals = np.array(vals, dtype=np.float32)
            out[key] = vals
    return out


class RPNInputPipeline(object):
    def __init__(self, npoints=16384, mode="TRAIN", use_intensity=True, reduce_by_range=True, pc_area_scope=PC_AREA_SCOPE,
                 aug_data=True, aug_method_list=("rotation", "scaling", "flip"), aug_method_prob=(0.5, 0.5, 0.5), aug_rot_range=18,
                 random_select=True, draw="device", device=None, gt_database=None, gt_aug_apply_prob=1.0, gt_extra_num=15,
                 gt_aug_rand_num=True, gt_aug_hard_ratio=0.6):
        assert mode in ("TRAIN", "EVAL", "TEST") and draw in ("device", "numpy")
        self.npoints, self.mode, self.use_intensity = int(npoints), mode, bool(use_intensity)
        self.reduce_by_range, self.scope = bool(reduce_by_range), pc_area_scope
        self.aug_data = bool(aug_data) and mode == "TRAIN"
        self.aug = (tuple(aug_method_list), tuple(aug_method_prob), aug_rot_range)
        self.random_select, self.draw = bool(random_select), draw
        self.device = _dev(device)
        # GT-paste (GT_AUG_* of tools/cfgs/default.yaml): TRAIN mode with a database only
        self.gt_database = gt_database if mode == "TRAIN" else None
        self.gt_aug = dict(apply_prob=float(gt_aug_apply_prob), extra_num=int(gt_extra_num), rand_num=bool(gt_aug_rand_num),
                           hard_ratio=float(gt_aug_hard_ratio))
        if self.gt_database is not None:
            self.gt_database.require_lists(self.gt_aug["hard_ratio"])
            self.gt_database.upload(self.device)
            self._paste_rng = np.random.RandomState()       # reseeded per (seed, scene) for draw='device'; seeding is cheap, construction is not

    # ---------------------------------------------------------------- device stages
    def _upload(self, scans):
        B = len(scans)
        counts = [int(s["lidar"].shape[0]) for s in scans]
        offsets = np.zeros(B + 1, dtype=np.int32)
        offsets[1:] = np.cumsum(counts)
        total = int(offsets[-1])
        stride = int(scans[0]["lidar"].shape[1])
        dev = self.device
        lidar = torch.empty((max(total, 1), stride), dtype=torch.float32, device=dev)
        for s, o in zip(scans, offsets[:-1]):      # one DMA per scan, straight from the caller's (ideally pinned) memory
            src = s["lidar"]
            n = int(src.shape[0])
            if n:
                src = src if torch.is_tensor(src) else torch.from_numpy(np.ascontiguousarray(src, dtype=np.float32))
                lidar[o:o + n].copy_(src, non_blocking=True)
        calib = np.stack([Calibration(s["calib"]).pack(s["img_shape"], self.scope if self.reduce_by_range else None) for s in scans])
        return (B, total, stride, torch.from_numpy(offsets).to(dev, non_blocking=True), lidar,
                torch.from_numpy(calib).to(dev, non_blocking=True), offsets)

    def _draw_candidates(self, scans, seed, rng):
        """per scene the GT-paste candidates: from rng (draw='numpy', the reference's stream) or from a RandomState of
        (seed, scene) (draw='device': nothing is read back from the device)"""
        out = []
        for b, s in enumerate(scans):
            if s.get("road_plane") is None:
                raise KeyError("GT-paste needs each scan's road_plane (a, b, c, d), as get_road_plane returns it")
            r = rng
            if self.draw == "device":
                r = self._paste_rng
                r.seed([int(seed) & 0xffffffff, b, 0x67a5])
            out.append(draw_gt_paste_candidates(self.gt_database, s["road_plane"], rng=r, scope=self.scope,
                                                reduce_by_range=self.reduce_by_range, **self.gt_aug))
        return out

    def _augment(self, scans, rng, cands):
        """data_augmentation's draws per scene and the label rows they give: the scene's own boxes, then one row per paste
        candidate (rows are augmented independently; the select stage keeps those of the accepted candidates)
        -> aug (B,4) float64 or None, aug_method per scene, GT rows per scene, candidate rows per scene"""
        aug_rows = np.zeros((len(scans), 4), dtype=np.float64) if self.aug_data else None
        methods, gts, cand_rows = [], [], []
        for b, s in enumerate(scans):
            g = np.asarray(s.get("gt_boxes3d", np.zeros((0, 7), np.float32)), dtype=np.float32).reshape(-1, 7)
            ng = len(g)
            alpha = np.asarray(s.get("gt_alpha", np.zeros(ng, np.float32)), dtype=np.float32).reshape(-1)
            if cands is not None:
                g = np.concatenate([g, cands[b]["boxes"]], 0)
                alpha = np.concatenate([alpha, self.gt_database.alpha[cands[b]["entries"]]])
            if self.aug_data:
                angle, scale, flip, method = draw_augmentation(rng=rng, aug_list=self.aug[0], aug_prob=self.aug[1], rot_range=self.aug[2])
                aug_rows[b] = (np.cos(angle) if angle is not None else 1.0, np.sin(angle) if angle is not None else 0.0,
                               float(np.float32(scale)) if scale is not None else 1.0, 1.0 if flip else 0.0)
                g = augment_gt_boxes3d(g, alpha, angle, scale, flip)
                methods.append(method)
            gts.append(g[:ng])
            cand_rows.append(g[ng:])
        return aug_rows, methods, gts, cand_rows

    def _paste(self, scans, B, total, stride, offsets, lidar, rect, flags, cands, K, aug):
        """GT-paste on the device: select (accept / reject every candidate, compact the label rows when `aug` is given)
        and paste (the post-paste ragged cloud).  Two launches and three uploads, no read-back."""
        lib, dev, db = C.lib(), self.device, self.gt_database
        ncand = np.array([len(c["entries"]) for c in cands], dtype=np.int32)
        cand_boxes = np.zeros((B, K, 7), np.float32)
        moves = np.zeros((B, K), np.float64)
        npts = np.zeros((B, K), np.int64)
        src = np.zeros((B, K), np.int64)
        for b, c in enumerate(cands):
            n = len(c["entries"])
            cand_boxes[b, :n], moves[b, :n] = c["boxes"], c["moves"]
            npts[b, :n], src[b, :n] = db.counts[c["entries"]], db.offsets[c["entries"]]
        first = np.zeros(B * K + 1, np.int64)
        first[1:] = np.cumsum(npts.reshape(-1))
        cand_total = int(first[-1])
        colls = [np.asarray(s.get("all_gt_boxes3d", s.get("gt_boxes3d", np.zeros((0, 7), np.float32))), dtype=np.float32).reshape(-1, 7)
                 for s in scans]
        M = max(len(x) for x in colls)
        coll = np.zeros((B, M, 7), np.float32)
        for b, x in enumerate(colls):
            coll[b, :len(x)] = x
        ncoll = np.array([len(x) for x in colls], dtype=np.int32)
        G = 0
        fparts, iparts = [cand_boxes.ravel(), coll.ravel()], [ncand, ncoll, first.astype(np.int32), src.astype(np.int32).ravel()]
        if aug is not None:
            gts, cand_rows = aug[2], aug[3]
            G = max(len(g) for g in gts)
            gt_rows = np.zeros((B, G, 7), np.float32)
            rows = np.zeros((B, K, 7), np.float32)
            for b in range(B):
                gt_rows[b, :len(gts[b])] = gts[b]
                rows[b, :len(cand_rows[b])] = cand_rows[b]
            fparts += [gt_rows.ravel(), rows.ravel()]
            iparts.append(np.array([len(g) for g in gts], dtype=np.int32))
        fbuf = torch.from_numpy(np.concatenate(fparts)).to(dev, non_blocking=True)
        ibuf = torch.from_numpy(np.concatenate(iparts)).to(dev, non_blocking=True)
        moves_t = torch.from_numpy(moves.reshape(-1)).to(dev, non_blocking=True)
        fo = np.cumsum([0] + [len(x) for x in fparts])
        io = np.cumsum([0] + [len(x) for x in iparts])
        fv = [fbuf[fo[j]:fo[j + 1]] for j in range(len(fparts))]
        iv = [ibuf[io[j]:io[j + 1]] for j in range(len(iparts))]
        place = torch.empty((B, K), dtype=torch.int32, device=dev)
        stats = torch.empty((B, 2), dtype=torch.int32, device=dev)
        counts = torch.empty((B, 2), dtype=torch.int32, device=dev)
        gt_out = gt_count = None
        if aug is not None:
            gt_out = torch.empty((B, G + K, 7), dtype=torch.float32, device=dev)
            gt_count = torch.empty(B, dtype=torch.int32, device=dev)
        C.check(lib.prb_gt_paste_select(B, K, M, G, C.ptr(fv[0]), C.ptr(iv[0]), C.ptr(iv[2]), C.ptr(fv[1]) if M else None, C.ptr(iv[1]),
                                        C.ptr(fv[2]) if aug is not None and G else None, C.ptr(iv[4]) if aug is not None else None,
                                        C.ptr(fv[3]) if aug is not None else None, C.ptr(place), C.ptr(stats), C.ptr(gt_out),
                                        C.ptr(gt_count), C.ptr(counts), C.stream()), "gt_paste_select")
        bound = total + cand_total
        offsets2 = torch.empty(B + 1, dtype=torch.int32, device=dev)
        rect2 = torch.empty((max(bound, 1), 3), dtype=torch.float32, device=dev)
        points2 = torch.empty((max(bound, 1), 4), dtype=torch.float32, device=dev)
        flags2 = torch.empty(max(bound, 1), dtype=torch.uint8, device=dev)
        C.check(lib.prb_gt_paste_points(B, total, K, cand_total, C.ptr(offsets), C.ptr(rect), C.ptr(lidar), stride, C.ptr(flags),
                                        C.ptr(fv[0]), C.ptr(iv[2]), C.ptr(iv[3]), C.ptr(moves_t), C.ptr(place), C.ptr(stats),
                                        C.ptr(db.upload(dev).points), C.ptr(offsets2), C.ptr(rect2), C.ptr(points2), C.ptr(flags2), C.ptr(counts),
                                        C.stream()), "gt_paste_points")
        return dict(bound=bound, offsets=offsets2, rect=rect2, points=points2, flags=flags2, counts=counts, place=place, stats=stats,
                    gt=gt_out, gt_count=gt_count, candidates=cands)

    def prepare_batch(self, scans, seed=0, rng=np.random):
        """-> dict of CUDA tensors with collate_batch's keys: pts_input (B,npoints,3|4), pts_rect (B,npoints,3),
        pts_features (B,npoints,1), and unless mode == 'TEST' gt_boxes3d (B,max_g,7) zero padded with gt_count (B,) rows per
        scene, rpn_cls_label (B,npoints) int32, rpn_reg_label (B,npoints,7); plus `choice` (B,npoints) int32 point indices
        and `aug_method` per scene.  With a GT-paste database (TRAIN): gt_boxes3d has max_g + max_candidates rows,
        `choice` indexes the post-paste cloud (the scene's raw points, then the pasted ones) and `valid_counts` counts it;
        when a scene had candidates, `gt_paste` holds the host candidate lists and, on the device, `accepted` (B,K) bool,
        `stats` (B,2) [accepted, pasted points] and the post-paste cloud (offsets, rect, points [x,y,z,intensity], flags)."""
        lib = C.lib()
        dev = self.device
        B, total, stride, offsets, lidar, calib, offsets_h = self._upload(scans)
        npoints = self.npoints
        channels = 4 if (self.use_intensity and stride > 3) else 3
        with torch.cuda.device(dev):
            rect = torch.empty((max(total, 1), 3), dtype=torch.float32, device=dev)
            flags = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
            counts = torch.empty((B, 2), dtype=torch.int32, device=dev)
            C.check(lib.prb_kitti_prepare_points(B, total, C.ptr(offsets), C.ptr(lidar), stride, C.ptr(calib), int(self.reduce_by_range),
                                                 C.ptr(rect), C.ptr(flags), C.ptr(counts), C.stream()), "kitti_prepare_points")
            # GT-paste (kitti_rcnn_dataset.py:273-282): after the validity flags, before the npoints draw
            cands = self._draw_candidates(scans, seed, rng) if self.gt_database is not None else None
            K = max([len(c["entries"]) for c in cands] + [0]) if cands is not None else 0
            aug = paste = None
            if K > 0:
                if self.draw == "device":       # the device draw takes nothing from rng: the label rows can go to select
                    aug = self._augment(scans, rng, cands)
                paste = self._paste(scans, B, total, stride, offsets, lidar, rect, flags, cands, K, aug)
                offsets, rect, lidar, flags, counts = paste["offsets"], paste["rect"], paste["points"], paste["flags"], paste["counts"]
                total, stride = paste["bound"], (4 if stride > 3 else 3)
            choice = torch.empty((B, npoints), dtype=torch.int32, device=dev)
            status = torch.empty(B, dtype=torch.int32, device=dev)
            if self.draw == "device":
                cand = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
                C.check(lib.prb_kitti_draw_points(B, total, C.ptr(offsets), C.ptr(flags), npoints, ctypes.c_uint(int(seed) & 0xffffffff),
                                                  C.ptr(cand), C.ptr(choice), C.ptr(status), C.stream()), "kitti_draw_points")
            else:
                # the reference's np.random stream: flags and depths come back to the host (one sync per batch)
                fl = flags.cpu().numpy()
                depth = rect[:, 2].cpu().numpy()
                offs = offsets_h if paste is None else offsets.cpu().numpy()
                rows = []
                for b in range(B):
                    f = fl[offs[b]:offs[b + 1]]
                    valid = np.nonzero(f & 1)[0]
                    if self.mode == "TRAIN" or self.random_select:
                        ch = draw_choice_numpy(depth[offs[b]:offs[b + 1]][valid], npoints, rng)
                    else:
                        raise RuntimeError("draw='numpy' without random_select returns ragged scenes; use the reference loader")
                    rows.append(valid[ch].astype(np.int32))
                choice.copy_(torch.from_numpy(np.stack(rows)))
                status.zero_()
            # augmentation parameters: the reference draws them per scene after the sample (host, a few numbers)
            if aug is None:
                aug = self._augment(scans, rng, cands if K > 0 else None)
            aug_rows, aug_methods, gts, cand_rows = aug
            aug_t = torch.from_numpy(aug_rows).to(dev, non_blocking=True) if aug_rows is not None else None
            pts_input = torch.empty((B, npoints, channels), dtype=torch.float32, device=dev)
            pts_rect = torch.empty((B, npoints, 3), dtype=torch.float32, device=dev)
            inten = torch.empty((B, npoints), dtype=torch.float32, device=dev)
            C.check(lib.prb_kitti_gather_points(B, npoints, C.ptr(offsets), C.ptr(rect), C.ptr(lidar), stride, C.ptr(choice), C.ptr(aug_t),
                                                C.ptr(status), channels, C.ptr(pts_input), C.ptr(pts_rect), C.ptr(inten), C.stream()), "kitti_gather_points")
            out = dict(pts_input=pts_input, pts_rect=pts_rect, pts_features=inten.unsqueeze(-1), choice=choice, status=status,
                       valid_counts=counts)
            if self.mode != "TEST":
                if paste is not None and paste["gt"] is not None:
                    gt_t, gcnt = paste["gt"], paste["gt_count"]        # compacted by the select stage
                else:
                    if paste is not None:       # draw='numpy': the accept flags are on the host after the sync above
                        acc = paste["place"].cpu().numpy() >= 0
                        gts = [np.concatenate([g, r[acc[b, :len(r)]]], 0) for b, (g, r) in enumerate(zip(gts, cand_rows))]
                    mg = max([len(g) for g in aug[2]] + [0]) + K
                    gpad = np.zeros((B, mg, 7), dtype=np.float32)
                    for b, g in enumerate(gts):
                        gpad[b, :len(g)] = g
                    gt_t = torch.from_numpy(gpad).to(dev, non_blocking=True)
                    gcnt = torch.tensor([len(g) for g in gts], dtype=torch.int32).to(dev, non_blocking=True)
                out["gt_boxes3d"], out["gt_count"] = gt_t, gcnt
                # like get_rpn_sample, every mode but TEST carries the per-point labels (kitti_rcnn_dataset.py:343-352)
                out["rpn_cls_label"], out["rpn_reg_label"] = generate_rpn_training_labels(pts_rect, gt_t, gt_count=gcnt)
            if self.aug_data:
                out["aug_method"] = aug_methods
            if paste is not None:
                out["gt_paste"] = dict(candidates=paste["candidates"], accepted=paste["place"] >= 0, stats=paste["stats"],
                                       offsets=paste["offsets"], rect=paste["rect"], points=paste["points"], flags=paste["flags"])
        return out

"""oracle/make_golden_eval_stats.py -- golden ret_dicts of the reference's three evaluation loops.

Runs the reference's OWN eval_one_epoch_rpn, eval_one_epoch_rcnn and eval_one_epoch_joint (their source taken from
tools/eval_rcnn.py, which parses the command line when imported) on the CPU with batch size 1, on synthetic scenes, and
writes their ret_dicts, logger lines and inputs to tests/golden/eval_stats.npz.  TEST INFRASTRUCTURE ONLY.
    python oracle/make_golden_eval_stats.py

Stand-ins, as oracle/make_golden_proposal.py uses them:
  - `Tensor.cuda()` is the identity and `Tensor.get_device()` names the CPU; iou3d_utils.boxes_iou3d_gpu and nms_gpu are served by the CPU oracle;
  - the model, dataloader and dataset are stubs that hand the loops fixed per-scene network outputs;
  - args: test=False, save_result=False, save_rpn_feature=False, batch_size=1; cfg.TEST.SPLIT='test' skips the AP step;
  - the RCNN loop's input comes from the reference's own get_proposal_from_file (ROI_SAMPLE_JIT: True) on feature and
    proposal files written to a temporary directory; kitti_utils.get_iou3d needs shapely, which is not installed, and
    oracle/gt_paste.py::iou3d (exact float64 clip) replaces it, so `gt_iou` is the exact IoU, not shapely's.
It also records the pooled rows the RCNN network sees, both ways the reference forms them (cfg.RCNN.NUM_POINTS = 32):
  - ROI_SAMPLE_JIT: True -- the eval branch of lib/net/rcnn_net.py:127-152 (its own statements, taken from the source), with
    roipool3d_utils.roipool3d_gpu served by the CPU oracle (oracle.enlarge_box3d + oracle.roipool3d, pinned to the
    reference's kernel by tests/golden/reference_kernels.npz) and the reference's torch canonical transform on the CPU;
  - ROI_SAMPLE_JIT: False -- get_proposal_from_file itself, whose roipool3d_cpu and numpy rotation are the reference's own
    lib/utils/roipool3d/roipool3d_utils.py on its own extension (roipool3d.cpp built unmodified by `make -C oracle ref_twins`).
A proposal file with no line cannot be evaluated by the reference (get_proposal_from_file concatenates an empty list and
raises); the scene "without proposals" here is the RPN's zero-padded proposal block, which every loop runs.
"""
import ast
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
sys.path.insert(0, ROOT)

# (seed, GT count, proposal count, proposals identical to a GT, all proposals zero)
SCENES = [(1, 5, 20, 2, False), (2, 0, 10, 0, False), (3, 40, 100, 3, False), (4, 3, 16, 0, True), (5, 8, 37, 1, False),
          (6, 1, 1, 1, False), (7, 12, 64, 0, False)]
N_PTS, N_FEAT, REG_CHANNEL, NUM_POINTS = 512, 4, 46, 32
STAT_PREFIXES = ("max number", "rpn iou avg", "total ", "final average")


def scene(seed, n_gt, n_roi, n_same, zero):
    """GT boxes in the KITTI camera frame, proposals jittered around them (some identical), point segmentation outputs"""
    rng = np.random.default_rng(seed)
    gt = np.stack([rng.uniform(-20, 20, n_gt), rng.uniform(0.5, 2.0, n_gt), rng.uniform(5, 60, n_gt), rng.uniform(1.3, 1.8, n_gt),
                   rng.uniform(1.4, 1.9, n_gt), rng.uniform(3.2, 4.8, n_gt), rng.uniform(-np.pi, np.pi, n_gt)], 1).astype(np.float32)
    src = gt[rng.integers(0, n_gt, n_roi)] if n_gt else np.tile(np.array([[0, 1, 20, 1.5, 1.6, 4, 0]], np.float32), (n_roi, 1))
    noise = rng.normal(0, 1, (n_roi, 7)) * np.array([0.4, 0.1, 0.4, 0.1, 0.1, 0.3, 0.2])
    rois = (src + noise).astype(np.float32)
    rois[:n_same] = gt[:n_same] if n_gt else rois[:n_same]
    if zero:
        rois[:] = 0
    label = rng.choice([-1, 0, 1], N_PTS, p=[0.1, 0.6, 0.3]).astype(np.int64)
    raw = (rng.normal(0, 2, N_PTS) + 1.5 * (label > 0)).astype(np.float32)
    reg = rng.normal(0, 0.5, (n_roi, REG_CHANNEL)).astype(np.float32)
    reg[:, [2, 3, 8, 9]] += 2.0                     # favour the centre x / z bins
    cls = rng.normal(0, 2, (n_roi, 1)).astype(np.float32)
    return dict(gt=gt, rois=rois, label=label, rpn_raw=raw, rcnn_reg=reg, rcnn_cls=cls, roi_scores=rng.normal(0, 1, n_roi).astype(np.float32),
                xyz=points(rng, rois), feat=rng.normal(0, 1, (N_PTS, N_FEAT)).astype(np.float32))


def points(rng, rois):
    """N_PTS points: 70 % around the proposals (so that pooled boxes hold from none to more than NUM_POINTS points), the rest
    uniform in the scope"""
    near = int(0.7 * N_PTS) if rois.any() else 0
    c = rois[rng.integers(0, len(rois), near), :3] if near else np.zeros((0, 3), np.float32)
    p = np.concatenate([c + rng.normal(0, 1.5, (near, 3)), rng.uniform(-30, 30, (N_PTS - near, 3)) + np.array([0, 0, 35])])
    return p.astype(np.float32)


def label_line(cls, box, score=None):
    x, y, z, h, w, l, ry = box
    vals = [cls, "0.00", "0", "-10", "0.0", "0.0", "100.0", "100.0"] + [repr(float(v)) for v in (h, w, l, x, y, z, ry)]
    return " ".join(vals + ([repr(float(score))] if score is not None else []))


def loops():
    src = open(os.path.join(REF, "tools", "eval_rcnn.py")).read()
    names = ("eval_one_epoch_rpn", "eval_one_epoch_rcnn", "eval_one_epoch_joint")
    nodes = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in names]
    return nodes


def jit_pool_fn(ns):
    """the eval branch of RCNNNet.forward under ROI_SAMPLE_JIT (rcnn_net.py:127-152), its own statements, as a function of
    input_data returning pts_input"""
    src = open(os.path.join(REF, "lib", "net", "rcnn_net.py")).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "RCNNNet")
    fwd = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "forward")
    jit = next(n for n in fwd.body if isinstance(n, ast.If))                 # if cfg.RCNN.ROI_SAMPLE_JIT:
    branch = jit.body[0].orelse                                               # if self.training: ... else: <eval>
    fn = ast.parse("def jit_pool(input_data):\n    return pts_input\n").body[0]
    fn.body = branch + fn.body
    exec(compile(ast.fix_missing_locations(ast.Module(body=[fn], type_ignores=[])), "rcnn_net.py", "exec"), ns)
    return ns["jit_pool"]


def reference_roipool3d_utils():
    """lib/utils/roipool3d/roipool3d_utils.py, unchanged, on the reference's own roipool3d extension (oracle/_ref)"""
    import importlib.util
    so = os.path.join(ROOT, "oracle", "_ref", "ref_roipool3d_cuda.so")
    if not os.path.exists(so):
        raise SystemExit("build the reference's roipool3d extension first: make -C oracle ref_twins")
    spec = importlib.util.spec_from_file_location("ref_roipool3d_cuda", so)
    ext = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ext)
    saved = sys.modules.get("roipool3d_cuda")
    sys.modules["roipool3d_cuda"] = ext
    try:
        spec = importlib.util.spec_from_file_location("ref_roipool3d_utils", os.path.join(REF, "lib", "utils", "roipool3d", "roipool3d_utils.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if saved is not None:
            sys.modules["roipool3d_cuda"] = saved
    return mod


class _Bar:
    def __init__(self, *a, **k):
        pass

    set_postfix = update = close = lambda self, *a, **k: None


class _Log:
    def __init__(self):
        self.lines = []

    def info(self, s):
        self.lines.append(s)


def main():
    from oracle import gt_paste as GP
    from oracle import oracle as O
    from pointrcnn_b200 import dropin
    sys.path.insert(0, REF)
    dropin.activate(compat=True)
    stub = types.ModuleType("lib.utils.iou3d.iou3d_utils")
    stub.boxes_iou3d_gpu = lambda a, b: torch.from_numpy(O.boxes_iou3d(a.float().numpy(), b.float().numpy()))

    def nms_gpu(boxes, scores, thresh):
        order = scores.sort(0, descending=True)[1]
        keep = O.nms(boxes[order].contiguous().numpy(), float(thresh), normal=False)
        return order[torch.from_numpy(keep)].contiguous()
    stub.nms_gpu = nms_gpu
    pkg = types.ModuleType("lib.utils.iou3d")
    pkg.__path__ = []
    sys.modules["lib.utils.iou3d"], sys.modules["lib.utils.iou3d.iou3d_utils"] = pkg, stub
    pkg.iou3d_utils = stub
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.Tensor.get_device = lambda self: "cpu"
    from lib.config import cfg, cfg_from_file
    cfg_from_file(os.path.join(REF, "tools/cfgs/default.yaml"))
    cfg.TEST.SPLIT = "test"
    cfg.INCLUDE_SIMILAR_TYPE, cfg.PC_REDUCE_BY_RANGE = False, False
    cfg.RCNN.ROI_SAMPLE_JIT = True
    cfg.RCNN.USE_SEG_SCORE = False
    cfg.RCNN.NUM_POINTS = NUM_POINTS
    import lib.datasets.kitti_rcnn_dataset as K
    import lib.utils.kitti_utils as kitti_utils
    from lib.utils import object3d
    from lib.utils.bbox_transform import decode_bbox_target
    kitti_utils.get_iou3d = lambda a, b, need_bev=False: GP.iou3d(a, b)

    data = [scene(*s) for s in SCENES]
    out = {}
    for i, d in enumerate(data):
        for k, v in d.items():
            out["s%d_%s" % (i, k)] = v

    rec = {"pred": [], "det": []}

    def decode(*a, **kw):
        r = decode_bbox_target(*a, **kw)
        rec["pred"].append(r.numpy().copy())
        return r

    def save_kitti_format(sample_id, calib, boxes, out_dir, scores, image_shape):
        rec["det"].append(len(boxes))

    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "ImageSets"))
        ids = list(range(len(data)))
        with open(os.path.join(tmp, "ImageSets", "val.txt"), "w") as f:
            f.write("\n".join("%06d" % k for k in ids) + "\n")
        feat_dir, roi_dir = os.path.join(tmp, "features"), os.path.join(tmp, "rois")
        os.makedirs(feat_dir)
        os.makedirs(roi_dir)
        for k, d in enumerate(data):
            seg = (torch.sigmoid(torch.from_numpy(d["rpn_raw"])) > cfg.RPN.SCORE_THRESH).float().numpy()
            for suffix, v in (("", d["feat"]), ("_xyz", d["xyz"]), ("_intensity", np.zeros(N_PTS, np.float32)), ("_seg", seg)):
                np.save(os.path.join(feat_dir, "%06d%s.npy" % (k, suffix)), v)
            with open(os.path.join(roi_dir, "%06d.txt" % k), "w") as f:
                f.write("".join(label_line("Car", b, sc) + "\n" for b, sc in zip(d["rois"], d["roi_scores"])))

        ds = object.__new__(K.KittiRCNNDataset)
        ds.mode, ds.classes, ds.split = "EVAL", ("Background", "Car"), "val"
        ds.imageset_dir = os.path.join(tmp, "a", "b")
        ds.image_idx_list = ["%06d" % k for k in ids]
        ds.rcnn_eval_roi_dir, ds.rcnn_eval_feature_dir = roi_dir, feat_dir
        ds.get_label = lambda sid: [object3d.Object3d(label_line("Car", b)) for b in data[sid]["gt"]]
        args = types.SimpleNamespace(test=False, save_result=False, save_rpn_feature=False, batch_size=1)
        ns = dict(os=os, np=np, torch=torch, F=torch.nn.functional, tqdm=types.SimpleNamespace(tqdm=_Bar), cfg=cfg, args=args,
                  iou3d_utils=stub, kitti_utils=kitti_utils, decode_bbox_target=decode, save_kitti_format=save_kitti_format,
                  datetime=__import__("datetime").datetime, kitti_evaluate=None)
        exec(compile(ast.Module(body=loops(), type_ignores=[]), "eval_rcnn.py", "exec"), ns)

        class Loader(list):
            pass

        class Dataset(types.SimpleNamespace):
            def __len__(self):
                return len(data)

        class Model:
            def __init__(self, outputs, proposal_layer=None):
                self.outputs = iter(outputs)
                self.rpn = types.SimpleNamespace(proposal_layer=proposal_layer)

            def eval(self):
                pass

            def __call__(self, input_data):
                return next(self.outputs)

        def run(name, batches, outputs, proposal_layer=None):
            loader = Loader(batches)
            loader.dataset = Dataset(imageset_dir=ds.imageset_dir, split="val", get_calib=lambda sid: None,
                                     get_image_shape=lambda sid: None)
            log = _Log()
            rec["pred"].clear()
            rec["det"].clear()
            with torch.no_grad():
                ret = ns[name](Model(outputs, proposal_layer), loader, 0, os.path.join(tmp, name), log)
            return ret, [s for s in log.lines if s.startswith(STAT_PREFIXES)]

        def detections(ids):
            """the per-scene counts of final detections: save_kitti_format runs for the scenes with a score over the threshold"""
            det = np.zeros(len(data), np.int64)
            hit = [k for k in ids if (torch.sigmoid(torch.from_numpy(data[k]["rcnn_cls"])) > cfg.RCNN.SCORE_THRESH).any()]
            det[hit] = rec["det"]
            return det

        def pack(name, ret, lines):
            ret = {k: v for k, v in ret.items() if k != "empty_cnt"}
            out[name + "_keys"] = np.array(list(ret.keys()))
            out[name + "_values"] = np.array([float(v) for v in ret.values()], np.float64)
            out[name + "_log"] = np.array(lines)

        # eval_one_epoch_rpn
        t = torch.from_numpy
        batches = [dict(sample_id=[k], pts_rect=d["xyz"][None], pts_features=np.zeros((1, N_PTS, 1), np.float32), pts_input=d["xyz"][None],
                        rpn_cls_label=d["label"][None], rpn_reg_label=None, gt_boxes3d=d["gt"][None]) for k, d in enumerate(data)]
        outputs = [dict(rpn_cls=t(d["rpn_raw"]).view(1, -1, 1), rpn_reg=None, backbone_xyz=t(d["xyz"])[None], backbone_features=None)
                   for d in data]
        props = iter([(t(d["rois"])[None], t(d["roi_scores"])[None]) for d in data])
        pack("rpn", *run("eval_one_epoch_rpn", batches, outputs, proposal_layer=lambda *a: next(props)))

        # eval_one_epoch_joint
        seg = [(torch.sigmoid(t(d["rpn_raw"])) > cfg.RPN.SCORE_THRESH).float()[None] for d in data]
        outputs = [dict(roi_scores_raw=t(d["roi_scores"])[None], rois=t(d["rois"])[None], seg_result=seg[k], rcnn_cls=t(d["rcnn_cls"]),
                        rcnn_reg=t(d["rcnn_reg"])) for k, d in enumerate(data)]
        pack("joint", *run("eval_one_epoch_joint", batches, outputs))
        for k in range(len(data)):
            out["s%d_joint_pred" % k] = rec["pred"][k].reshape(-1, 7)
        out["joint_det"] = detections(range(len(data)))

        # eval_one_epoch_rcnn on get_proposal_from_file's output for the files written above
        batches = []
        for k in range(len(data)):
            b = ds.get_proposal_from_file(k)
            out["s%d_gt_iou" % k] = np.asarray(b["gt_iou"], np.float32)
            b["sample_id"] = k
            batches.append(b)
        outputs = [dict(rcnn_cls=t(d["rcnn_cls"]), rcnn_reg=t(d["rcnn_reg"])) for d in data]
        pack("rcnn", *run("eval_one_epoch_rcnn", batches, outputs))
        for k in range(len(data)):
            out["s%d_rcnn_pred" % k] = rec["pred"][k]
        out["rcnn_det"] = detections(range(len(data)))

        # the pooled rows: ROI_SAMPLE_JIT True (rcnn_net's eval branch on get_proposal_from_file's JIT sample) ...
        rp_stub = types.SimpleNamespace()

        def roipool3d_gpu(pts, pts_feature, boxes3d, pool_extra_width, sampled_pt_num=512):
            big = O.enlarge_box3d(boxes3d.numpy().reshape(-1, 7), pool_extra_width).reshape(boxes3d.shape)
            pooled, empty = O.roipool3d(pts.numpy(), pts_feature.numpy(), big, sampled_pt_num)
            return torch.from_numpy(pooled), torch.from_numpy(empty)
        rp_stub.roipool3d_gpu = roipool3d_gpu
        jit_pool = jit_pool_fn(dict(torch=torch, cfg=cfg, kitti_utils=kitti_utils, roipool3d_utils=rp_stub))
        for k, b in enumerate(batches):
            inp = {key: t(np.asarray(v)).float().unsqueeze(0) for key, v in b.items() if key not in ("sample_id", "gt_iou", "gt_boxes3d")}
            out["s%d_rows_jit" % k] = jit_pool(inp).numpy()
        # ... and ROI_SAMPLE_JIT False (get_proposal_from_file's roipool3d_cpu and numpy canonical transform)
        cfg.RCNN.ROI_SAMPLE_JIT = False
        K.roipool3d_utils = reference_roipool3d_utils()
        for k in range(len(data)):
            b = ds.get_proposal_from_file(k)
            out["s%d_rows_cpu" % k] = np.concatenate([b["pts_input"], b["pts_features"]], axis=2).astype(np.float32)
            np.testing.assert_array_equal(b["gt_iou"], out["s%d_gt_iou" % k])
        cfg.RCNN.ROI_SAMPLE_JIT = True
    path = os.path.join(ROOT, "tests", "golden", "eval_stats.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")
    for name in ("rpn", "rcnn", "joint"):
        print(name, dict(zip(out[name + "_keys"].tolist(), out[name + "_values"].tolist())))


if __name__ == "__main__":
    main()

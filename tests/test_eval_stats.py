"""Evaluation statistics: the oracle against what the reference's own eval_one_epoch_rpn / _rcnn / _joint returned
(oracle/make_golden_eval_stats.py), the logger lines, the proposal reader; on the GPU the eval_stats.cu kernels against
prb_boxes_iou3d and the reference's torch lines, EvalStats against the golden, the offline evaluation batch against
RCNNStage.pool, padded-batch detections, and the absence of host synchronisation."""
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import eval_stats as OE
from oracle import make_golden_eval_stats as MG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "eval_stats.npz")
NS = len(MG.SCENES)


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD, allow_pickle=False)


def _seg(raw):
    return (torch.sigmoid(torch.from_numpy(raw)) > 0.3).long().numpy()


def _pred_cls(cls):
    return (torch.sigmoid(torch.from_numpy(cls).view(-1)) > 0.3).long().numpy()


def _scenes(gold):
    out = []
    for k in range(NS):
        g = lambda key: gold["s%d_%s" % (k, key)]
        out.append(dict(rois=g("rois"), gt=g("gt"), seg=_seg(g("rpn_raw")), label=g("label"), rcnn_pred=g("rcnn_pred"),
                        joint_pred=g("joint_pred"), pred_cls=_pred_cls(g("rcnn_cls")), gt_iou=g("gt_iou"),
                        rcnn_det=int(gold["rcnn_det"][k]), joint_det=int(gold["joint_det"][k]), xyz=g("xyz"), feat=g("feat"),
                        roi_scores=g("roi_scores")))
    return out


def _golden_ret(gold, name):
    return dict(zip(gold[name + "_keys"].tolist(), gold[name + "_values"].tolist()))


def _oracle(gold, name):
    sc = _scenes(gold)
    if name == "rpn":
        return OE.rpn_loop(sc)
    key = "rcnn" if name == "rcnn" else "joint"
    return OE.rcnn_loop([dict(s, pred=s[key + "_pred"], n_det=s[key + "_det"]) for s in sc], joint=name == "joint")


def _assert_ret(got, want, counts_exact=True, tol=None):
    assert list(got.keys()) == list(want.keys())
    for k, v in want.items():
        if "recall" in k or k in ("max_obj_num", "rcnn_avg_num"):
            assert got[k] == v, k                                     # ratios of integer counts: exact
        else:
            assert abs(got[k] - v) <= (tol or {}).get(k, 1e-12), (k, got[k], v)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", ["rpn", "rcnn", "joint"])
def test_oracle_reproduces_the_reference_loops(gold, name):
    ret, counts = _oracle(gold, name)
    _assert_ret(ret, _golden_ret(gold, name))
    # the fixture covers: a scene without GT, all-zero proposals, more than 32 GT, proposals identical to a GT (IoU 1)
    sc = _scenes(gold)
    assert any(len(s["gt"]) == 0 for s in sc) and any(not s["rois"].any() for s in sc) and any(len(s["gt"]) > 32 for s in sc)
    assert counts["rpn_recalled"][4] > 0 and counts["gt_total"] == sum(len(s["gt"]) for s in sc)


def test_oracle_gt_iou_against_the_reference(gold):
    # get_proposal_from_file's gt_iou comes from an exact float64 clip; the fp32 overlap is within 1e-5 of it
    for s in _scenes(gold):
        np.testing.assert_allclose(OE.gt_iou(s["rois"], s["gt"]), s["gt_iou"], rtol=0, atol=1e-5)


@pytest.mark.parametrize("name", ["rpn", "rcnn", "joint"])
def test_log_lines_byte_for_byte(gold, name):
    from pointrcnn_b200.datasets.eval_stats import log_lines
    _, counts = _oracle(gold, name)
    lines = log_lines(name, _golden_ret(gold, name), counts)
    assert lines == gold[name + "_log"].tolist()


def test_read_rois_reads_the_score_column(gold):
    from pointrcnn_b200.datasets.rcnn_offline import read_rois
    s = _scenes(gold)[0]
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "000004.txt"), "w") as f:
            f.write("".join(MG.label_line("Car", b, sc) + "\n" for b, sc in zip(s["rois"], s["roi_scores"])))
        boxes, scores = read_rois(d, 4, with_scores=True)
        np.testing.assert_array_equal(boxes, s["rois"])
        np.testing.assert_array_equal(scores, s["roi_scores"])
        np.testing.assert_array_equal(read_rois(d, 4), s["rois"])


# ------------------------------------------------------------------------------------------------ GPU
def _boxes(rng, n):
    return np.stack([rng.uniform(-6, 6, n), rng.uniform(0.5, 2.0, n), rng.uniform(5, 17, n), rng.uniform(1.3, 1.8, n),
                     rng.uniform(1.4, 1.9, n), rng.uniform(3.2, 4.8, n), rng.uniform(-np.pi, np.pi, n)], -1).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 37, 100, 512])
@pytest.mark.parametrize("g", [0, 1, 33])
@pytest.mark.parametrize("with_count", [False, True])
def test_box_recall_matches_the_iou_matrix(cuda, m, g, with_count):
    from pointrcnn_b200 import _cabi as C
    from pointrcnn_b200.datasets.eval_stats import EvalStats
    B = 64
    rng = np.random.default_rng(m * 100 + g)
    gt = torch.from_numpy(_boxes(rng, (B, g))).to(cuda).view(B, g, 7)
    boxes = torch.from_numpy(_boxes(rng, (B, m))).to(cuda)
    if g:
        boxes[:, : min(m, g)] = gt[:, : min(m, g)]                   # IoU 1 pairs
    gt_count = torch.from_numpy(rng.integers(0, g + 1, B).astype(np.int32)).to(cuda)
    box_count = torch.from_numpy(rng.integers(0, m + 1, B).astype(np.int32)).to(cuda) if with_count else None
    n = box_count.long() if with_count else torch.full((B,), m, device=cuda)
    st = EvalStats(device=cuda)
    T = len(st.thresh_list)
    recalled = torch.zeros(T, dtype=torch.int64, device=cuda)
    total = torch.zeros(1, dtype=torch.int64, device=cuda)
    best = torch.full((B, m), -7.0, device=cuda)
    st._recall(boxes, box_count, gt, gt_count, recalled, total, best)
    # reference: the IoU matrix, a masked torch max, then > thresh
    iou = torch.empty((B, m, g), device=cuda)
    if g:
        C.check(C.lib().prb_boxes_iou3d(B, m, C.ptr(boxes), g, C.ptr(gt), C.ptr(iou), C.stream()), "boxes_iou3d")
    row_ok = torch.arange(m, device=cuda)[None, :] < n[:, None]
    col_ok = torch.arange(g, device=cuda)[None, :] < gt_count.long()[:, None]
    masked = iou.masked_fill(~(row_ok[:, :, None] & col_ok[:, None, :]), float("-inf"))
    want_best = torch.zeros((B, m), device=cuda)
    if g:
        rb = masked.max(dim=2)[0]
        want_best = torch.where(row_ok & (gt_count.long() > 0)[:, None], rb, want_best)
        gmax = masked.max(dim=1)[0]
        want_rec = [int(((gmax > t) & col_ok).sum()) for t in st.thresh_list]
    else:
        want_rec = [0] * T
    assert torch.equal(best, want_best)
    assert recalled.tolist() == want_rec
    assert int(total) == int(gt_count.sum())
    if g and m >= g:
        assert want_rec[-1] > 0


@pytest.mark.gpu
def test_seg_iou_and_cls_acc_bit_identical_to_the_reference_lines(cuda):
    from pointrcnn_b200.datasets.eval_stats import EvalStats
    rng = np.random.default_rng(3)
    B, N, M = 24, 4000, 100
    seg = torch.from_numpy(rng.integers(0, 2, (B, N))).to(cuda)
    label = torch.from_numpy(rng.choice([-1, 0, 1], (B, N), p=[0.1, 0.5, 0.4])).to(cuda)
    label[0] = 0                                                     # no foreground: union clamps to 1
    seg[1] = 0
    st = EvalStats(device=cuda)
    st._seg_iou(seg, label)
    for b in range(B):
        fg_mask = label[b] > 0
        correct = ((seg[b] == label[b]) & fg_mask).sum().float()
        union = fg_mask.sum().float() + (seg[b] > 0).sum().float() - correct
        want = correct / torch.clamp(union, min=1.0)
        assert torch.equal(st._seg.data[b], want), b
    # classification accuracy over the real RoIs, with IoUs exactly at the thresholds
    gt_iou = torch.from_numpy(rng.choice([0.0, 0.3, 0.45, 0.5, 0.6, 0.65, 0.7, 0.9], (B, M)).astype(np.float32)).to(cuda)
    gt_iou += torch.from_numpy(rng.choice([0.0, 0.0, 1e-3], (B, M)).astype(np.float32)).to(cuda)
    pred = torch.from_numpy(rng.integers(0, 2, (B, M))).to(cuda)
    count = torch.from_numpy(rng.integers(0, M + 1, B).astype(np.int32)).to(cuda)
    count[0], count[1] = 0, M
    acc, acc_r = st._acc.take(B), st._acc_refined.take(B)
    from pointrcnn_b200 import _cabi as C
    C.check(C.lib().prb_eval_cls_acc(B, M, C.ptr(count), C.ptr(pred.int()), C.ptr(gt_iou), 0.6, 0.45, 0.7, C.ptr(acc), C.ptr(acc_r),
                                     C.stream()), "eval_cls_acc")
    for b in range(B):
        n = int(count[b])
        gi, pc = gt_iou[b, :n], pred[b, :n]
        cls_label = (gi > 0.6).float()
        cls_valid_mask = ((gi >= 0.6) | (gi <= 0.45)).float()
        cls_acc = ((pc == cls_label.long()).float() * cls_valid_mask).sum() / max(cls_valid_mask.sum(), 1.0)
        cls_label_refined = (gi >= 0.7).float()
        cls_acc_refined = (pc == cls_label_refined.long()).float().sum() / max(cls_label_refined.shape[0], 1.0)
        assert torch.equal(acc[b], cls_acc), b
        assert torch.equal(acc_r[b], cls_acc_refined), b


def _pad(arrs, n, value=0.0):
    out = np.full((len(arrs), n) + arrs[0].shape[1:], value, arrs[0].dtype)
    for k, a in enumerate(arrs):
        out[k, :len(a)] = a
    return out


def _batches(name, sc, cuda, batch):
    """the golden scenes as padded device batches of `batch` scenes: a list of (EvalStats method name, args, kwargs)"""
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    out = []
    for i in range(0, len(sc), batch):
        part = sc[i:i + batch]
        M = max(len(s["rois"]) for s in part)
        G = max(max(len(s["gt"]) for s in part), 1)
        gt = t(_pad([s["gt"].reshape(-1, 7) for s in part], G))
        gt_count = t(np.array([len(s["gt"]) for s in part], np.int32))
        rois = t(_pad([s["rois"] for s in part], M))
        seg, label = t(np.stack([s["seg"] for s in part])), t(np.stack([s["label"] for s in part]))
        if name == "rpn":
            out.append(("add_rpn", (rois, gt, gt_count), dict(seg_result=seg, rpn_cls_label=label)))
            continue
        count = t(np.array([len(s["rois"]) for s in part], np.int32))
        pred = t(_pad([s[name + "_pred"] for s in part], M))
        ndet = np.array([s[name + "_det"] for s in part])
        kw = dict(box_count=count, select=t(np.arange(M)[None, :] < ndet[:, None]))
        if name == "rcnn":
            kw.update(pred_classes=t(_pad([s["pred_cls"] for s in part], M)), gt_iou=t(_pad([s["gt_iou"] for s in part], M)))
        else:
            kw.update(seg_result=seg, rpn_cls_label=label)
        out.append(("add_rcnn", (pred, rois, gt, gt_count), kw))
    return out


def _feed(st, batches):
    for method, args, kw in batches:
        getattr(st, method)(*args, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rpn", "rcnn", "joint"])
@pytest.mark.parametrize("batch", [1, 8])
def test_eval_stats_equals_the_golden(cuda, gold, name, batch):
    from pointrcnn_b200.datasets.eval_stats import EvalStats
    st = EvalStats(device=cuda)
    _feed(st, _batches(name, _scenes(gold), cuda, batch))
    # cls acc refined divides by a Python number: torch on the GPU multiplies by the fp32 reciprocal, the golden (a CPU
    # run) divides; the two differ by at most one fp32 ulp per scene
    _assert_ret(st.result(), _golden_ret(gold, name), tol={"rcnn_cls_acc_refined": 6e-8})
    assert st.log_lines() == gold[name + "_log"].tolist()


def _sampler(cuda, **kw):
    from pointrcnn_b200.datasets.rcnn_offline import DEFAULT_CFG, RCNNOfflineSampler, _ns
    d = {k: v for k, v in DEFAULT_CFG.items() if k != "RCNN"}
    d["RCNN"] = dict(DEFAULT_CFG["RCNN"], **kw)
    return RCNNOfflineSampler(cfg=_ns(d), device=cuda)


def _device_scenes(gold, cuda, n_feat=None):
    rng = np.random.default_rng(5)
    out = []
    for s in _scenes(gold):
        feat = s["feat"] if n_feat is None else rng.standard_normal((len(s["xyz"]), n_feat)).astype(np.float32)
        d = dict(rpn_xyz=s["xyz"], rpn_features=feat, rpn_intensity=np.zeros(len(s["xyz"]), np.float32), seg_mask=s["seg"].astype(np.float32),
                 roi_boxes3d=s["rois"], roi_scores=s["roi_scores"], gt_boxes3d=s["gt"].reshape(-1, 7))
        out.append({k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda) for k, v in d.items()})
    return out


@pytest.mark.gpu
def test_prepare_eval_batch_pools_like_rcnn_stage(cuda, gold):
    from pointrcnn_b200.datasets.rcnn_offline import FAR, _pad as pad
    from pointrcnn_b200.rcnn.stage import RCNNStage
    scenes = _device_scenes(gold, cuda)
    batch = _sampler(cuda).prepare_eval_batch(scenes)
    B, M = len(scenes), max(len(s["roi_boxes3d"]) for s in scenes)
    N = max(len(s["rpn_xyz"]) for s in scenes)
    xyz = pad([s["rpn_xyz"] for s in scenes], N, FAR)
    feats = pad([s["rpn_features"] for s in scenes], N, 0.0)
    seg = pad([s["seg_mask"].view(-1, 1) for s in scenes], N, 0.0)[..., 0]
    rois = pad([s["roi_boxes3d"] for s in scenes], M, 0.0)
    stage = RCNNStage(input_channels=feats.shape[2]).to(cuda)
    rows, empty = stage.pool(xyz, feats, seg, torch.norm(xyz, p=2, dim=2), rois)
    assert torch.equal(batch["rows"], rows)
    assert torch.equal(batch["pooled_empty_flag"], empty)
    assert torch.equal(batch["roi_boxes3d"], rois)
    assert batch["roi_count"].tolist() == [len(s["roi_boxes3d"]) for s in scenes]
    assert batch["gt_count"].tolist() == [len(s["gt_boxes3d"]) for s in scenes]
    for k, s in enumerate(_scenes(gold)):
        n = len(s["rois"])
        np.testing.assert_array_equal(batch["roi_scores"][k, :n].cpu().numpy(), s["roi_scores"])
        # fp32 iou3d against the reference's exact clip
        np.testing.assert_allclose(batch["gt_iou"][k, :n].cpu().numpy(), s["gt_iou"], rtol=0, atol=1e-5)
        assert not batch["gt_iou"][k, n:].any()
    # numpy input gives the same batch.  Its depth column is computed on the host (norm / 70.0, a true division), the device
    # path's by torch on the GPU, which multiplies by the fp32 reciprocal: one ulp apart at most; every other column is exact
    host = _sampler(cuda).prepare_eval_batch([{k: v.cpu().numpy() for k, v in s.items()} for s in scenes])
    for k in ("roi_boxes3d", "roi_scores", "roi_count", "gt_boxes3d", "gt_count", "gt_iou", "pooled_empty_flag"):
        assert torch.equal(host[k], batch[k]), k
    assert torch.equal(host["rows"][..., [0, 1, 2, 3]], batch["rows"][..., [0, 1, 2, 3]])
    assert torch.equal(host["rows"][..., 5:], batch["rows"][..., 5:])
    torch.testing.assert_close(host["rows"][..., 4], batch["rows"][..., 4], rtol=0, atol=2.5e-7)


# the xyz columns after the canonical transform: the device rotates in fp32 (cosf / sinf, fused into the pooling kernel);
# the reference's ROI_SAMPLE_JIT branch rotates with torch's fp32 cos / sin and a matmul, its roipool3d_cpu branch with
# numpy (float64 cos / sin of ry mod 2 pi, rounded to float32).  Coordinates within a few metres of the RoI centre agree to
# a few fp32 ulp
XYZ_TOL = 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["device", "host"])
@pytest.mark.parametrize("jit", [True, False])
def test_prepare_eval_batch_matches_the_reference_rows(cuda, gold, source, jit):
    """the golden rows of both ways the reference pools for evaluation: rcnn_net's ROI_SAMPLE_JIT branch (roipool3d kernel
    + torch canonical transform) and get_proposal_from_file's roipool3d_cpu + numpy canonical transform"""
    scenes = _device_scenes(gold, cuda)
    if source == "host":
        scenes = [{k: v.cpu().numpy() for k, v in s.items()} for s in scenes]
    batch = _sampler(cuda, NUM_POINTS=MG.NUM_POINTS).prepare_eval_batch(scenes)
    B, M = batch["roi_boxes3d"].shape[:2]
    rows = batch["rows"].view(B, M, MG.NUM_POINTS, -1).cpu().numpy()
    pooled = 0
    for k, s in enumerate(_scenes(gold)):
        n = len(s["rois"])
        got, want = rows[k, :n], gold["s%d_%s" % (k, "rows_jit" if jit else "rows_cpu")]
        assert got.shape == want.shape
        # the same points pooled in the same order: RPN feature and segmentation columns exact
        np.testing.assert_array_equal(got[..., 5:], want[..., 5:])
        np.testing.assert_array_equal(got[..., 3], want[..., 3])
        # depth / 70 - 0.5: the device divides as torch on the GPU does, the golden's CPU run with a true division
        np.testing.assert_allclose(got[..., 4], want[..., 4], rtol=0, atol=2.5e-7)
        np.testing.assert_allclose(got[..., 0:3], want[..., 0:3], rtol=0, atol=XYZ_TOL)
        pooled += int((want[..., 5:] != 0).any(axis=(1, 2)).sum())
    assert pooled > 200                      # most golden RoIs hold points: the comparison is not of empty rows


@pytest.mark.gpu
def test_forward_offline_selects_as_each_scene_alone(cuda, gold):
    from pointrcnn_b200.point_rcnn import PointRCNNInference
    torch.manual_seed(0)
    model = PointRCNNInference().to(cuda).eval()
    smp = _sampler(cuda)
    scenes = _device_scenes(gold, cuda, n_feat=128)
    with torch.no_grad():
        boxes, raw, select = model.detections_device(model.forward_offline(smp.prepare_eval_batch(scenes)))
        assert select.any()
        for k, s in enumerate(scenes):
            b1, r1, s1 = model.detections_device(model.forward_offline(smp.prepare_eval_batch([s])))
            n = int(s1.sum())
            assert int(select[k].sum()) == n, k
            # the network's TF32 layers round differently with the number of RoIs in the launch (about 1e-3 relative), which
            # can swap the order of two detections with nearly equal scores: the same detections, matched one to one
            a = torch.cat([boxes[k][select[k]], raw[k][select[k]].unsqueeze(1)], 1)
            b = torch.cat([b1[0][s1[0]], r1[0][s1[0]].unsqueeze(1)], 1)
            close = ((a[:, None, :] - b[None, :, :]).abs() <= 2e-3 * (1 + b[None, :, :].abs())).all(dim=2)
            assert close.any(dim=1).all() and close.any(dim=0).all(), k
            # padding RoIs can never be selected
            assert not select[k, len(s["roi_boxes3d"]):].any()


@pytest.mark.gpu
def test_optional_statistics_are_given_for_every_batch_or_none(cuda, gold):
    from pointrcnn_b200.datasets.eval_stats import EvalStats
    (m, args, kw), = _batches("rcnn", _scenes(gold), cuda, 8)
    st = EvalStats(device=cuda)
    st.add_rcnn(*args, **kw)
    with pytest.raises(ValueError, match="pred_classes"):
        st.add_rcnn(*args, **dict(kw, pred_classes=None))
    (m, args, kw), = _batches("rpn", _scenes(gold), cuda, 8)
    st = EvalStats(device=cuda)
    st.add_rpn(*args)
    with pytest.raises(ValueError, match="seg_result"):
        st.add_rpn(*args, **kw)
    assert st.scenes == NS


@pytest.mark.gpu
def test_no_host_synchronisation(cuda, gold):
    from pointrcnn_b200 import _cabi as C
    from pointrcnn_b200.datasets.eval_stats import EvalStats
    from pointrcnn_b200.ext import roipool3d_cuda
    scenes = _device_scenes(gold, cuda)
    smp = _sampler(cuda)
    ref = smp.prepare_eval_batch(scenes)
    B, M, N = len(scenes), ref["roi_boxes3d"].shape[1], max(len(s["rpn_xyz"]) for s in scenes)
    K = ref["rows"].shape[2] - 3
    lc = C.launch_count()                                # the pooling's own launches at these shapes
    roipool3d_cuda.forward(torch.zeros((B, N, 3), device=cuda), torch.zeros((B, M, 7), device=cuda), torch.zeros((B, N, K), device=cuda),
                           torch.empty((B, M, 512, 3 + K), device=cuda), torch.zeros((B, M), dtype=torch.int32, device=cuda),
                           torch.zeros((B, M, 7), device=cuda), True)
    pool_launches = C.launch_count() - lc
    fed = {name: _batches(name, _scenes(gold), cuda, 8) for name in ("rpn", "rcnn", "joint")}
    stats = {name: EvalStats(device=cuda) for name in fed}
    launches = {}
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        lc = C.launch_count()
        out = smp.prepare_eval_batch(scenes)
        n_prep = C.launch_count() - lc
        for name, batches in fed.items():
            lc = C.launch_count()
            _feed(stats[name], batches)
            launches[name] = C.launch_count() - lc
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert n_prep == pool_launches + 1, (n_prep, pool_launches)        # pooling, gt_iou
    # one batch each: recall + seg; two recalls + cls acc; two recalls + seg
    assert launches == {"rpn": 2, "rcnn": 3, "joint": 3}, launches
    for k, v in ref.items():
        assert torch.equal(v, out[k]), k
    for name, st in stats.items():
        _assert_ret(st.result(), _golden_ret(gold, name), tol={"rcnn_cls_acc_refined": 6e-8})

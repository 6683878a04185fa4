"""CPU suite: the oracle against the golden vectors produced by the reference's own CUDA kernels
(oracle/make_golden.py run on a GPU; tests/golden/reference_kernels.npz)."""
import os
import sys

import numpy as np
import pytest

import inbox_reference as IR
import synth
from oracle import oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
from make_golden import GOLDEN_CASES, cloud  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_kernels.npz")


@pytest.fixture(scope="module")
def gold():
    if not os.path.exists(GOLDEN):
        pytest.skip("golden vectors not generated yet (oracle/make_golden.py needs a GPU box)")
    return np.load(GOLDEN)


@pytest.mark.parametrize("i", range(len(GOLDEN_CASES["fps"])))
def test_fps_golden(gold, i):
    B, N, M, kind, seed = GOLDEN_CASES["fps"][i]
    idx, temp = O.fps(cloud(kind, B, N, seed), M, return_temp=True)
    assert np.array_equal(idx, gold["fps_idx_%d" % i])
    assert np.array_equal(temp, gold["fps_temp_%d" % i])


@pytest.mark.parametrize("i", range(len(GOLDEN_CASES["ball_query"])))
def test_ball_query_golden(gold, i):
    B, N, M, kind, r, ns, seed = GOLDEN_CASES["ball_query"][i]
    xyz = cloud(kind, B, N, seed)
    fidx = O.fps(xyz, M)
    new_xyz = np.stack([xyz[b][fidx[b]] for b in range(B)])
    assert np.array_equal(O.ball_query(r, ns, xyz, new_xyz), gold["bq_idx_%d" % i])


@pytest.mark.parametrize("i", range(len(GOLDEN_CASES["three_nn"])))
def test_three_nn_interpolate_golden(gold, i):
    B, n, m, kind, seed = GOLDEN_CASES["three_nn"][i]
    unknown = cloud(kind, B, n, seed)
    known = np.ascontiguousarray(unknown[:, ::max(1, n // m)][:, :m])
    d2, idx = O.three_nn(unknown, known)
    assert np.array_equal(idx, gold["nn_idx_%d" % i])
    assert np.array_equal(d2, gold["nn_d2_%d" % i])
    rng = np.random.default_rng(seed)
    feats = rng.standard_normal((B, 7, m)).astype(np.float32)
    w = rng.random((B, n, 3)).astype(np.float32)
    assert np.array_equal(O.three_interpolate(feats, idx, w), gold["interp_%d" % i])


@pytest.mark.parametrize("i", range(len(GOLDEN_CASES["nms"])))
def test_nms_golden(gold, i):
    n, thresh, normal, seed = GOLDEN_CASES["nms"][i]
    boxes = synth.sorted_bev(n, seed)
    keep = O.nms(boxes, thresh, bool(normal))
    want = gold["nms_keep_%d" % i]
    if normal:  # pure +,-,*,/,min,max arithmetic: bit-exact on the host
        assert np.array_equal(keep, want)
        rowxor = np.bitwise_xor.reduce(O.nms_mask(boxes, thresh, True), axis=1)
        assert np.array_equal(rowxor, gold["nms_maskrowxor_%d" % i])
    else:       # rotated IoU goes through sinf/cosf/atan2f: host libm vs libdevice may flip borderline pairs
        agree = len(set(keep.tolist()) & set(want.tolist())) / max(1, len(want))
        assert agree >= 0.98


def test_overlap_iou_golden(gold):
    a, b = synth.sorted_bev(120, 17), synth.sorted_bev(90, 18)
    b[:40] = a[10:50] + np.float32(0.02)
    np.testing.assert_allclose(O.boxes_overlap_bev(a, b), gold["overlap"], rtol=2e-4, atol=2e-4)
    np.testing.assert_allclose(O.boxes_iou_bev(a, b), gold["iou_bev"], rtol=2e-4, atol=2e-5)


def test_roipool3d_golden(gold):
    xyz = synth.u_kitti(2, 4096, 19)
    boxes = np.stack([synth.boxes3d(24, 20 + bb)[0] for bb in range(2)])
    rng = np.random.default_rng(21)
    for bb in range(2):
        pick = rng.integers(0, 4096, 12)
        boxes[bb, :12, 0], boxes[bb, :12, 2], boxes[bb, :12, 1] = xyz[bb, pick, 0], xyz[bb, pick, 2], xyz[bb, pick, 1] + 0.8
        boxes[bb, :4, 3:6] *= 6.0
    feat = rng.standard_normal((2, 4096, 5)).astype(np.float32)
    boxes = boxes.astype(np.float32)
    pooled, empty = O.roipool3d(xyz, feat, boxes, 64)
    # the reference kernel's rows (libdevice cos / sin) and the oracle's (host libm): every decision of either agrees with
    # float64 membership outside its band
    for rows, em, who in ((gold["roi_pooled"], gold["roi_empty"], "reference"), (pooled, empty, "oracle")):
        for b in range(2):
            idx = IR.rows_to_index(rows[b], xyz[b], feat[b])
            IR.check_pool_selection(np.where(em[b][:, None] == 1, 0, idx), em[b], xyz[b], boxes[b], where="%s scene %d" % (who, b))
    assert 0 < empty.sum() < empty.size


# ------------------------------------------------------------------------------------------------ CPU twins (row a17)
TWINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "roipool3d_cpu_twins.npz")


@pytest.mark.parametrize("case", ["a", "b", "c"])
def test_cpu_twins_match_the_reference_extension(case):
    """pts_in_boxes3d_cpu / roipool_pc_cpu / roipool3d_cpu of the mirror (numpy twins in ext/roipool3d_cuda.py) against
    the outputs of the reference's OWN roipool3d.cpp (:82-195) + roipool3d_utils.py (:31-108), compiled and run in the
    build container by oracle/make_golden_cpu_twins.py"""
    import torch
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    from make_golden_cpu_twins import CASES, scene
    from pointrcnn_b200.roipool3d import roipool3d_utils as ru
    g = np.load(TWINS)
    name, N, M, C, S, extra, seed = [c for c in CASES if c[0] == case][0]
    pts, boxes, feat = scene(N, M, C, seed)
    masks = ru.pts_in_boxes3d_cpu(torch.from_numpy(pts), torch.from_numpy(boxes))
    assert np.array_equal(np.stack([m.numpy() for m in masks]), g[name + "_mask"])
    pp, pf, pe = ru.roipool_pc_cpu(torch.from_numpy(pts), torch.from_numpy(feat), torch.from_numpy(boxes), S)
    assert np.array_equal(pe.numpy(), g[name + "_pc_empty"])
    assert np.array_equal(pp.numpy(), g[name + "_pc_pts"]) and np.array_equal(pf.numpy(), g[name + "_pc_feat"])
    ex = feat[:, :2].copy()
    a, b, e = ru.roipool3d_cpu(boxes, pts, feat, ex, extra, sampled_pt_num=S, canonical_transform=False)
    assert np.array_equal(e, g[name + "_rp_empty"]) and np.array_equal(a, g[name + "_rp_input"]) and np.array_equal(b, g[name + "_rp_feat"])
    keep = g[name + "_rpc_keep"]
    a2, b2 = ru.roipool3d_cpu(boxes[keep], pts, feat, ex, extra, sampled_pt_num=S, canonical_transform=True)
    assert np.array_equal(b2, g[name + "_rpc_feat"])
    # the canonical rotation goes through float64 cos/sin + np.dot in the reference (kitti_utils.py:33-43): same here
    np.testing.assert_allclose(a2, g[name + "_rpc_input"], rtol=0, atol=1e-6)


# ------------------------------------------------------------------------------------------------ host-side torch mirrors
def test_decode_and_losses_match_the_reference_python():
    """bbox_transform.decode_bbox_target and train.losses against the outputs of the reference's own
    lib/utils/bbox_transform.py / loss_utils.py (oracle/make_golden_head_math.py)"""
    import torch
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import make_golden_head_math as G
    from pointrcnn_b200 import bbox_transform as bt
    from pointrcnn_b200.train import losses as L
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "head_math.npz"))
    anchor = torch.tensor(G.ANCHOR)
    for i, case in enumerate(G.DECODE_CASES):
        scope, bs, nh, fine, ybin, cols = case
        roi, reg = G.decode_inputs(i, case)
        got = bt.decode_bbox_target(roi, reg, scope, bs, nh, anchor, True, ybin, 0.5, 0.25, fine).numpy()
        assert np.array_equal(got, g["decode_%d" % i]), "decode case %d" % i
    for i, case in enumerate(G.LOSS_CASES):
        scope, nh, fine, ybin = case
        pred, lab = G.loss_inputs(i, case)
        loc, ang, size, _ = L.get_reg_loss(pred, lab, scope, 0.5, nh, anchor, True, ybin, 0.5, 0.25, fine)
        np.testing.assert_allclose([float(loc), float(ang), float(size)], g["reg_loss_%d" % i], rtol=2e-6, atol=1e-6)
    logits, tgt, w = G.cls_inputs()
    assert np.array_equal(L.SigmoidFocalClassificationLoss(2.0, 0.25)(logits, tgt, w).numpy(), g["focal"])
    np.testing.assert_allclose(float(L.DiceLoss()(logits, tgt)), g["dice"][0], rtol=1e-6)


def test_stage_losses_match_the_reference_functions():
    """train.losses.rpn_loss / rcnn_loss against get_rpn_loss / get_rcnn_loss of lib/net/train_functions.py:55-209 (their own
    source, run by oracle/make_golden_stage_losses.py with tools/cfgs/default.yaml)"""
    import torch
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import make_golden_stage_losses as G
    from pointrcnn_b200.rpn.stage import CLS_MEAN_SIZE
    from pointrcnn_b200.train import losses as L
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stage_losses.npz"))
    mean = torch.from_numpy(CLS_MEAN_SIZE[0])
    cls, reg, lab, rl = G.rpn_inputs()
    for name in ("SigmoidFocalLoss", "DiceLoss", "BinaryCrossEntropy"):
        total, t = L.rpn_loss(cls, reg, lab, rl, mean, loss_cls=name)
        got = [float(total), float(t["rpn_loss_cls"]), float(t["rpn_loss_reg"]), float(t["loss_loc"]), float(t["loss_angle"]), 3 * float(t["loss_size"])]
        np.testing.assert_allclose(got, g["rpn_%s" % name], rtol=3e-6, atol=1e-6, err_msg=name)
    rc, rr, rlab, valid, roi, gt = G.rcnn_inputs()
    for name in ("BinaryCrossEntropy", "SigmoidFocalLoss"):
        for on_roi in (False, True):
            lab_in = rlab.clamp(min=0) if name == "BinaryCrossEntropy" else rlab      # see the generator: {0,1} labels for this variant
            total, t = L.rcnn_loss(rc, rr, lab_in, valid, roi, gt, mean, loss_cls=name, size_res_on_roi=on_roi)
            want = g["rcnn_%s_%d" % (name, int(on_roi))]
            np.testing.assert_allclose([float(total), float(t["rcnn_loss_cls"]), float(t["rcnn_loss_reg"])], want[:3], rtol=3e-6, atol=1e-6,
                                       err_msg="%s %s" % (name, on_roi))
            assert int((valid > 0).sum()) == int(want[3])
    # ignore labels (-1) in the cross-entropy variant: the same loss as on the valid rows alone
    total, t = L.rcnn_loss(rc, rr, rlab, valid, roi, gt, mean, loss_cls="BinaryCrossEntropy")
    keep = rlab >= 0
    ref = torch.nn.functional.binary_cross_entropy(torch.sigmoid(rc.view(-1)[keep]), rlab[keep].float())
    np.testing.assert_allclose(float(t["rcnn_loss_cls"]), float(ref), rtol=1e-6)
    # no foreground row at all: the regression term is an exact zero that still carries the graph
    total0, t0 = L.rcnn_loss(rc.requires_grad_(True), rr, rlab, torch.zeros_like(valid), roi, gt, mean)
    assert float(t0["rcnn_loss_reg"]) == 0.0 and total0.requires_grad

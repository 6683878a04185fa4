"""GPU suite: every device point-in-box decision against the float64 membership of tests/inbox_reference.py, on the
face-hugging, capped, degenerate and far-range families.  A decision outside the band is a kernel bug."""
import numpy as np
import pytest
import torch

import inbox_reference as IR
from oracle import refgpu as R

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200.datasets.kitti_rcnn_dataset import generate_rpn_training_labels  # noqa: E402
from pointrcnn_b200.ext import roipool3d_cuda  # noqa: E402

HAVE_REF = R.available()
# every form of the pooling entries: the one-pass kernel, the binned two-kernel default and its pass-B variants, the
# exhaustive assign pass, the binned pass fused into the copy kernel
FORMS = {"one_pass": None, "binned": {}, "exhaustive": dict(roipool_exhaustive=1), "fused": dict(roipool_fused=1),
         "direct": dict(roipool_direct=1), "stage_kb8": dict(roipool_stage_kb=8), "parts3": dict(roipool_parts=3)}
# (S, C): boxes that saturate S, a row width that is not a multiple of four floats (scalar stores), boxes that do not
SHAPES = [(16, 2), (37, 2), (128, 5)]


def _scenes(family, C_):
    """two scenes of one family; feature 0 is the point index (exact in fp32 below 2^24)"""
    pts, boxes = zip(*(IR.family(family, seed) for seed in (11, 12)))
    xyz, boxes = np.stack(pts), np.stack(boxes)
    rng = np.random.default_rng(len(family))
    feat = rng.standard_normal((2, xyz.shape[1], C_)).astype(np.float32)
    feat[..., 0] = np.arange(xyz.shape[1], dtype=np.float32)
    return xyz, boxes, feat


def _pool(form, x, bx, f, S, rois=None):
    B, M = bx.shape[:2]
    pooled = torch.zeros((B, M, S, 3 + f.shape[2]), device=x.device)
    empty = torch.zeros((B, M), dtype=torch.int32, device=x.device)
    if FORMS[form] is None:
        roipool3d_cuda.forward_one_pass(x, bx, f, pooled, empty, rois_canonical=rois)
    else:
        with C.options(**FORMS[form]):
            roipool3d_cuda.forward(x, bx, f, pooled, empty, rois_canonical=rois)
    torch.cuda.synchronize()
    return pooled.cpu().numpy(), empty.cpu().numpy()


def _check_pooled(pooled, empty, xyz, boxes, feat, rule="pool", where=""):
    """the per-box selection checks of inbox_reference plus bit copies of xyz and features"""
    for b in range(len(xyz)):
        idx = pooled[b, ..., 3].astype(np.int64)
        e = empty[b].astype(bool)
        idx[e] = 0
        IR.check_pool_selection(idx, e, xyz[b], boxes[b], rule, where="%s scene %d" % (where, b))
        want = np.concatenate([xyz[b], feat[b]], 1)[idx]
        got = pooled[b]
        assert np.array_equal(got[~e].view(np.uint32), want[~e].view(np.uint32)), "%s: rows are not bit copies" % where
        assert not got[e].any(), "%s: rows of an empty box were written" % where


def _canonical_bound(pts, rois):
    """|fp32 - float64| of the canonical transform (x, z rotated by the RoI heading after the centre is subtracted): the
    rotation bound of inbox_reference (7U of the products) plus U of each difference"""
    r = rois.astype(np.float64)
    c, s = np.cos(r[..., 6])[..., None], np.sin(r[..., 6])[..., None]
    d = pts.astype(np.float64) - r[..., None, 0:3]
    want = np.stack([d[..., 0] * c - d[..., 2] * s, d[..., 1], d[..., 0] * s + d[..., 2] * c], -1)
    bx = 7 * IR.U * (np.abs(d[..., 0] * c) + np.abs(d[..., 2] * s))
    bz = 7 * IR.U * (np.abs(d[..., 0] * s) + np.abs(d[..., 2] * c))
    bnd = np.stack([bx, IR.U * np.abs(d[..., 1]), bz], -1) * (1 + 2.0 ** -10)
    return want, bnd


@pytest.mark.parametrize("S,C_", SHAPES)
@pytest.mark.parametrize("family", IR.FAMILIES)
def test_roipool3d_every_form_against_float64(cuda, family, S, C_):
    xyz, boxes, feat = _scenes(family, C_)
    x, bx, f = (torch.from_numpy(a).to(cuda) for a in (xyz, boxes, feat))
    first = None
    for form in FORMS:
        pooled, empty = _pool(form, x, bx, f, S)
        _check_pooled(pooled, empty, xyz, boxes, feat, where="%s %s S=%d" % (family, form, S))
        if first is None:
            first = (pooled, empty)
    pooled, empty = first
    if family not in ("degenerate",):
        assert (empty == 0).any(), "the family must fill boxes"
    if HAVE_REF:
        rp, re = R.roipool3d(x, f, bx, S)
        rp, re = rp.cpu().numpy(), re.cpu().numpy()
        _check_pooled(rp, re, xyz, boxes, feat, where="%s reference kernel S=%d" % (family, S))    # tests the band itself
        assert np.array_equal(re, empty) and np.array_equal(rp.view(np.uint32), pooled.view(np.uint32)), \
            "%s: rows differ from the reference kernel" % family


@pytest.mark.parametrize("family", ["random", "faces", "headings", "cap", "far", "degenerate"])
def test_roipool3d_canonical_rows_against_float64(cuda, family):
    """with canonical RoIs the selection is the same, xyz lies within the derived bound of the float64 transform of the
    selected point, features stay bit copies, and empty boxes get the transformed zero rows"""
    S, C_ = 37, 2
    xyz, boxes, feat = _scenes(family, C_)
    rois = boxes.copy()
    rois[..., 6] += np.float32(0.3)                                 # the transform's heading need not be the pool box's
    x, bx, f, r = (torch.from_numpy(a).to(cuda) for a in (xyz, boxes, feat, rois))
    for form in FORMS:
        plain, pe = _pool(form, x, bx, f, S)
        pooled, empty = _pool(form, x, bx, f, S, rois=r)
        assert np.array_equal(pe, empty)
        assert np.array_equal(pooled[..., 3:].view(np.uint32), plain[..., 3:].view(np.uint32)), "%s %s: features" % (family, form)
        e = empty.astype(bool)
        idx = np.where(e[..., None], 0, pooled[..., 3].astype(np.int64))
        got = pooled[..., 0:3].astype(np.float64)
        for b in range(2):
            for m in range(boxes.shape[1]):
                p = np.zeros((S, 3), np.float32) if e[b, m] else xyz[b][idx[b, m]]
                w, bd = _canonical_bound(p[None], rois[b, m][None])
                w, bd = w[0], bd[0]
                fin = np.isfinite(w)
                err = np.abs(got[b, m][fin] - w[fin])
                assert (err <= bd[fin]).all(), "%s %s box %d: canonical xyz off by %g (bound %g)" % (
                    family, form, m, err.max(), bd[fin][np.argmax(err - bd[fin])])
                assert np.array_equal(np.isnan(got[b, m]), np.isnan(w)), "%s %s box %d: NaN pattern" % (family, form, m)
        if e.any():
            assert not pooled[e][..., 3:].any(), "features of empty boxes must stay zero"


# ------------------------------------------------------------------------------------------------ RPN labels
@pytest.mark.parametrize("family", IR.FAMILIES)
def test_rpn_labels_against_float64(cuda, family):
    """cls equals the float64 replay wherever every decision is certain, else is a label the replay allows; reg equals the
    fp32 restatement bit for bit where certain.  Batched with zero rows (skipped without gt_count) and with gt_count (rows
    past the count ignored, whatever they hold); up to 128 boxes per scene"""
    G = 128
    pts0, b0 = IR.family(family, 21, m=G, per=18)                   # 128 real boxes
    pts1, b1 = IR.family(family, 22, m=8, per=18 * 16)
    n = min(len(pts0), len(pts1))
    pts = np.stack([pts0[:n], pts1[:n]])
    gt = np.zeros((2, G, 7), np.float32)
    gt[0, :len(b0)] = b0
    gt[1, 0:16:2] = b1                                              # zero rows between the boxes of scene 1
    p, g = torch.from_numpy(pts).to(cuda), torch.from_numpy(gt).to(cuda)
    cls, reg = generate_rpn_training_labels(p, g)
    cls, reg = cls.cpu().numpy(), reg.cpu().numpy()
    for b in range(2):
        IR.check_labels(cls[b], reg[b], pts[b], gt[b], where="%s scene %d" % (family, b))
    # gt_count: scene 0 keeps its first 40 rows, scene 1 all 128 (its zero rows count as boxes that hold nothing)
    junk = gt.copy()
    junk[0, 40:] = np.resize(b0, (G - 40, 7))                       # real-looking boxes past the count
    cnt = np.array([40, G], np.int32)
    cls2, reg2 = generate_rpn_training_labels(p, torch.from_numpy(junk).to(cuda), gt_count=torch.from_numpy(cnt).to(cuda))
    cls2, reg2 = cls2.cpu().numpy(), reg2.cpu().numpy()
    for b in range(2):
        IR.check_labels(cls2[b], reg2[b], pts[b], junk[b], count=int(cnt[b]), where="%s gt_count scene %d" % (family, b))
    if family in ("random", "faces", "overlap"):
        assert (cls == 1).sum() > 100 and (cls == -1).sum() > 10, "the family must produce foreground and ignore labels"


def test_rpn_labels_host_and_device_entry_agree(cuda):
    """the numpy entry (one scene, gt_count = G) and the batched entry give the same labels"""
    pts, boxes = IR.family("overlap", 5, m=64, per=32)
    c1, r1 = generate_rpn_training_labels(pts, boxes)
    IR.check_labels(c1, r1, pts, boxes, count=len(boxes), where="numpy entry")
    c2, r2 = generate_rpn_training_labels(torch.from_numpy(pts[None]).to(cuda), torch.from_numpy(boxes[None]).to(cuda))
    assert np.array_equal(c2[0].cpu().numpy(), c1) and np.array_equal(r2[0].cpu().numpy().view(np.uint32), r1.view(np.uint32))


# ------------------------------------------------------------------------------------------------ RCNN targets
@pytest.mark.parametrize("recipe", ["loader", "layer"])
@pytest.mark.parametrize("family", ["random", "faces", "cap", "far", "overlap"])
def test_rcnn_targets_pool_the_enlarged_rois(cuda, family, recipe):
    """rcnn/targets.run with the point index as a feature: each sampled RoI's rows are the first S points of its box
    enlarged by POOL_EXTRA_WIDTH (fp32, as enlarge_box3d), checked like every pooling form; ignored rows pool a box with
    negative sizes and come back empty"""
    from oracle import oracle as O
    from pointrcnn_b200.rcnn import targets as T
    cfg = T.ns(dict(T.DEFAULT_CFG, AUG_DATA=False))
    rc = T.loader_recipe(cfg, "TRAIN") if recipe == "loader" else T.layer_recipe(cfg)
    rc = rc._replace(num_points=32)                                 # boxes that fill S and boxes that do not
    xyz, boxes, feat = _scenes(family, 2)
    rng = np.random.default_rng(len(family))
    gts = boxes[:, :12].copy()
    rois = np.repeat(gts, 4, 1)
    rois[..., [0, 2]] += rng.normal(0, 0.4, rois[..., [0, 2]].shape).astype(np.float32)
    rois[..., 6] += rng.normal(0, 0.2, rois[..., 6].shape).astype(np.float32)
    rois = np.ascontiguousarray(rois, np.float32)
    counts = torch.tensor([[rois.shape[1]] * 2, [gts.shape[1]] * 2], dtype=torch.int32, device=cuda)
    x, f, r, g = (torch.from_numpy(np.ascontiguousarray(a)).to(cuda) for a in (xyz, feat, rois, gts))
    o = T.run(rc, x, f, r, g, counts, seed=7)
    torch.cuda.synchronize()
    pooled, empty = o["pooled"].cpu().numpy(), o["empty"].cpu().numpy()
    pb, sampled = o["pool_boxes"].cpu().numpy(), o["rois"].cpu().numpy()
    ignored = (pb[..., 3:6] == -1).all(-1)
    assert empty[ignored].all(), "ignored rows must come back empty"
    want = O.enlarge_box3d(sampled, cfg.RCNN.POOL_EXTRA_WIDTH)
    assert np.array_equal(pb[~ignored].view(np.uint32), want[~ignored].view(np.uint32)), "pool boxes are not the enlarged RoIs"
    for b in range(2):
        e = empty[b].astype(bool)
        idx = np.where(e[:, None], 0, pooled[b, ..., 3].astype(np.int64))
        IR.check_pool_selection(idx, e, xyz[b], pb[b], where="%s %s scene %d" % (family, recipe, b))
        assert np.array_equal(pooled[b][~e][..., 3:].view(np.uint32), feat[b][idx[~e]].view(np.uint32)), "features are not bit copies"
    assert (empty == 0).sum() > 10, "the sampled RoIs must hold points"

"""Input pipeline / KITTI output (SURVEY 8(f) rank 4): oracle and host mirrors against the golden vectors the reference's
own Python produced (oracle/make_golden_kitti_io.py) on CPU; the device pipeline against both on the GPU."""
import os

import numpy as np
import pytest

import inbox_reference as IR
from oracle import kitti_io as KO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "kitti_io.npz")
NPOINTS = 4096
SCENES = [(11, 30000, 6), (12, 4500, 3)]


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD, allow_pickle=False)


def _scans():
    out = []
    for seed, n, g in SCENES:
        lidar, gt, alpha = KO.synth_scan(seed, n, g)
        out.append(dict(lidar=lidar, calib=KO.CALIB, img_shape=KO.IMG_SHAPE, gt_boxes3d=gt, gt_alpha=alpha))
    return out


def _labels_in_band(cls, reg, pts, gt, count="all", delaunay=False, where=""):
    """every label agrees with the float64 replay of generate_rpn_training_labels outside the band of its decisions
    (tests/inbox_reference.py); delaunay=True for the reference's own labels (its hull of the fp32 corners)"""
    gt = np.asarray(gt, np.float32).reshape(-1, 7)
    IR.check_labels(cls, reg, np.asarray(pts)[:, :3], gt, count=len(gt) if count == "all" else count, delaunay=delaunay, where=where)


# ------------------------------------------------------------------------------------------------ CPU: oracle + host mirrors
def test_oracle_reproduces_the_reference_samples(gold):
    scans = _scans()
    np.random.seed(2024)
    for i, s in enumerate(scans):
        o = KO.rpn_sample(s["lidar"], KO.CALIB, KO.IMG_SHAPE, s["gt_boxes3d"], s["gt_alpha"], NPOINTS, np.random, train=True)
        np.testing.assert_allclose(o["pts_input"], gold["train%d_pts_input" % i], rtol=0, atol=2e-5)
        np.testing.assert_allclose(o["gt_boxes3d"], gold["train%d_gt_boxes3d" % i], rtol=0, atol=2e-5)
        assert repr(o["aug_method"]) == str(gold["train%d_aug" % i])
        _labels_in_band(o["rpn_cls_label"], o["rpn_reg_label"], o["pts_input"], o["gt_boxes3d"], where="oracle %d" % i)
        _labels_in_band(gold["train%d_rpn_cls_label" % i], gold["train%d_rpn_reg_label" % i], gold["train%d_pts_input" % i],
                        gold["train%d_gt_boxes3d" % i], delaunay=True, where="reference %d" % i)
        assert (gold["train%d_rpn_cls_label" % i] == 1).sum() > 50, "the fixture must contain foreground points"
    rect = KO.lidar_to_rect(scans[0]["lidar"], KO.CALIB)
    np.testing.assert_allclose(rect, gold["rect0"], rtol=0, atol=1e-5)
    uv, depth = KO.rect_to_img(rect, KO.CALIB)
    assert np.array_equal(KO.get_valid_flag(rect, uv, depth, KO.IMG_SHAPE), gold["valid0"])
    # the reference's flags against the float64 frustum of the packed calibration the device reads
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import Calibration, PC_AREA_SCOPE
    _, cv, ci = IR.frustum(scans[0]["lidar"], Calibration(KO.CALIB).pack(KO.IMG_SHAPE, PC_AREA_SCOPE))
    assert not (gold["valid0"] & ci).any() and not (~gold["valid0"] & cv).any()


def test_oracle_labels_match_the_reference_hull_test(gold):
    cls, reg = KO.rpn_training_labels(gold["probe_pts"], _scans()[0]["gt_boxes3d"])
    _labels_in_band(cls, reg, gold["probe_pts"], _scans()[0]["gt_boxes3d"], where="oracle probe")
    assert (cls == 1).sum() > 500 and (cls == -1).sum() > 200


def test_oracle_kitti_text_matches_the_reference(gold):
    text = KO.kitti_lines(gold["kitti_boxes"], gold["kitti_scores"], KO.CALIB["P2"], KO.IMG_SHAPE)
    names, vals = KO.parse_kitti_text(text)
    gnames, gvals = KO.parse_kitti_text(str(gold["kitti_text"]))
    assert names == gnames and len(gnames) < len(gold["kitti_boxes"]), "the fixture must contain boxes the 0.8 rule drops"
    np.testing.assert_allclose(vals, gvals, rtol=0, atol=2e-4)


def test_host_mirrors_follow_the_reference_random_stream(gold):
    from pointrcnn_b200.datasets import kitti_rcnn_dataset as D
    scans = _scans()
    np.random.seed(2024)
    samples = []
    for i, s in enumerate(scans):
        rect = KO.lidar_to_rect(s["lidar"], KO.CALIB)
        uv, depth = KO.rect_to_img(rect, KO.CALIB)
        ok = KO.get_valid_flag(rect, uv, depth, KO.IMG_SHAPE)
        ch = D.draw_choice_numpy(rect[ok][:, 2], NPOINTS, np.random)
        angle, scale, flip, method = D.draw_augmentation(rng=np.random)
        assert repr(method) == str(gold["train%d_aug" % i])
        g = D.augment_gt_boxes3d(s["gt_boxes3d"], s["gt_alpha"], angle, scale, flip)
        np.testing.assert_allclose(g, gold["train%d_gt_boxes3d" % i], rtol=0, atol=1e-6)
        samples.append(dict(sample_id=i, gt_boxes3d=g, pts_input=gold["train%d_pts_input" % i], random_select=True))
        assert len(ch) == NPOINTS
    batch = D.collate_batch(samples)
    np.testing.assert_allclose(batch["gt_boxes3d"], gold["collate_gt_boxes3d"], rtol=0, atol=1e-6)
    assert tuple(batch["pts_input"].shape) == tuple(gold["collate_pts_input_shape"])
    assert np.array_equal(batch["sample_id"], gold["collate_sample_id"]) and batch["sample_id"].dtype == np.int32


def test_host_formatter_writes_the_reference_text(gold):
    """prb_kitti_format_detections is host code of the C ABI library: runs without a GPU"""
    from pointrcnn_b200.datasets import kitti_output
    ib, alpha, valid = KO.image_boxes(gold["kitti_boxes"], KO.CALIB["P2"], KO.IMG_SHAPE)
    text = kitti_output.format_kitti_lines(gold["kitti_boxes"], ib, alpha, gold["kitti_scores"], valid.astype(np.int32))
    names, vals = KO.parse_kitti_text(text)
    gnames, gvals = KO.parse_kitti_text(str(gold["kitti_text"]))
    assert names == gnames
    np.testing.assert_allclose(vals, gvals, rtol=0, atol=2e-4)
    assert text.count("\n") == len(gnames) and text.startswith("Car -1 -1 ")


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_pipeline_with_the_reference_stream_matches_the_reference(cuda, gold):
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import RPNInputPipeline
    pipe = RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="numpy", device=cuda)
    np.random.seed(2024)
    # the reference draws sample 0's choice, then sample 0's augmentation, then sample 1's: one scene per call keeps that order
    scans = _scans()
    for i, s in enumerate(scans):
        out = pipe.prepare_batch([s], rng=np.random)
        np.testing.assert_allclose(out["pts_input"][0].cpu().numpy(), gold["train%d_pts_input" % i], rtol=0, atol=2e-5)
        np.testing.assert_allclose(out["pts_features"][0].cpu().numpy(), gold["train%d_pts_features" % i], rtol=0, atol=1e-7)
        np.testing.assert_allclose(out["gt_boxes3d"][0].cpu().numpy(), gold["train%d_gt_boxes3d" % i], rtol=0, atol=1e-6)
        assert repr(out["aug_method"][0]) == str(gold["train%d_aug" % i])
        _labels_in_band(out["rpn_cls_label"][0].cpu().numpy(), out["rpn_reg_label"][0].cpu().numpy(), out["pts_input"][0].cpu().numpy(),
                        out["gt_boxes3d"][0].cpu().numpy(), where="device %d" % i)
    ev = RPNInputPipeline(npoints=NPOINTS, mode="EVAL", draw="numpy", device=cuda)
    np.random.seed(7)
    out = ev.prepare_batch([scans[0]], rng=np.random)
    np.testing.assert_allclose(out["pts_input"][0].cpu().numpy(), gold["eval0_pts_input"], rtol=0, atol=2e-5)
    assert "aug_method" not in out
    _labels_in_band(out["rpn_cls_label"][0].cpu().numpy(), out["rpn_reg_label"][0].cpu().numpy(), out["pts_input"][0].cpu().numpy(),
                    out["gt_boxes3d"][0].cpu().numpy(), where="device eval")
    np.testing.assert_allclose(out["gt_boxes3d"][0].cpu().numpy(), gold["eval0_gt_boxes3d"], rtol=0, atol=1e-6)
    test = RPNInputPipeline(npoints=NPOINTS, mode="TEST", draw="device", device=cuda).prepare_batch(scans)
    assert "rpn_cls_label" not in test and "gt_boxes3d" not in test


@pytest.mark.gpu
def test_prepare_kernel_matches_the_reference_calibration(cuda, gold):
    import torch
    from pointrcnn_b200 import _cabi as C
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import Calibration, PC_AREA_SCOPE
    s = _scans()[0]
    n = len(s["lidar"])
    lidar = torch.from_numpy(s["lidar"]).to(cuda)
    calib = torch.from_numpy(Calibration(KO.CALIB).pack(KO.IMG_SHAPE, PC_AREA_SCOPE)[None]).to(cuda)
    offsets = torch.tensor([0, n], dtype=torch.int32, device=cuda)
    rect = torch.empty((n, 3), device=cuda)
    flags = torch.empty(n, dtype=torch.uint8, device=cuda)
    counts = torch.empty((1, 2), dtype=torch.int32, device=cuda)
    C.check(C.lib().prb_kitti_prepare_points(1, n, C.ptr(offsets), C.ptr(lidar), 4, C.ptr(calib), 1, C.ptr(rect), C.ptr(flags), C.ptr(counts),
                                             C.stream()), "prepare")
    np.testing.assert_allclose(rect.cpu().numpy(), gold["rect0"], rtol=0, atol=2e-5)
    valid = (flags.cpu().numpy() & 1).astype(bool)
    # the flags against the float64 frustum and range box outside its band; the near bit is rect z < 40 m of the kernel's
    # own rect; the counts are the population counts of the kernel's own flags
    _, cv, ci = IR.frustum(s["lidar"], calib[0].cpu().numpy())
    assert not (valid & ci).any() and not (~valid & cv).any(), "validity flags outside the band of the float64 frustum"
    near = (flags.cpu().numpy() & 2).astype(bool)
    assert np.array_equal(near, rect.cpu().numpy()[:, 2] < np.float32(40.0))
    assert int(counts[0, 0]) == int(valid.sum()) and int(counts[0, 1]) == int((valid & ~near).sum())
    assert 0 < int(counts[0, 1]) < int(counts[0, 0]) < n


@pytest.mark.gpu
def test_device_draw_has_the_reference_distribution_rules(cuda):
    import torch
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import RPNInputPipeline
    scans = _scans()
    pipe = RPNInputPipeline(npoints=NPOINTS, mode="TEST", draw="device", device=cuda)
    a = pipe.prepare_batch(scans, seed=5)
    b = pipe.prepare_batch(scans, seed=5)
    c = pipe.prepare_batch(scans, seed=6)
    assert torch.equal(a["choice"], b["choice"]) and not torch.equal(a["choice"], c["choice"])
    assert a["status"].tolist() == [0, 0]
    for i, s in enumerate(scans):
        rect = KO.lidar_to_rect(s["lidar"], KO.CALIB)
        uv, depth = KO.rect_to_img(rect, KO.CALIB)
        ok = KO.get_valid_flag(rect, uv, depth, KO.IMG_SHAPE)
        ch = a["choice"][i].cpu().numpy()
        assert ok[ch].mean() > 0.999, "only valid points may be drawn"
        got = a["pts_input"][i].cpu().numpy()
        np.testing.assert_allclose(got[:, :3], rect[ch], rtol=0, atol=2e-5)
        np.testing.assert_allclose(got[:, 3], s["lidar"][ch, 3] - 0.5, rtol=0, atol=1e-7)
        nv = int(ok.sum())
        uniq, cnt = np.unique(ch, return_counts=True)
        if nv > NPOINTS:           # every far point + distinct near points
            assert cnt.max() == 1
            far = np.nonzero(ok & (rect[:, 2] >= 40.0))[0]
            assert np.isin(far, ch).mean() > 0.999
        else:                      # every valid point once + distinct extra copies
            assert len(uniq) >= nv - 2 and cnt.max() == 2 and (cnt == 2).sum() == NPOINTS - len(uniq)
        # shuffled: the far points are not bunched at either end, indices are not sorted
        assert np.abs(np.corrcoef(np.arange(NPOINTS), ch)[0, 1]) < 0.1
    # a uniform draw: every seed takes exactly `need` of the near points, each with the same probability
    rect = KO.lidar_to_rect(scans[0]["lidar"], KO.CALIB)
    uv, depth = KO.rect_to_img(rect, KO.CALIB)
    ok = KO.get_valid_flag(rect, uv, depth, KO.IMG_SHAPE)
    near = ok & (rect[:, 2] < 40.0)
    q = (NPOINTS - int((ok & ~near).sum())) / float(near.sum())
    hits = np.zeros(len(rect))
    for seed in range(24):
        ch = pipe.prepare_batch(scans[:1], seed=100 + seed)["choice"][0].cpu().numpy()
        hits[ch] += 1
    p = hits[near] / 24.0
    assert abs(p.mean() - q) < 2e-3 and p.std() < 1.5 * np.sqrt(q * (1 - q) / 24.0), (p.mean(), q, p.std())


@pytest.mark.gpu
def test_empty_and_degenerate_scenes(cuda):
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import RPNInputPipeline
    scans = _scans()
    behind = scans[1]["lidar"].copy()
    behind[:, 0] = -np.abs(behind[:, 0]) - 1.0          # everything behind the camera: no valid point
    few = scans[1]["lidar"][:900].copy()                # far fewer valid points than npoints / 2: whole extra copies
    batch = [dict(scans[0]), dict(scans[1], lidar=behind), dict(scans[1], lidar=few), dict(scans[1], lidar=few[:0])]
    out = RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="device", aug_data=False, device=cuda).prepare_batch(batch, seed=1)
    assert out["status"].tolist() == [0, 1, 0, 1]
    assert float(out["pts_rect"][3].abs().max()) == 0.0 and float(out["pts_input"][1].abs().max()) == 0.0
    ch = out["choice"][2].cpu().numpy()
    nv = int(out["valid_counts"][2, 0])
    assert 0 < nv < NPOINTS // 2
    uniq, cnt = np.unique(ch, return_counts=True)
    assert len(uniq) == nv and cnt.max() - cnt.min() <= 1
    assert (out["rpn_cls_label"][0] == 1).sum() > 0 and tuple(out["gt_boxes3d"].shape) == (4, 6, 7)


@pytest.mark.gpu
def test_labels_kernel_vs_oracle_and_reference(cuda, gold):
    import torch
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import generate_rpn_training_labels
    gt = _scans()[0]["gt_boxes3d"]
    cls, reg = generate_rpn_training_labels(gold["probe_pts"], gt)            # numpy in, numpy out (reference signature)
    assert cls.dtype == np.int32 and reg.dtype == np.float32
    _labels_in_band(cls, reg, gold["probe_pts"], gt, where="device probe")
    # batched, zero-padded GT rows are skipped; overlapping boxes: the later box wins, as in the reference's loop
    pts = torch.from_numpy(np.stack([gold["probe_pts"], gold["probe_pts"]])).to(cuda)
    g2 = np.zeros((2, 8, 7), np.float32)
    g2[0, :6] = gt
    g2[1, :6] = gt
    g2[1, 6] = gt[0] + np.array([0.3, 0, 0.2, 0, 0, 0, 0.1], np.float32)       # overlaps box 0
    c2, r2 = generate_rpn_training_labels(pts, torch.from_numpy(g2).to(cuda))
    assert np.array_equal(c2[0].cpu().numpy(), cls)
    _labels_in_band(c2[1].cpu().numpy(), r2[1].cpu().numpy(), gold["probe_pts"], g2[1], count=None, where="device batched")


@pytest.mark.gpu
def test_save_kitti_format_writes_the_reference_file(cuda, gold, tmp_path):
    import torch
    from pointrcnn_b200.datasets.kitti_output import save_kitti_format
    boxes = torch.from_numpy(gold["kitti_boxes"]).to(cuda)
    scores = torch.from_numpy(gold["kitti_scores"]).to(cuda)
    path = save_kitti_format(42, KO.CALIB, boxes, str(tmp_path), scores, KO.IMG_SHAPE)
    assert os.path.basename(path) == "000042.txt"
    names, vals = KO.parse_kitti_text(open(path).read())
    gnames, gvals = KO.parse_kitti_text(str(gold["kitti_text"]))
    assert names == gnames
    np.testing.assert_allclose(vals, gvals, rtol=0, atol=2e-4)
    empty = save_kitti_format(43, KO.CALIB, boxes[:0], str(tmp_path), scores[:0], KO.IMG_SHAPE)
    assert open(empty).read() == ""

"""Offline RCNN training samples: the oracle against what the reference's own get_rcnn_training_sample_batch produced
(oracle/make_golden_rcnn_offline.py), the feature-file reader / writer, the hash restatement; on the GPU the sample and
targets stages against the oracle in its device mode, seeding, synchronisation and the offline training step."""
import os
import tempfile

import numpy as np
import pytest

from oracle import make_golden_rcnn_offline as MG
from oracle import rcnn_offline as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "rcnn_offline.npz")
RUN_CFG = dict(MG.CFG)


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD, allow_pickle=False)


def _cfg(method, **kw):
    return dict(RUN_CFG, REG_AUG_METHOD=method, **kw)


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_reproduces_the_reference_sample(gold):
    np.random.seed(MG.SEED)
    seen_tries, branches = set(), set()
    for i, (seed, kind, method) in enumerate(MG.RUNS):
        o = RO.sample_scene(RO.synth_scene(seed, kind), _cfg(method), draw="numpy", iou="exact", rng=np.random)
        np.testing.assert_array_equal(o["sel"], gold["run%d_sel" % i])
        np.testing.assert_array_equal(o["iou"], gold["run%d_iou" % i])
        np.testing.assert_array_equal(o["rois"], gold["run%d_rois" % i])
        np.testing.assert_array_equal(o["pooled_input"], gold["run%d_pooled_input" % i])
        np.testing.assert_array_equal(o["pooled_features"], gold["run%d_pooled_features" % i])
        np.testing.assert_array_equal(o["empty"], gold["run%d_empty" % i])
        for k in MG.KEYS:
            np.testing.assert_array_equal(o[k], gold["run%d_%s" % (i, k)], err_msg="run %d %s" % (i, k))
        seen_tries |= set(o["sel"][:, 2].tolist())
        branches.add(o["branch"])
        assert o["empty"].any() or kind == "hard"
    np.testing.assert_array_equal(np.random.get_state()[1], gold["rng_state"])
    # the fixture covers early stops and full 10-try loops, the fg+bg and bg-only branches
    assert 1 in seen_tries and 10 in seen_tries and len(seen_tries) > 4
    assert branches == {"fg+bg", "bg"}


def test_fixture_covers_the_candidate_lists():
    from oracle import gt_paste as GP
    for seed, kind, _ in MG.RUNS:
        s = RO.synth_scene(seed, kind)
        m = GP.iou3d(RO.corners3d(s["roi_boxes3d"]), RO.corners3d(s["gt_boxes3d"]))
        mo = m.max(1)
        for t in RO.THRESHOLDS:
            assert np.abs(m - t).min() >= 1e-5
        hard, easy = ((mo < 0.45) & (mo >= 0.05)).sum(), (mo < 0.05).sum()
        if kind == "hard":
            assert hard and not easy
        if kind == "easy":
            assert easy and not hard
        if kind == "mixed":
            ra = m.argmax(0)[m.max(0) > 0]
            assert (mo[ra] >= 0.55).any() and (mo[ra] < 0.55).any(), "roi_assignment rows over and under the threshold"


def test_feature_files_round_trip_byte_for_byte(gold):
    import torch
    from pointrcnn_b200.datasets.rcnn_offline import read_rpn_features, write_rpn_features_batch
    fs = MG.file_scene()
    with tempfile.TemporaryDirectory() as d:
        t = lambda a: torch.from_numpy(a)[None]
        write_rpn_features_batch(d, [7], t(fs["seg"]), t(fs["rawscore"]), t(fs["pts_features"][:, 0]), t(fs["xyz"]), t(fs["features"]))
        for suffix in ("", "_xyz", "_seg", "_intensity", "_rawscore"):
            with open(os.path.join(d, "%06d%s.npy" % (7, suffix)), "rb") as f:
                assert f.read() == gold["file%s" % (suffix or "_features")].tobytes(), suffix
        xyz, feat, inten, seg = read_rpn_features(d, 7)
        np.testing.assert_array_equal(xyz, fs["xyz"])
        np.testing.assert_array_equal(feat, fs["features"].T)
        np.testing.assert_array_equal(inten, fs["pts_features"][:, 0])
        np.testing.assert_array_equal(seg, fs["seg"])
        seg2 = read_rpn_features(d, 7, use_seg_score=True)[3]
        np.testing.assert_allclose(seg2, 1 / (1 + np.exp(-fs["rawscore"].astype(np.float64))), rtol=1e-6)


def test_read_rois_parses_proposal_files():
    from pointrcnn_b200.datasets.rcnn_offline import read_rois
    s = RO.synth_scene(11, "mixed")
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "000003.txt"), "w") as f:
            f.write("\n".join(MG.label_line("Car", b, 0.25) for b in s["roi_boxes3d"]) + "\n")
        np.testing.assert_array_equal(read_rois(d, 3), s["roi_boxes3d"])


def test_hash_restatement_fixed_values():
    # pinned values of common.cuh's mix32 / draw_key and rcnn_sample.cu's key layout; the GPU tests check the device
    # against this restatement draw by draw (selections and jittered boxes bit for bit)
    assert RO.mix32(0) == 0 and RO.mix32(1) == 0x688990c0
    assert RO.draw_key(0, 0, 1, 0) == 0x1efee872 and RO.draw_key(2026, 3, 17, RO.SALT_FG) == 0xeddc6aec
    assert RO.rs_key(7, 3, RO.SALT_JITTER, 5, 2, 4) == 0xf3539bde == RO.draw_key(7, 3, (5 << 12) | (2 << 6) | 4, RO.SALT_JITTER)
    assert RO.u01(0xffffffff) == np.float32(1 - 2.0 ** -24) and RO.u01(0xff) == 0
    assert RO.pick(0xffffffff, 5) == 4 and RO.pick(0, 5) == 0
    assert [RO.draw_key(0, 0, i, 0) for i in range(3)] == [0, RO.mix32(0x85ebca6b), RO.mix32((2 * 0x85ebca6b) & 0xffffffff)]


# ------------------------------------------------------------------------------------------------ GPU
SCENES = [(31, "mixed", 0), (32, "hard", 0), (33, "easy", 0), (34, "bg", 0), (35, "mixed", 1), (36, "mixed", 2), (37, "mixed", 3)]
STATUS = [0, 0, 0, 0, 0, 2, 2]


def _scenes():
    out = []
    for seed, kind, special in SCENES:
        s = RO.synth_scene(seed, kind)
        if special == 1:        # every RoI over the threshold: the fg-only branch
            s["roi_boxes3d"] = np.repeat(s["gt_boxes3d"], 3, 0)
        if special == 2:        # no RoI: status 2
            s["roi_boxes3d"] = np.zeros((0, 7), np.float32)
        if special == 3:        # no GT box: status 2
            s["gt_boxes3d"] = np.zeros((0, 7), np.float32)
        out.append(s)
    return out


def _sampler(method, cuda, **kw):
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    from pointrcnn_b200.rcnn.targets import DEFAULT_CFG, ns
    d = {k: v for k, v in DEFAULT_CFG.items() if k != "RCNN"}
    d["RCNN"] = dict(DEFAULT_CFG["RCNN"], REG_AUG_METHOD=method, **{k: v for k, v in dict(RUN_CFG, **kw).items()})
    return RCNNOfflineSampler(cfg=ns(d), device=cuda)


def _np(batch):
    return {k: v.cpu().numpy() for k, v in batch.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["multiple", "single", "normal"])
def test_device_sample_matches_the_oracle(cuda, method):
    scenes = _scenes()
    seed = 77
    out = _np(_sampler(method, cuda).prepare_batch(scenes, seed=seed))
    R, S = RUN_CFG["ROI_PER_IMAGE"], RUN_CFG["NUM_POINTS"]
    assert out["sample_status"].tolist() == STATUS
    branches = set()
    for b, s in enumerate(scenes):
        o = RO.sample_scene(s, _cfg(method), draw="hash", iou="fp32", seed=seed, scene_index=b)
        rows = slice(b * R, (b + 1) * R)
        assert out["sample_status"][b] == o["status"]
        branches.add(o["branch"])
        np.testing.assert_array_equal(out["cls_label"][rows], o["cls_label"])
        np.testing.assert_array_equal(out["reg_valid_mask"][rows], o["reg_valid_mask"])
        np.testing.assert_array_equal(out["pooled_empty_flag"][rows], o["empty"])
        if method != "normal":
            np.testing.assert_array_equal(out["sample_index"][rows], o["sel"])
            # oracle.boxes_iou3d is the overlap's op sequence compiled for the host: a few ulp from the device's inline IoU, so
            # the IoUs agree within a bound; selections and tries agree exactly as long as no IoU lies that close to a threshold
            np.testing.assert_allclose(out["gt_iou"][rows], o["iou"], rtol=0, atol=1e-5)
            # the pooled feature columns pin which points were pooled; xyz moved with the augmentation (bounded below)
            np.testing.assert_array_equal(out["pts_features"][rows], o["pts_features"])
            np.testing.assert_array_equal(out["pts_input"][rows][..., 3:4], o["pooled_input"][..., 3:4])
            np.testing.assert_allclose(out["pts_input"][rows][..., 4], o["pooled_input"][..., 4], rtol=0, atol=1e-6)
        else:
            # Box-Muller through logf / sinf: sources and GT assignment exact, boxes and IoUs within fp32 rounding
            np.testing.assert_array_equal(out["sample_index"][rows][:, :2], o["sel"][:, :2])
            same = out["sample_index"][rows][:, 2] == o["sel"][:, 2]
            assert same.mean() > 0.9
            np.testing.assert_allclose(out["gt_iou"][rows][same], o["iou"][same], rtol=0, atol=1e-4)
        bound = lambda a: 2e-5 * max(1.0, np.abs(a).max())
        close = lambda a, e, tol: np.testing.assert_allclose(a, e, rtol=0, atol=tol)
        # augmented and canonical values go through sinf / cosf / atan2f: within 2e-5 of the coordinate range; for "normal"
        # on the rows whose jitter loops agree
        keep = slice(None) if method != "normal" else same
        close(out["pts_input"][rows][keep][..., 0:3], o["pts_input"][keep][..., 0:3], bound(o["pts_input"][..., 0:3]))
        close(out["roi_boxes3d"][rows][keep], o["roi_boxes3d"][keep], bound(o["roi_boxes3d"]))
        close(out["gt_boxes3d"][rows][keep], o["gt_boxes3d"][keep], bound(o["gt_boxes3d"]))
        close(out["gt_boxes3d_ct"][rows][keep], o["gt_boxes3d_ct"][keep], bound(o["gt_boxes3d"]))
    assert branches == {"fg+bg", "bg", "fg", "none"}


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["multiple", "single", "normal"])
def test_device_jitter_without_augmentation(cuda, method):
    scenes = _scenes()
    out = _np(_sampler(method, cuda).prepare_batch(scenes, seed=5, mode="EVAL"))
    R = RUN_CFG["ROI_PER_IMAGE"]
    agree = []
    for b, s in enumerate(scenes):
        o = RO.sample_scene(s, _cfg(method), draw="hash", iou="fp32", seed=5, scene_index=b, train=False)
        rows = slice(b * R, (b + 1) * R)
        np.testing.assert_array_equal(out["gt_boxes3d"][rows], o["gt_of_rois"])
        if method != "normal":
            np.testing.assert_array_equal(out["roi_boxes3d"][rows], o["rois"])          # jittered boxes, bit for bit
        else:
            # Box-Muller with logf / sincospif against float64: boxes within 1e-5 where the loops took the same tries
            same = out["sample_index"][rows][:, 2] == o["sel"][:, 2]
            agree.append(same.mean())
            np.testing.assert_allclose(out["roi_boxes3d"][rows][same], o["rois"][same], rtol=0, atol=1e-5)
    assert not agree or min(agree) > 0.9


@pytest.mark.gpu
def test_status_one_when_no_roi_is_fg_or_bg(cuda):
    scenes = _scenes()[3:4]       # no RoI overlaps a GT: with both bg thresholds at 0 nothing is fg or bg
    out = _np(_sampler("multiple", cuda, CLS_BG_THRESH=0.0, CLS_BG_THRESH_LO=0.0).prepare_batch(scenes, seed=1))
    assert out["sample_status"].tolist() == [1]
    assert (out["cls_label"] == -1).all() and not out["reg_valid_mask"].any() and not out["rows"].any()


@pytest.mark.gpu
def test_non_positive_rotation_range_is_rejected(cuda):
    smp = _sampler("multiple", cuda)
    smp.cfg.AUG_ROT_RANGE = 0           # -pi / 0: the rotation interval is not finite
    with pytest.raises(RuntimeError, match="rotation interval"):
        smp.prepare_batch(_scenes()[:1], seed=1)


def test_loader_recipe_requires_the_counts():
    from pointrcnn_b200.rcnn import targets
    with pytest.raises(ValueError, match="counts"):
        targets.run(targets.loader_recipe(targets.ns(targets.DEFAULT_CFG), "TRAIN"), None, None, None, None, None, 0)


@pytest.mark.gpu
def test_device_sample_is_seeded(cuda):
    import torch
    smp = _sampler("multiple", cuda)
    scenes = _scenes()
    runs = [smp.prepare_batch(scenes, seed=sd) for sd in (3, 3, 4)]
    for k, v in runs[0].items():
        assert torch.equal(v, runs[1][k]), k
    assert not torch.equal(runs[0]["rows"], runs[2]["rows"])
    assert not torch.equal(runs[0]["sample_index"], runs[2]["sample_index"])


@pytest.mark.gpu
def test_device_input_does_not_synchronise(cuda):
    import torch
    from pointrcnn_b200 import _cabi as C
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    scenes = [{k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda) for k, v in s.items()} for s in _scenes()]
    from pointrcnn_b200.ext import roipool3d_cuda
    smp = RCNNOfflineSampler(device=cuda)                # the recipe's defaults: 64 RoIs, 512 points
    ref = smp.prepare_batch(scenes, seed=2)
    B, N, K = len(scenes), max(len(s["rpn_xyz"]) for s in scenes), ref["rows"].shape[2] - 3
    lc = C.launch_count()                                # the pooling's own launches at these shapes (two or three passes)
    roipool3d_cuda.forward(torch.zeros((B, N, 3), device=cuda), torch.zeros((B, 64, 7), device=cuda), torch.zeros((B, N, K), device=cuda),
                           torch.empty((B, 64, 512, 3 + K), device=cuda), torch.zeros((B, 64), dtype=torch.int32, device=cuda), None, True)
    pool_launches = C.launch_count() - lc
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        lc = C.launch_count()
        out = smp.prepare_batch(scenes, seed=2)
        launches = C.launch_count() - lc
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert launches == 3 + pool_launches, (launches, pool_launches)       # iou3d, sample, pool, targets
    assert out["rows"].shape == (len(scenes) * 64, 512, 3 + 2 + 3)
    for k, v in ref.items():
        assert torch.equal(v, out[k]), k
    # numpy input gives the same batch
    host = smp.prepare_batch(_scenes(), seed=2)
    for k, v in ref.items():
        if k != "rows" and k != "pts_input":
            assert torch.equal(v, host[k]), k
    assert out["pts_input"].data_ptr() == out["rows"].data_ptr()


@pytest.mark.gpu
def test_offline_training_step(cuda):
    import torch
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    from pointrcnn_b200.train.losses import rcnn_loss
    from pointrcnn_b200.train.step import RCNNTrainer
    rng = np.random.default_rng(0)
    scenes = _scenes()[:4]
    for s in scenes:
        s["rpn_features"] = rng.standard_normal((len(s["rpn_xyz"]), 128)).astype(np.float32)
    batch = RCNNOfflineSampler(device=cuda).prepare_batch(scenes, seed=9)
    tr = RCNNTrainer(device=cuda)
    c = tr.model.cfg
    loss, _ = tr.forward_loss_offline(batch)
    cls, reg = tr.model.forward_pts(batch["rows"])
    again, _ = rcnn_loss(cls, reg, batch["cls_label"], batch["reg_valid_mask"], batch["roi_boxes3d"], batch["gt_boxes3d_ct"], tr.mean_size,
                         loc_scope=c["LOC_SCOPE"], loc_bin_size=c["LOC_BIN_SIZE"], num_head_bin=c["NUM_HEAD_BIN"], loc_y_by_bin=c["LOC_Y_BY_BIN"],
                         loc_y_scope=c["LOC_Y_SCOPE"], loc_y_bin_size=c["LOC_Y_BIN_SIZE"])
    assert torch.allclose(loss, again, rtol=1e-5, atol=1e-6)
    before = [p.detach().clone() for p in tr.params]
    loss, terms = tr.step_offline(batch)
    assert torch.isfinite(loss).item() and (batch["reg_valid_mask"] > 0).any().item()
    assert any(not torch.equal(a, p.detach()) for a, p in zip(before, tr.params))

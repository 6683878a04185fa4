"""RCNN targets of the in-network recipe (ROI_SAMPLE_JIT): the CPU restatement (oracle/rcnn_offline.py, recipe "layer") against what the
reference's own ProposalTargetLayer produced (tests/golden/proposal_target_layer.npz), prepare_jit_batch's packing
against collate_batch; on the GPU ProposalTargetLayer(draw="device") against the restatement with the device's keys,
seeding, synchronisation, draw statistics and the training steps."""
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import make_golden_proposal_target as MGT
from oracle import make_golden_rcnn_offline as MG
from oracle import rcnn_offline as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "proposal_target_layer.npz")
SMALL = dict(NUM_POINTS=64, ROI_PER_IMAGE=32)


def _layer_oracle(scene, cfg, draw, **kw):
    """the layer's restatement of one scene, with its outputs under the layer's keys: sampled_pts (R,S,3) and pts_feature
    (R,S,F) after the canonical transform, gt_of_rois_ct (R,7)"""
    o = RO.sample_scene(scene, cfg, draw=draw, iou="fp32", recipe="layer", **kw)
    return dict(o, sampled_pts=o["pts_input"][..., 0:3], pts_feature=np.concatenate([o["pooled_input"][..., 3:], o["pooled_features"]], axis=2),
                gt_of_rois_ct=o["gt_boxes3d_ct"])


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_reproduces_the_reference_layer():
    g = np.load(GOLD)
    inp = MGT.inputs()
    np.random.seed(MGT.SEED)
    torch.manual_seed(MGT.SEED)
    outs = [_layer_oracle({k: v[b] for k, v in inp.items()}, dict(ROI_FG_AUG_TIMES=0, AUG_DATA=False), "ref") for b in range(2)]
    cat = lambda k: np.concatenate([o[k] for o in outs])
    for gk, ok in (("roi_boxes3d", "roi_boxes3d"), ("gt_iou", "iou"), ("gt_of_rois", "gt_of_rois_ct"), ("sampled_pts", "sampled_pts"),
                   ("pts_feature", "pts_feature"), ("cls_label", "cls_label"), ("reg_valid_mask", "reg_valid_mask")):
        np.testing.assert_array_equal(cat(ok).astype(g[gk].dtype), g[gk], err_msg=gk)
    # the fixture's GT lists are zero-padded (7 and 6 of 12 rows): the trimming decides the GT assignment
    assert [len(RO.trimmed_gt(inp["gt_boxes3d"][b])) for b in range(2)] == [7, 6]
    assert (cat("sel")[:, 2] == 0).all() and {o["branch"] for o in outs} == {"fg+bg"}


def _collate(scenes):
    """collate_batch (kitti_rcnn_dataset.py:1104-1137) with ROI_SAMPLE_JIT on get_rcnn_sample_jit dicts of one N"""
    out = {}
    for key in ("roi_boxes3d", "gt_boxes3d"):
        m = max(len(s[key]) for s in scenes)
        a = np.zeros((len(scenes), m, 7), np.float32)
        for i, s in enumerate(scenes):
            a[i, :len(s[key])] = s[key]
        out[key] = a
    for key in ("rpn_xyz", "rpn_features", "rpn_intensity", "seg_mask", "pts_depth"):
        out[key] = np.concatenate([s[key][np.newaxis, ...] for s in scenes], axis=0)
    return out


def test_jit_packing_follows_collate_batch():
    from pointrcnn_b200.datasets.rcnn_offline import pack_jit_scenes
    scenes = [RO.synth_scene(s, k) for s, k in ((1, "mixed"), (2, "hard"), (3, "bg"))]
    scenes[2]["gt_boxes3d"] = scenes[2]["gt_boxes3d"][:1]
    ref = _collate([dict(s, pts_depth=np.linalg.norm(s["rpn_xyz"], ord=2, axis=1)) for s in scenes])
    buf, v = pack_jit_scenes(scenes)
    for k, a in ref.items():
        assert v[k].dtype == np.float32 and v[k].shape == a.shape, k
        np.testing.assert_array_equal(v[k], a, err_msg=k)
    assert v["roi_count"].tolist() == [len(s["roi_boxes3d"]) for s in scenes] and v["gt_count"].tolist() == [3, 3, 1]
    assert all(np.shares_memory(buf, a) for a in v.values())           # one buffer: one upload
    # a shorter scene: points at infinity, which no box contains
    short = dict(scenes[0], rpn_xyz=scenes[0]["rpn_xyz"][:100], rpn_features=scenes[0]["rpn_features"][:100],
                 rpn_intensity=scenes[0]["rpn_intensity"][:100], seg_mask=scenes[0]["seg_mask"][:100])
    _, v = pack_jit_scenes([scenes[1], short])
    assert np.isinf(v["rpn_xyz"][1, 100:]).all() and np.isinf(v["pts_depth"][1, 100:]).all() and not v["rpn_features"][1, 100:].any()


# ------------------------------------------------------------------------------------------------ GPU
KINDS = [(41, "mixed"), (42, "hard"), (43, "easy"), (44, "bg"), (45, "mixed"), (46, "mixed")]


def _scenes():
    out = [RO.synth_scene(seed, kind) for seed, kind in KINDS]
    out[4]["gt_boxes3d"] = np.zeros((2, 7), np.float32)        # every GT row is padding: status 2
    return out


def _layer(cuda, **kw):
    from pointrcnn_b200.rcnn.targets import DEFAULT_CFG, ns
    from pointrcnn_b200.rpn.proposal_target_layer import ProposalTargetLayer
    d = {k: v for k, v in DEFAULT_CFG.items() if k != "RCNN"}
    d["RCNN"] = dict(DEFAULT_CFG["RCNN"], **{k: v for k, v in kw.items() if k not in d})
    d.update({k: v for k, v in kw.items() if k in d})
    return ProposalTargetLayer(cfg=ns(d), draw="device")


def _batch(cuda, scenes):
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    return RCNNOfflineSampler(device=cuda).prepare_jit_batch(scenes)


def _np(d):
    return {k: v.cpu().numpy() for k, v in d.items()}


def _oracle_scene(batch, b, n_pts):
    """scene b of a packed batch as the layer sees it: every RoI row (zero padding included), the real points"""
    h = {k: v[b].cpu().numpy() for k, v in batch.items() if k not in ("roi_count", "gt_count")}
    for k in ("rpn_xyz", "rpn_features", "rpn_intensity", "seg_mask", "pts_depth"):
        h[k] = h[k][:n_pts]
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["multiple", "single", "normal"])
def test_device_layer_matches_the_oracle(cuda, method):
    scenes = _scenes()
    batch = _batch(cuda, scenes)
    seed = 123
    with torch.no_grad():
        out = _np(_layer(cuda, REG_AUG_METHOD=method)(batch, seed=seed))
    R = 64
    assert out["sample_status"].tolist() == [0, 0, 0, 0, 2, 0]
    assert out["sampled_pts"].shape == (6 * R, 512, 3) and out["pts_feature"].shape == (6 * R, 512, 5)
    assert out["cls_label"].dtype == np.int64 and out["reg_valid_mask"].dtype == np.int64
    branches, padded = set(), 0
    for b, s in enumerate(scenes):
        o = _layer_oracle(_oracle_scene(batch, b, len(s["rpn_xyz"])), dict(REG_AUG_METHOD=method), "hash", seed=seed, scene_index=b)
        rows = slice(b * R, (b + 1) * R)
        assert out["sample_status"][b] == o["status"]
        branches.add(o["branch"])
        padded += int((o["sel"][:, 0] >= len(s["roi_boxes3d"])).sum())
        np.testing.assert_array_equal(out["cls_label"][rows], o["cls_label"])
        np.testing.assert_array_equal(out["reg_valid_mask"][rows], o["reg_valid_mask"])
        if method != "normal":
            np.testing.assert_array_equal(out["sample_index"][rows], o["sel"])
            keep = slice(None)
        else:      # Box-Muller through logf / sincospif: sources and GT exact, tries where the jittered IoUs agree
            np.testing.assert_array_equal(out["sample_index"][rows][:, :2], o["sel"][:, :2])
            keep = out["sample_index"][rows][:, 2] == o["sel"][:, 2]
            assert keep.mean() > 0.9
        np.testing.assert_allclose(out["gt_iou"][rows][keep], o["iou"][keep], rtol=0, atol=1e-5)
        # pooled features exactly; the depth column is torch's pts_depth / 70 on the device (a reciprocal multiply): one ulp
        pf, of = out["pts_feature"][rows][keep], o["pts_feature"][keep]
        np.testing.assert_allclose(pf[..., 1], of[..., 1], rtol=0, atol=1e-6)
        np.testing.assert_array_equal(np.delete(pf, 1, axis=2), np.delete(of, 1, axis=2))
        bound = lambda a: 2e-5 * max(1.0, np.abs(a).max())
        close = lambda a, e: np.testing.assert_allclose(a, e, rtol=0, atol=bound(e))
        close(out["sampled_pts"][rows][keep], o["sampled_pts"][keep])
        close(out["roi_boxes3d"][rows][keep], o["roi_boxes3d"][keep])
        close(out["gt_of_rois"][rows][keep], o["gt_of_rois_ct"][keep])
    assert branches == {"fg+bg", "bg", "none"} and padded > 0, (branches, padded)


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["multiple", "single", "normal"])
def test_device_jitter_without_augmentation(cuda, method):
    scenes = _scenes()
    batch = _batch(cuda, scenes)
    with torch.no_grad():
        out = _np(_layer(cuda, REG_AUG_METHOD=method, AUG_DATA=False)(batch, seed=8))
    R = 64
    for b, s in enumerate(scenes):
        o = _layer_oracle(_oracle_scene(batch, b, len(s["rpn_xyz"])), dict(REG_AUG_METHOD=method, AUG_DATA=False), "hash", seed=8,
                          scene_index=b)
        rows = slice(b * R, (b + 1) * R)
        if method != "normal":
            np.testing.assert_array_equal(out["roi_boxes3d"][rows], o["rois"])          # jittered boxes, bit for bit
        else:
            same = out["sample_index"][rows][:, 2] == o["sel"][:, 2]
            assert same.mean() > 0.9
            np.testing.assert_allclose(out["roi_boxes3d"][rows][same], o["rois"][same], rtol=0, atol=1e-5)


@pytest.mark.gpu
def test_zero_aug_times_keeps_the_sources(cuda):
    scenes = _scenes()
    batch = _batch(cuda, scenes)
    with torch.no_grad():
        out = _np(_layer(cuda, ROI_FG_AUG_TIMES=0, AUG_DATA=False)(batch, seed=4))
    R = 64
    rois = batch["roi_boxes3d"].cpu().numpy()
    for b, s in enumerate(scenes):
        o = _layer_oracle(_oracle_scene(batch, b, len(s["rpn_xyz"])), dict(ROI_FG_AUG_TIMES=0, AUG_DATA=False), "hash", seed=4,
                          scene_index=b)
        rows = slice(b * R, (b + 1) * R)
        np.testing.assert_array_equal(out["sample_index"][rows], o["sel"])
        assert (out["sample_index"][rows][:, 2] == 0).all()
        np.testing.assert_allclose(out["gt_iou"][rows], o["iou"], rtol=0, atol=1e-5)
        np.testing.assert_array_equal(out["cls_label"][rows], o["cls_label"])
        if o["status"] == 0:
            np.testing.assert_array_equal(out["roi_boxes3d"][rows], rois[b][o["sel"][:, 0]])


@pytest.mark.gpu
def test_status_one_when_no_roi_is_fg_or_bg(cuda):
    batch = _batch(cuda, _scenes()[3:4])          # no RoI overlaps a GT: with both bg thresholds at 0 nothing is fg or bg
    with torch.no_grad():
        out = _np(_layer(cuda, CLS_BG_THRESH=0.0, CLS_BG_THRESH_LO=0.0)(batch, seed=1))
    assert out["sample_status"].tolist() == [1]
    assert (out["cls_label"] == -1).all() and not out["reg_valid_mask"].any() and not out["pts_feature"].any()


@pytest.mark.gpu
def test_device_layer_is_seeded_and_does_not_synchronise(cuda):
    layer = _layer(cuda)
    batch = _batch(cuda, _scenes())
    with torch.no_grad():
        runs = [layer(batch, seed=sd) for sd in (3, 3, 4)]
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            quiet = layer(batch, seed=3)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        counted = [layer(batch), layer(batch)]          # no seed: the call counter
    for k, v in runs[0].items():
        assert torch.equal(v, runs[1][k]) and torch.equal(v, quiet[k]), k
    assert not torch.equal(runs[0]["sample_index"], runs[2]["sample_index"])
    assert not torch.equal(runs[0]["roi_boxes3d"], runs[2]["roi_boxes3d"])
    assert not torch.equal(counted[0]["roi_boxes3d"], counted[1]["roi_boxes3d"]) and layer.calls == 6


@pytest.mark.gpu
def test_draw_statistics(cuda):
    """B = 64 scenes whose RoIs all equal their one GT box, no jitter loop beyond what the fg rows need: every row is a
    copy of the GT box, so the first try's keep, the flip and the rotation angle can be read off the outputs"""
    B, R = 64, 64
    box = np.array([0.0, 1.0, 10.0, 1.5, 1.6, 3.9, 0.0], np.float32)
    rng = np.random.default_rng(0)
    scenes = [dict(rpn_xyz=rng.uniform(-2, 2, (256, 3)).astype(np.float32) + box[:3], rpn_features=np.zeros((256, 2), np.float32),
                   rpn_intensity=np.zeros(256, np.float32), seg_mask=np.zeros(256, np.float32), roi_boxes3d=np.tile(box, (4, 1)),
                   gt_boxes3d=box[None]) for _ in range(B)]
    batch = _batch(cuda, scenes)
    with torch.no_grad():
        plain = _np(_layer(cuda, AUG_DATA=False)(batch, seed=11))
        aug = _np(_layer(cuda)(batch, seed=11))
    n = B * R
    sd = lambda p: 5 * np.sqrt(p * (1 - p) / n)
    assert (plain["sample_status"] == 0).all()
    first_keep = ((plain["sample_index"][:, 2] == 1) & (plain["roi_boxes3d"] == box).all(1)).mean()
    assert abs(first_keep - 0.2) < sd(0.2), first_keep
    # augmented boxes of the rows that kept the GT box: centre (0, 1, 10) -> flip(scale * rot(angle))
    kept = (plain["roi_boxes3d"] == box).all(1)
    x, y, z = (aug["roi_boxes3d"][kept, q].astype(np.float64) for q in range(3))
    scale = y / 1.0
    angle = np.arctan2(-np.abs(x), z)
    flip = x < 0
    assert kept.sum() > 0.15 * n
    assert abs(flip.mean() - 0.5) < 5 * np.sqrt(0.25 / kept.sum()), flip.mean()
    assert (angle < 0).all() and (angle >= -np.pi / 18 - 1e-6).all(), (angle.min(), angle.max())
    assert abs(angle.mean() + np.pi / 36) < 5 * (np.pi / 18) / np.sqrt(12 * kept.sum())
    assert (scale >= 0.95 - 1e-6).all() and (scale < 1.05 + 1e-6).all()


@pytest.mark.gpu
def test_rcnn_trainer_learns_with_device_targets(cuda):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import synth
    from pointrcnn_b200.train.step import RCNNTrainer
    tr = RCNNTrainer(input_channels=1, device=cuda, world=1, lr=0.002, seed=5, target_draw="device")
    with torch.no_grad():
        tr.rpn.rpn_reg_layer[-1].conv.weight.mul_(0.2)
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 321, channels=4)).to(cuda)
    rois = tr.rpn_outputs(pc, None)["roi_boxes3d"]
    gt = torch.zeros((2, 12, 7), device=cuda)
    gt[:, :8] = rois[:, ::40][:, :8]

    def eval_loss():
        tr.model.proposal_target_layer.calls = 0          # the same draws at every evaluation
        with torch.no_grad():
            return float(tr.forward_loss(pc, gt)[0])
    tr.forward_loss(pc, gt)                               # builds the layer
    before = eval_loss()
    for _ in range(10):
        loss, terms = tr.step(pc, gt, grad_norm_clip=1.0)
        assert np.isfinite(float(loss))
    assert eval_loss() < before
    ret = tr.model.forward_train(tr.rpn_outputs(pc, gt), target_draw="device")
    assert ret["sample_status"].tolist() == [0, 0] and int((ret["reg_valid_mask"] > 0).sum()) > 0
    assert ret["rcnn_cls"].shape[0] == 2 * 64 and ret["pts_input"].shape[1:] == (512, 133)


@pytest.mark.gpu
def test_step_jit_on_saved_features(cuda):
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler, read_rois, read_rpn_features, write_rpn_features_batch
    from pointrcnn_b200.train.step import RCNNTrainer
    scenes = [RO.synth_scene(s, k, n_feat=128) for s, k in ((51, "mixed"), (52, "hard"))]
    with tempfile.TemporaryDirectory() as d:
        fd, rd = os.path.join(d, "features"), os.path.join(d, "rois")
        os.makedirs(rd)
        t = lambda key: torch.from_numpy(np.stack([s[key] for s in scenes]))
        write_rpn_features_batch(fd, [0, 1], t("seg_mask"), t("seg_mask"), t("rpn_intensity"), t("rpn_xyz"),
                                 t("rpn_features").permute(0, 2, 1))
        for i, s in enumerate(scenes):
            with open(os.path.join(rd, "%06d.txt" % i), "w") as f:
                f.write("\n".join(MG.label_line("Car", b, 0.5) for b in s["roi_boxes3d"]) + "\n")
        loaded = []
        for i, s in enumerate(scenes):
            xyz, feat, inten, seg = read_rpn_features(fd, i)
            loaded.append(dict(rpn_xyz=xyz, rpn_features=feat, rpn_intensity=inten, seg_mask=seg, roi_boxes3d=read_rois(rd, i),
                               gt_boxes3d=s["gt_boxes3d"]))
    batch = RCNNOfflineSampler(device=cuda).prepare_jit_batch(loaded)
    assert batch["roi_count"].tolist() == [len(s["roi_boxes3d"]) for s in scenes]
    tr = RCNNTrainer(device=cuda, target_draw="device")
    before = [p.detach().clone() for p in tr.params]
    loss, terms = tr.step_jit(batch)
    assert torch.isfinite(loss).item()
    assert any(not torch.equal(a, p.detach()) for a, p in zip(before, tr.params))
    # device-resident scenes pack to the same batch
    on_dev = RCNNOfflineSampler(device=cuda).prepare_jit_batch([{k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda) for k, v in s.items()}
                                                                for s in loaded])
    for k, v in batch.items():
        assert torch.equal(v, on_dev[k]) if k != "pts_depth" else torch.allclose(v, on_dev[k], rtol=1e-6, atol=0), k

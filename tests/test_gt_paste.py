"""GT-paste augmentation in the RPN input pipeline: the oracle and the host candidate draw against the vectors the reference's
own get_rpn_sample produced with GT_AUG_ENABLED (oracle/make_golden_gt_paste.py) on CPU; the device select / paste stages
against the golden vectors and the oracle's geometry on the GPU."""
import os
import types

import numpy as np
import pytest

import inbox_reference as IR
from oracle import gt_paste as GP
from oracle import kitti_io as KO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "gt_paste.npz")
NPOINTS = 4096
DB_SEED, DB_SIZE = 31, 40
SCENES = [(21, 30000, 4), (22, 30000, 16), (23, 2500, 2)]
SEED = 2025


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD, allow_pickle=False)


def _extra_labels(seed):
    rng = np.random.default_rng(seed + 1000)
    return np.array([rng.uniform(-8, 8), 1.7, rng.uniform(12, 30), 1.75, 0.65, 0.9, rng.uniform(-3, 3)], np.float32)


def _scans(scenes=SCENES):
    out = []
    for seed, n, g in scenes:
        lidar, gt, alpha = KO.synth_scan(seed, n, g)
        coll = np.concatenate([gt, _extra_labels(seed)[None]], 0)       # cars + the pedestrian; DontCare is in neither list
        out.append(dict(lidar=lidar, calib=KO.CALIB, img_shape=KO.IMG_SHAPE, gt_boxes3d=gt, gt_alpha=alpha, all_gt_boxes3d=coll,
                        road_plane=GP.road_plane()))
    return out


def _db():
    return GP.synth_gt_database(DB_SEED, DB_SIZE)


def _gt_database(db=None):
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import GTDatabase
    db = _db() if db is None else db
    return GTDatabase.from_reference([dict(e, obj=types.SimpleNamespace(alpha=e["alpha"])) for e in db])


def _labels_in_band(cls, reg, pts, gt, delaunay=False, where=""):
    """every label agrees with the float64 replay of generate_rpn_training_labels outside the band of its decisions"""
    gt = np.asarray(gt, np.float32).reshape(-1, 7)
    IR.check_labels(cls, reg, np.asarray(pts)[:, :3], gt, count=len(gt), delaunay=delaunay, where=where)


def _oracle(s, rng):
    return GP.rpn_sample_with_paste(s["lidar"], KO.CALIB, KO.IMG_SHAPE, s["gt_boxes3d"], s["gt_alpha"], NPOINTS, rng, train=True, gt_db=_db(),
                                    road_plane=s["road_plane"], all_gt_boxes3d=s["all_gt_boxes3d"])


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_reproduces_the_reference_gt_paste(gold):
    np.testing.assert_array_equal(gold["plane"], GP.road_plane())
    np.random.seed(SEED)
    for i, s in enumerate(_scans()):
        o = _oracle(s, np.random)
        np.testing.assert_allclose(o["pts_input"], gold["train%d_pts_input" % i], rtol=0, atol=2e-5)
        np.testing.assert_allclose(o["gt_boxes3d"], gold["train%d_gt_boxes3d" % i], rtol=0, atol=1e-6)
        assert repr(o["aug_method"]) == str(gold["train%d_aug" % i])
        _labels_in_band(o["rpn_cls_label"], o["rpn_reg_label"], o["pts_input"], o["gt_boxes3d"], where="oracle %d" % i)
        _labels_in_band(gold["train%d_rpn_cls_label" % i], gold["train%d_rpn_reg_label" % i], gold["train%d_pts_input" % i], gold["train%d_gt_boxes3d" % i],
                        delaunay=True, where="reference %d" % i)
        assert o["pasted"] >= 5, "every fixture scene must paste several objects"
        if i == 2:
            assert len(o["pts_all"]) < NPOINTS, "scene 2 must have fewer valid points than npoints after the paste"


def test_host_candidate_draw_follows_the_reference_stream(gold):
    from pointrcnn_b200.datasets import kitti_rcnn_dataset as D
    gdb = _gt_database()
    np.random.seed(SEED)
    rejected = 0
    for i, s in enumerate(_scans()):
        before = np.random.get_state()
        cand = D.draw_gt_paste_candidates(gdb, s["road_plane"], rng=np.random)
        after = np.random.get_state()
        # the oracle's paste from the same state consumes exactly the same draws
        r = np.random.RandomState()
        r.set_state(before)
        assert r.rand() < 1.0
        rect = KO.lidar_to_rect(s["lidar"], KO.CALIB)
        uv, depth = KO.rect_to_img(rect, KO.CALIB)
        ok = KO.get_valid_flag(rect, uv, depth, KO.IMG_SHAPE)
        pts, inten, extra, _ = GP.gt_paste_scene(rect[ok][:, :3], s["lidar"][ok, 3], s["all_gt_boxes3d"], _db(), s["road_plane"], r)
        st = r.get_state()
        assert st[2] == after[2] and np.array_equal(st[1], after[1])
        assert cand["applied"] and 11 <= len(cand["entries"]) <= 15
        # the accepted boxes are candidates, bit for bit, in candidate order
        pos = [next(j for j in range(len(cand["boxes"])) if np.array_equal(cand["boxes"][j], b)) for b in extra]
        assert pos == sorted(pos) and len(set(pos)) == len(pos)
        rejected += len(cand["entries"]) - len(extra)
        assert np.all(np.isin(cand["entries"], np.nonzero((gdb.counts >= 5))[0]))
        # the rest of the reference's stream: the npoints draw on the post-paste cloud, then data_augmentation
        D.draw_choice_numpy(pts[:, 2], NPOINTS, np.random)
        angle, scale, flip, method = D.draw_augmentation(rng=np.random)
        assert repr(method) == str(gold["train%d_aug" % i])
    assert rejected > 0, "the fixture must reject candidates"


def test_database_split_follows_the_reference():
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import GTDatabase
    db = _db()
    gdb = _gt_database(db)
    assert list(gdb.easy) == [k for k, e in enumerate(db) if e["points"].shape[0] > 100]
    assert list(gdb.hard) == [k for k, e in enumerate(db) if e["points"].shape[0] <= 100]
    assert len(gdb.easy) and len(gdb.hard) and int(gdb.counts.min()) < 5
    np.testing.assert_array_equal(gdb.boxes, np.stack([e["gt_box3d"] for e in db]))
    np.testing.assert_array_equal(gdb.alpha, np.array([e["alpha"] for e in db], np.float32))
    k = 7
    np.testing.assert_array_equal(gdb.host_points[gdb.offsets[k]:gdb.offsets[k + 1], :3], db[k]["points"])
    np.testing.assert_array_equal(gdb.host_points[gdb.offsets[k]:gdb.offsets[k + 1], 3], db[k]["intensity"])
    easy_only = GTDatabase.from_arrays(gdb.boxes[gdb.easy], [gdb.host_points[gdb.offsets[e]:gdb.offsets[e + 1]] for e in gdb.easy],
                                       gdb.alpha[gdb.easy])
    with pytest.raises(ValueError):
        easy_only.require_lists(0.6)
    easy_only.require_lists(0.0)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_pipeline_with_the_reference_stream_pastes_like_the_reference(cuda, gold):
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import RPNInputPipeline
    pipe = RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="numpy", device=cuda, gt_database=_gt_database())
    np.random.seed(SEED)
    for i, s in enumerate(_scans()):
        out = pipe.prepare_batch([s], rng=np.random)
        np.testing.assert_allclose(out["pts_input"][0].cpu().numpy(), gold["train%d_pts_input" % i], rtol=0, atol=2e-5)
        np.testing.assert_allclose(out["pts_features"][0].cpu().numpy(), gold["train%d_pts_features" % i], rtol=0, atol=1e-7)
        g = gold["train%d_gt_boxes3d" % i]
        n = int(out["gt_count"][0])
        assert n == len(g)
        got = out["gt_boxes3d"][0].cpu().numpy()
        np.testing.assert_allclose(got[:n], g, rtol=0, atol=1e-6)
        assert not got[n:].any()
        assert repr(out["aug_method"][0]) == str(gold["train%d_aug" % i])
        _labels_in_band(out["rpn_cls_label"][0].cpu().numpy(), out["rpn_reg_label"][0].cpu().numpy(), out["pts_input"][0].cpu().numpy(),
                        got[:n], where="device %d" % i)


def _batch8():
    scenes = [(40 + k, 30000 if k % 3 else 6000, 3 + 2 * k) for k in range(8)]
    scans = _scans(scenes)
    for k, s in enumerate(scans):
        s["road_plane"] = GP.road_plane(tilt=0.004 * (k - 3), height=1.6 + 0.02 * k)
    return scans


@pytest.mark.gpu
def test_device_paste_geometry(cuda):
    import torch
    from pointrcnn_b200 import _cabi as C
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import Calibration, PC_AREA_SCOPE, RPNInputPipeline
    gdb = _gt_database()
    scans = _batch8()
    pipe = RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="device", aug_data=False, device=cuda, gt_database=gdb)
    out = pipe.prepare_batch(scans, seed=3)
    gp = out["gt_paste"]
    acc = gp["accepted"].cpu().numpy()
    offs = gp["offsets"].cpu().numpy()
    rect2, pts2, flags2 = gp["rect"].cpu().numpy(), gp["points"].cpu().numpy(), gp["flags"].cpu().numpy()
    stats, gcount = gp["stats"].cpu().numpy(), out["gt_count"].cpu().numpy()
    gt_out = out["gt_boxes3d"].cpu().numpy()
    choice, cls = out["choice"].cpu().numpy(), out["rpn_cls_label"].cpu().numpy()
    counts = out["valid_counts"].cpu().numpy()
    assert acc.sum() >= 8 * 5 and (~acc[:, :11]).sum() > 0, "the batch must accept and reject candidates"
    for b, s in enumerate(scans):
        cand = gp["candidates"][b]
        k = len(cand["entries"])
        a = acc[b, :k]
        assert not acc[b, k:].any()
        boxes = cand["boxes"][a]
        # nothing accepted overlaps: each other or the enlarged collision boxes (the oracle's exact clip)
        big = GP.enlarged_wl(boxes)
        cur = np.concatenate([GP.enlarged_wl(s["all_gt_boxes3d"]), big], 0)
        iou = GP.iou3d(KO.corners3d(big), KO.corners3d(cur))
        for j in range(len(big)):
            iou[j, len(s["all_gt_boxes3d"]) + j] = 0
        assert iou.max() < 1e-6
        # a rejected candidate overlaps a box that was current when it was tested
        for j in np.nonzero(~a)[0]:
            prev = np.concatenate([GP.enlarged_wl(s["all_gt_boxes3d"]), GP.enlarged_wl(cand["boxes"][:j][a[:j]])], 0)
            assert GP.iou3d(KO.corners3d(GP.enlarged_wl(cand["boxes"][j:j + 1])), KO.corners3d(prev)).max() > 1e-9
        # the raw segment: rect as prepared, the valid bit cleared exactly on the valid points inside an accepted box (h + 2)
        n = len(s["lidar"])
        lidar = torch.from_numpy(s["lidar"]).to(cuda)
        calib = torch.from_numpy(Calibration(KO.CALIB).pack(KO.IMG_SHAPE, PC_AREA_SCOPE)[None]).to(cuda)
        o1 = torch.tensor([0, n], dtype=torch.int32, device=cuda)
        rect = torch.empty((n, 3), device=cuda)
        flags = torch.empty(n, dtype=torch.uint8, device=cuda)
        C.check(C.lib().prb_kitti_prepare_points(1, n, C.ptr(o1), C.ptr(lidar), 4, C.ptr(calib), 1, C.ptr(rect), C.ptr(flags), None,
                                                 C.stream()), "prepare")
        rect, flags = rect.cpu().numpy(), flags.cpu().numpy()
        seg = slice(offs[b], offs[b] + n)
        np.testing.assert_array_equal(rect2[seg], rect)
        np.testing.assert_array_equal(pts2[seg][:, 3], s["lidar"][:, 3])
        inside = np.zeros(n, bool)
        for bx in boxes:
            tall = bx.copy()
            tall[3] += np.float32(2)
            inside |= GP.paste_in_box(rect, tall)
        assert (inside & (flags & 1).astype(bool)).sum() > 0
        # against float64 membership: cleared on every valid point certainly inside an accepted box, kept on every valid
        # point certainly outside all of them
        _, cin, cout = IR.classify(rect, boxes, "paste")
        valid, kept = (flags & 1).astype(bool), (flags2[seg] & 1).astype(bool)
        assert not (valid & cin.any(0) & kept).any() and not (valid & cout.all(0) & ~kept).any()
        expect = (flags & 2) | (((flags & 1).astype(bool) & ~inside).astype(np.uint8))
        np.testing.assert_array_equal(flags2[seg], expect)
        # then the accepted entries' points, moved by their move height, in acceptance order
        ents, moves = cand["entries"][a], cand["moves"][a]
        p = offs[b] + n
        for e, mv in zip(ents, moves):
            src = gdb.host_points[gdb.offsets[e]:gdb.offsets[e + 1]]
            got = pts2[p:p + len(src)]
            np.testing.assert_array_equal(got[:, [0, 2, 3]], src[:, [0, 2, 3]])
            np.testing.assert_array_equal(got[:, 1], (src[:, 1].astype(np.float64) - mv).astype(np.float32))
            np.testing.assert_array_equal(rect2[p:p + len(src)], got[:, :3])
            np.testing.assert_array_equal(flags2[p:p + len(src)], 1 | np.where(src[:, 2] < 40.0, 2, 0))
            p += len(src)
        assert p == offs[b + 1] and stats[b, 0] == a.sum() and stats[b, 1] == p - offs[b] - n
        post = flags2[offs[b]:offs[b + 1]]
        assert counts[b, 0] == (post & 1).sum() and counts[b, 1] == ((post & 1) & ~(post >> 1) & 1).sum()
        # label rows: the scene's boxes, then the accepted candidates' (unaugmented here)
        ng = len(s["gt_boxes3d"])
        assert gcount[b] == ng + a.sum()
        np.testing.assert_array_equal(gt_out[b, :ng], s["gt_boxes3d"])
        np.testing.assert_array_equal(gt_out[b, ng:gcount[b]], boxes)
        assert not gt_out[b, gcount[b]:].any()
        # drawn pasted points are foreground
        pasted = choice[b] >= n
        assert pasted.sum() > 50 and (cls[b][pasted] == 1).mean() > 0.99


@pytest.mark.gpu
def test_device_paste_is_seeded(cuda):
    import torch
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import RPNInputPipeline
    pipe = RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="device", device=cuda, gt_database=_gt_database())
    scans = _batch8()
    runs = [pipe.prepare_batch(scans, seed=sd, rng=np.random.RandomState(1)) for sd in (5, 5, 6)]
    for key in ("pts_input", "gt_boxes3d", "gt_count", "rpn_cls_label", "rpn_reg_label", "choice", "valid_counts"):
        assert torch.equal(runs[0][key], runs[1][key]), key
    assert not torch.equal(runs[0]["gt_paste"]["accepted"], runs[2]["gt_paste"]["accepted"]) or \
        not torch.equal(runs[0]["gt_boxes3d"], runs[2]["gt_boxes3d"])
    assert not torch.equal(runs[0]["pts_input"], runs[2]["pts_input"])


@pytest.mark.gpu
def test_no_paste_is_bit_identical_to_no_database(cuda):
    import torch
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import RPNInputPipeline
    scans = _batch8()
    far = _db()
    for e in far:
        e["gt_box3d"] = e["gt_box3d"].copy()
        e["gt_box3d"][2] = 100.0                    # every centre outside the range box
    base = RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="device", device=cuda).prepare_batch(
        scans, seed=9, rng=np.random.RandomState(4))
    for pipe in (RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="device", device=cuda, gt_database=_gt_database(), gt_aug_apply_prob=0.0),
                 RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="device", device=cuda, gt_database=_gt_database(far))):
        out = pipe.prepare_batch(scans, seed=9, rng=np.random.RandomState(4))
        assert "gt_paste" not in out and out["aug_method"] == base["aug_method"]
        for key, v in base.items():
            if torch.is_tensor(v):
                assert torch.equal(out[key], v), key


@pytest.mark.gpu
def test_device_paste_does_not_synchronise(cuda):
    import torch
    from pointrcnn_b200 import _cabi as C
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import RPNInputPipeline
    scans = _batch8()
    base = RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="device", device=cuda)
    pipe = RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="device", device=cuda, gt_database=_gt_database())
    base.prepare_batch(scans, seed=1)
    pipe.prepare_batch(scans, seed=1)
    torch.cuda.synchronize()
    launches = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for p in (base, pipe):
            lc = C.launch_count()
            out = p.prepare_batch(scans, seed=2)
            launches.append(C.launch_count() - lc)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert "gt_paste" in out
    assert launches[1] - launches[0] == 2, launches

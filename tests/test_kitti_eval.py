"""KITTI AP evaluation: the numpy oracle and the host label parser against the golden vectors the reference's own
evaluator produced (oracle/make_golden_kitti_eval.py) on the CPU; the device evaluation against both on the GPU, plus the
in-memory path against the result files it stands for."""
import os
import sys

import numpy as np
import pytest

from oracle import kitti_eval as OK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "kitti_eval.npz")
KEYS = ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD, allow_pickle=False)


def _annos(g, tag):
    out, start = [], 0
    for n in g[tag + "_counts"]:
        a = {}
        for k in KEYS:
            v = g["%s_%s" % (tag, k)]
            a[k] = v[start:start + n] if n else (np.zeros((0,) + v.shape[1:]) if k != "name" else np.array([]))
        out.append(a)
        start += n
    return out


def _ret_dict(g):
    return dict(zip([str(k) for k in g["ret_keys"]], g["ret_values"]))


def _write(dirname, texts):
    os.makedirs(dirname, exist_ok=True)
    for k, t in enumerate(texts):
        with open(os.path.join(dirname, "%06d.txt" % k), "w") as f:
            f.write(str(t))


def _flat(ovs, m):
    return np.concatenate([o[m].reshape(-1) for o in ovs])


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_reproduces_the_reference_evaluation(gold):
    r = OK.evaluate(_annos(gold, "gt"), _annos(gold, "dt"), [int(c) for c in gold["classes"]])
    assert np.array_equal(_flat(r["overlaps"], 0), gold["overlaps0"])
    for m in (1, 2):
        np.testing.assert_allclose(_flat(r["overlaps"], m), gold["overlaps%d" % m], rtol=0, atol=1e-5)
    for idx in np.ndindex(*gold["nthr"].shape):
        t = r["thresholds"][idx]
        assert len(t) == gold["nthr"][idx] and np.array_equal(t, gold["thresholds"][idx][:len(t)]), idx
        assert np.array_equal(r["pr"][idx][:, :3], gold["pr"][idx][:len(t), :3]), idx
    assert 0 < gold["nthr"].max() <= 41
    assert np.array_equal(r["precision"], gold["precision"]) and np.array_equal(r["recall"], gold["recall"])
    np.testing.assert_allclose(r["orientation"], gold["orientation"], rtol=0, atol=1e-9)
    assert r["result_str"] == str(gold["result_str"])
    assert r["ret_dict"] == _ret_dict(gold)


def test_read_label_annos_reproduces_the_reference_parser(gold, tmp_path):
    from pointrcnn_b200.datasets import kitti_eval as KE
    _write(tmp_path / "label", gold["gt_text"])
    _write(tmp_path / "result", gold["dt_text"])
    n = len(gold["gt_text"])
    for tag, annos in (("gt", KE.read_label_annos(tmp_path / "label", list(range(n)))), ("dt", KE.read_label_annos(tmp_path / "result"))):
        want = _annos(gold, tag)
        assert len(annos) == len(want) == n
        for a, w in zip(annos, want):
            assert set(a) == set(KEYS)
            for k in KEYS:
                assert a[k].shape == w[k].shape and np.array_equal(a[k], w[k]), (tag, k)
                if len(w["name"]):
                    assert a[k].dtype.kind == w[k].dtype.kind, (tag, k)


def test_text_rounding_equals_the_printed_value():
    rng = np.random.default_rng(5)
    f = np.concatenate([rng.normal(0, 50, 200000), rng.uniform(-4, 4, 50000),
                        (rng.integers(-10 ** 6, 10 ** 6, 50000) + 0.5) / 1e4]).astype(np.float32)   # exact ties
    q = np.rint(f.astype(np.float64) * 1e4) / 1e4
    assert all(float("%.4f" % v) == w for v, w in zip(f.tolist(), q.tolist()))


# ------------------------------------------------------------------------------------------------ GPU
def _device_vs_oracle(gts, dts, classes):
    """the device evaluation against the oracle fed the device's overlaps (so a pair within fp32 noise of a threshold
    cannot decide differently), and the device overlaps against the oracle's"""
    from pointrcnn_b200.datasets import kitti_eval as KE
    r, ov = KE.evaluate_annos(gts, dts, classes, return_overlaps=True)
    mats, start = [], 0
    for g, d in zip(gts, dts):
        nd, ng = len(d["name"]), len(g["name"])
        mats.append(ov[:, start:start + nd * ng].reshape(3, nd, ng))
        start += nd * ng
    o = OK.evaluate(gts, dts, classes, ovs=mats)
    ref = [OK.overlaps(d, g) for g, d in zip(gts, dts)]
    assert np.array_equal(_flat(mats, 0), _flat(ref, 0))
    # random splits keep small and nearly parallel pairs, where any fp32 clipper is ~1e-4 off the exact area (the golden
    # split, which avoids them, pins the device overlaps to 1e-5)
    for m in (1, 2):
        np.testing.assert_allclose(_flat(mats, m), _flat(ref, m), rtol=0, atol=5e-4)
    assert np.array_equal(r.precision, o["precision"]) and np.array_equal(r.recall, o["recall"])
    np.testing.assert_allclose(r.orientation, o["orientation"], rtol=0, atol=1e-9)
    assert r.result_str == o["result_str"]
    return r


@pytest.mark.gpu
def test_device_overlaps_match_the_reference(cuda, gold):
    from pointrcnn_b200.datasets import kitti_eval as KE
    _, ov = KE.evaluate_annos(_annos(gold, "gt"), _annos(gold, "dt"), [0, 1, 2], return_overlaps=True)
    assert np.array_equal(ov[0], gold["overlaps0"])
    for m in (1, 2):
        np.testing.assert_allclose(ov[m], gold["overlaps%d" % m], rtol=0, atol=1e-5)


@pytest.mark.gpu
def test_device_official_result_matches_the_reference(cuda, gold):
    from pointrcnn_b200.datasets import kitti_eval as KE
    gts, dts = _annos(gold, "gt"), _annos(gold, "dt")
    r = KE.evaluate_annos(gts, dts, [0, 1, 2])
    assert r.result_str == str(gold["result_str"]) and r.ret_dict == _ret_dict(gold)
    assert np.array_equal(r.num_thresholds, gold["nthr"])
    assert np.array_equal(r.thresholds, gold["thresholds"])
    assert np.array_equal(r.counts[..., :3], gold["pr"][..., :3])
    assert np.array_equal(r.precision, gold["precision"]) and np.array_equal(r.recall, gold["recall"])
    np.testing.assert_allclose(r.orientation, gold["orientation"], rtol=0, atol=1e-9)
    assert KE.get_official_eval_result(gts, dts, [0, 1, 2]) == (r.result_str, r.ret_dict)
    # one class by name, filed under the Car_* keys as the reference does
    s, d = KE.get_official_eval_result(gts, dts, "Pedestrian")
    assert s.startswith("Pedestrian AP@0.50, 0.50, 0.50:\n") and d["Car_3d_moderate"] == r.mAP_R11[2, 1, 1, 0]
    assert r.mAP_R40.shape == (3, 3, 3, 2) and np.all(r.mAP_R40 >= 0)


def _scenes(seed, n_img, m):
    """GT as result-format label files written from 3D boxes (so image boxes and alpha are consistent), and (B, M, 7)
    detections around them"""
    import torch
    from oracle import kitti_io as KO
    rng = np.random.default_rng(seed)
    g = 12
    gt = np.zeros((n_img, g, 7), np.float32)
    gt[..., 0] = rng.uniform(-15, 15, (n_img, g))
    gt[..., 1] = rng.uniform(1.5, 1.8, (n_img, g))
    gt[..., 2] = rng.uniform(6, 50, (n_img, g))
    gt[..., 3:6] = np.array([1.5, 1.6, 3.9], np.float32) * rng.uniform(0.3, 1.1, (n_img, g, 1))
    gt[..., 6] = rng.uniform(-np.pi, np.pi, (n_img, g))
    src = rng.integers(0, g, (n_img, m))
    det = gt[np.arange(n_img)[:, None], src] + rng.normal(0, 0.15, (n_img, m, 7)).astype(np.float32) * [1, 0.2, 1, 0.1, 0.1, 0.1, 1]
    free = rng.random((n_img, m)) < 0.3
    det[free, 0] += rng.uniform(-10, 10, int(free.sum()))
    scores = rng.normal(0, 2, (n_img, m)).astype(np.float32)
    select = rng.random((n_img, m)) < 0.8
    select[1] = False                                       # an image without detections
    calib = [KO.CALIB] * n_img
    shapes = [KO.IMG_SHAPE] * n_img
    names = rng.choice(["Car", "Car", "Car", "Van", "Pedestrian", "DontCare"], (n_img, g))
    return gt, names, det.astype(np.float32), scores, select, calib, shapes, torch


@pytest.mark.gpu
def test_in_memory_evaluation_equals_the_result_files(cuda, tmp_path):
    from pointrcnn_b200.datasets import kitti_eval as KE
    from pointrcnn_b200.datasets import kitti_output as KW
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import Calibration
    n_img, m, B = 32, 24, 8
    gt, names, det, scores, select, calib, shapes, torch = _scenes(3, n_img, m)
    # labels: the writer's text for the GT boxes, renamed, without the score column (truncation / occlusion -1: every band)
    texts = KW.write_kitti_batch(range(n_img), calib, shapes, torch.from_numpy(gt).cuda(), torch.ones(gt.shape[:2], device="cuda"),
                                 torch.ones(gt.shape[:2], dtype=torch.bool, device="cuda"))
    labels = []
    for k, t in enumerate(texts):
        rows = [line.split(" ") for line in t.splitlines()]
        labels.append("".join(" ".join([names[k, i]] + r[1:15]) + "\n" for i, r in enumerate(rows)))
    _write(tmp_path / "label", labels)
    with open(tmp_path / "split.txt", "w") as f:
        f.write("".join("%d\n" % k for k in range(n_img)))
    gt_annos = KE.read_label_annos(tmp_path / "label", list(range(n_img)))
    assert sum(len(a["name"]) for a in gt_annos) > 100

    ev = KE.KittiEvaluator(gt_annos, [0, 1], "cuda")
    os.makedirs(tmp_path / "result")
    P2 = np.stack([Calibration(c).P2 for c in calib]).astype(np.float32)
    hw = np.array([s[:2] for s in shapes], np.float32)
    for b0 in range(0, n_img, B):
        sl = slice(b0, b0 + B)
        bx, sc, se = torch.from_numpy(det[sl]).cuda(), torch.from_numpy(scores[sl]).cuda(), torch.from_numpy(select[sl]).cuda()
        ev.add_batch(list(range(b0, b0 + B)), bx, sc, se, P2[sl], hw[sl])
        KW.write_kitti_batch(range(b0, b0 + B), calib[sl], shapes[sl], bx, sc, se, str(tmp_path / "result"))
    mem = ev.result()
    files = KE.evaluate_annos(gt_annos, KE.read_label_annos(tmp_path / "result"), [0, 1])
    assert files.precision[0].max() > 0.3, "the fixture must produce matches"
    for k in ("precision", "recall", "orientation", "counts", "thresholds"):
        assert np.array_equal(getattr(mem, k), getattr(files, k)), k
    assert mem.result_str == files.result_str
    assert KE.evaluate(tmp_path / "label", tmp_path / "result", tmp_path / "split.txt", [0, 1]) == (mem.result_str, mem.ret_dict)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["few_images", "class_without_valid_gt", "detections_under_min_height", "large"])
def test_device_agrees_with_the_oracle_where_the_reference_cannot_run(cuda, case):
    if case == "large":
        gts, dts = OK.synth_split(11, 500, 40, 100)
    else:
        gts, dts = OK.synth_split(12, 20, 10, 12)
    if case == "class_without_valid_gt":
        for g in gts:
            g["name"] = np.array(["Misc" if n == "Cyclist" else n for n in g["name"]])
    if case == "detections_under_min_height":
        for d in dts:
            d["bbox"][:, 3] = d["bbox"][:, 1] + 24.0
    r = _device_vs_oracle(gts, dts, [0, 1, 2])
    if case == "class_without_valid_gt":
        assert np.all(r.precision[:, 2] == 0) and np.all(r.num_thresholds[:, 2] == 0)
    if case == "detections_under_min_height":
        assert np.all(r.precision == 0) and r.counts[..., 0].sum() == 0
    else:
        assert r.precision.max() > 0


@pytest.mark.gpu
def test_add_batch_does_not_synchronise_and_result_is_reproducible(cuda):
    import torch
    from pointrcnn_b200.datasets import kitti_eval as KE
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import Calibration
    n_img, m = 16, 40
    gts, _ = OK.synth_split(4, n_img, 10, 0)
    gt, names, det, scores, select, calib, shapes, torch = _scenes(5, n_img, m)
    ev = KE.KittiEvaluator(gts, [0, 1, 2], "cuda")
    P2 = torch.from_numpy(np.stack([Calibration(c).P2 for c in calib]).astype(np.float32)).cuda()
    hw = torch.tensor([s[:2] for s in shapes], dtype=torch.float32, device="cuda")
    bx, sc, se = torch.from_numpy(det).cuda(), torch.from_numpy(scores).cuda(), torch.from_numpy(select).cuda()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for b0 in range(0, n_img, 4):
            ev.add_batch(list(range(b0, b0 + 4)), bx[b0:b0 + 4], sc[b0:b0 + 4], se[b0:b0 + 4], P2[b0:b0 + 4], hw[b0:b0 + 4])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    a, b = ev.result(), ev.result()
    for k in ("precision", "recall", "orientation", "counts", "thresholds"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    assert a.result_str == b.result_str


@pytest.mark.gpu
def test_dropin_evaluate_reads_a_directory(cuda, gold, tmp_path):
    assert not any(p.rstrip("/").endswith("reference") for p in sys.path)
    saved = {k: v for k, v in sys.modules.items() if k == "tools" or k.startswith("tools.")}
    try:
        from pointrcnn_b200 import dropin
        dropin.activate()
        from tools.kitti_object_eval_python.evaluate import evaluate
        from tools.kitti_object_eval_python.eval import get_official_eval_result
        _write(tmp_path / "label", gold["gt_text"])
        _write(tmp_path / "result", gold["dt_text"])
        with open(tmp_path / "val.txt", "w") as f:
            f.write("".join("%d\n" % k for k in range(len(gold["gt_text"]))))
        s, d = evaluate(str(tmp_path / "label"), str(tmp_path / "result"), str(tmp_path / "val.txt"), current_class=[0, 1, 2])
        assert s == str(gold["result_str"]) and d == _ret_dict(gold)
        assert get_official_eval_result(_annos(gold, "gt"), _annos(gold, "dt"), [0, 1, 2])[0] == s
    finally:
        for k in [k for k in sys.modules if k == "tools" or k.startswith("tools.")]:
            del sys.modules[k]
        sys.modules.update(saved)

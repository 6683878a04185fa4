"""COCO-style KITTI AP (ten overlap sets per class) and the score filter: the numpy oracle and the host filter against the
golden vectors the reference's own evaluator produced (oracle/make_golden_kitti_eval_coco.py) on the CPU; on the GPU,
the device evaluation against them, the K-set entry against the official one, the device filter against the host one,
the in-memory path against the result files, the drop-in route and the refusals."""
import os
import sys

import numpy as np
import pytest

from oracle import kitti_eval as OK
from oracle import kitti_eval_coco as OKC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "kitti_eval_coco.npz")
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


def _write(dirname, texts):
    os.makedirs(dirname, exist_ok=True)
    for k, t in enumerate(texts):
        with open(os.path.join(dirname, "%06d.txt" % k), "w") as f:
            f.write(str(t))


def _split_file(path, n):
    with open(path, "w") as f:
        f.write("".join("%d\n" % k for k in range(n)))


# ------------------------------------------------------------------------------------------------ CPU
def test_coco_overlap_sets_are_numpys_linspace():
    from pointrcnn_b200.datasets import kitti_eval as KE
    mo = KE.coco_min_overlaps([0, 1, 2])
    assert mo.shape == (10, 3, 3) and np.array_equal(mo, OKC.coco_min_overlaps([0, 1, 2]))
    assert mo[8, 0, 0] == 0.8999999999999999 and mo[8, 2, 1] == 0.6499999999999999 and mo[9, 1, 0] == 0.95
    for j, (a, b) in enumerate(((0.5, 0.95), (0.25, 0.7), (0.25, 0.7))):
        for m in range(3):
            assert np.array_equal(mo[:, m, j], np.linspace(a, b, 10))
    assert np.array_equal(KE.official_min_overlaps([1, 0]), KE.MIN_OVERLAPS[:, :, [1, 0]])


def test_oracle_reproduces_the_reference_coco_evaluation(gold):
    gts, dts = _annos(gold, "gt"), _annos(gold, "dt")
    r = OKC.coco_evaluate(gts, dts, [int(c) for c in gold["classes"]])
    for idx in np.ndindex(*gold["nthr"].shape):
        t = r["thresholds"][idx]
        assert len(t) == gold["nthr"][idx] and np.array_equal(t, gold["thresholds"][idx][:len(t)]), idx
        assert np.array_equal(r["pr"][idx][:, :3], gold["pr"][idx][:len(t), :3]), idx
    assert gold["nthr"].shape == (3, 3, 3, 10) and 0 < gold["nthr"].max() <= 41
    assert np.array_equal(r["precision"], gold["precision"]) and np.array_equal(r["recall"], gold["recall"])
    np.testing.assert_allclose(r["orientation"], gold["orientation"], rtol=0, atol=1e-9)
    assert r["coco_str"] == str(gold["coco_str"])
    assert OKC.coco_evaluate(gts, dts, "Pedestrian")["coco_str"] == str(gold["coco_str_pedestrian"])
    assert OKC.coco_evaluate(gts, _annos(gold, "dtf"), [0, 1, 2])["coco_str"] == str(gold["coco_str_score_thresh"])


def test_host_filter_reproduces_the_reference_filter(gold):
    from pointrcnn_b200.datasets import kitti_eval as KE
    got, want = KE.filter_annos_low_score(_annos(gold, "dt"), float(gold["score_thresh"])), _annos(gold, "dtf")
    assert len(got) == len(want)
    assert 0 < sum(len(a["name"]) for a in want) < sum(gold["dt_counts"])
    for a, w in zip(got, want):
        assert set(a) == set(KEYS)
        for k in KEYS:
            assert a[k].shape == w[k].shape and np.array_equal(a[k], w[k]), k
    # a score equal to the threshold stays
    a = dict(name=np.array(["Car", "Car", "Car"]), score=np.array([0.3, 0.5, 0.7]), alpha=np.array([1.0, 2.0, 3.0]))
    f = KE.filter_annos_low_score([a], 0.5)[0]
    assert list(f["score"]) == [0.5, 0.7] and list(f["alpha"]) == [2.0, 3.0]


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_device_coco_result_matches_the_reference(cuda, gold):
    from pointrcnn_b200.datasets import kitti_eval as KE
    gts, dts = _annos(gold, "gt"), _annos(gold, "dt")
    r = KE.evaluate_annos(gts, dts, [0, 1, 2], coco=True)
    assert r.min_overlaps.shape == (10, 3, 3) and r.ret_dict is None
    assert np.array_equal(r.num_thresholds, gold["nthr"])
    assert np.array_equal(r.thresholds, gold["thresholds"])
    assert np.array_equal(r.counts[..., :3], gold["pr"][..., :3])
    assert np.array_equal(r.precision, gold["precision"]) and np.array_equal(r.recall, gold["recall"])
    np.testing.assert_allclose(r.orientation, gold["orientation"], rtol=0, atol=1e-9)
    assert r.result_str == str(gold["coco_str"])
    assert KE.get_coco_eval_result(gts, dts, [0, 1, 2]) == str(gold["coco_str"])
    assert KE.get_coco_eval_result(gts, dts, "Pedestrian") == str(gold["coco_str_pedestrian"])
    t = float(gold["score_thresh"])
    assert KE.evaluate_annos(gts, dts, [0, 1, 2], coco=True, score_thresh=t).result_str == str(gold["coco_str_score_thresh"])
    assert KE.get_coco_eval_result(gts, _annos(gold, "dtf"), [0, 1, 2]) == str(gold["coco_str_score_thresh"])


def _raw(entry, gts, dts, classes, mo=None):
    """one call of prb_kitti_eval or prb_kitti_eval_sets on packed annotations -> (out, overlaps) host arrays"""
    import ctypes
    import torch
    from pointrcnn_b200 import _cabi as C
    from pointrcnn_b200.datasets import kitti_eval as KE
    lib = C.lib()
    gt, gc = KE.pack_annos(gts)
    dt, dc = KE.pack_annos(dts)
    n_img, nc = len(gts), len(classes)
    pair_off = KE._offsets(gc * dc)
    n_pairs = int(pair_off[-1])
    up = lambda a, t=torch.float64: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", t)
    cls = np.ascontiguousarray(classes, np.int32)
    mo = KE.official_min_overlaps(classes) if mo is None else np.ascontiguousarray(mo, np.float64)
    ns = mo.shape[0]
    g, d, go, do, dcount, po = up(gt), up(dt), up(KE._offsets(gc), torch.int32), up(KE._offsets(dc), torch.int32), up(dc, torch.int32), up(pair_off, torch.int64)
    ov = torch.full((max(3 * n_pairs, 1),), np.nan, dtype=torch.float64, device="cuda")
    out = torch.full((9 * ns * nc * 41 * 8 + 1 + 9 * ns * nc,), np.nan, dtype=torch.float64, device="cuda")
    P = ctypes.c_void_p
    common = (C.ptr(g), C.ptr(go), int(gc.sum()), C.ptr(d), C.ptr(do), C.ptr(dcount), int(dc.sum()), int(dc.max()), C.ptr(po),
              ctypes.c_longlong(n_pairs), C.ptr(ov), C.ptr(out))
    if entry == "prb_kitti_eval":
        nbytes = lib.prb_kitti_eval_workspace_bytes(n_img, int(gc.sum()), int(dc.sum()), nc)
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        rc = lib.prb_kitti_eval(n_img, nc, P(cls.ctypes.data), P(mo.ctypes.data), *common, C.ptr(ws), ctypes.c_size_t(nbytes), C.stream())
    else:
        nbytes = lib.prb_kitti_eval_sets_workspace_bytes(n_img, int(gc.sum()), int(dc.sum()), nc, ns)
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        rc = lib.prb_kitti_eval_sets(n_img, nc, P(cls.ctypes.data), ns, P(mo.ctypes.data), ctypes.c_double(-1.0), *common, C.ptr(ws),
                                     ctypes.c_size_t(nbytes), C.stream())
    C.check(rc, entry)
    return out.cpu().numpy(), ov.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("split", ["golden", "synth"])
def test_sets_entry_with_the_official_sets_equals_the_official_entry(cuda, gold, split):
    if split == "golden":
        gts, dts = _annos(gold, "gt"), _annos(gold, "dt")
    else:
        gts, dts = OK.synth_split(21, 80, 12, 16)
    a_out, a_ov = _raw("prb_kitti_eval", gts, dts, [0, 1, 2])
    b_out, b_ov = _raw("prb_kitti_eval_sets", gts, dts, [0, 1, 2])
    assert a_out.tobytes() == b_out.tobytes() and a_ov.tobytes() == b_ov.tobytes()
    assert not np.isnan(a_out).any() and a_out[:18 * 3 * 41 * 8].reshape(-1, 8)[:, 5].max() > 0


def _same(a, b):
    for k in ("precision", "recall", "orientation", "counts", "thresholds", "num_thresholds", "mAP_R11"):
        assert getattr(a, k).tobytes() == getattr(b, k).tobytes(), k
    assert a.compute_aos == b.compute_aos and a.result_str == b.result_str


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["mid", "first_image_removed", "all_removed", "tie"])
def test_device_score_filter_equals_evaluating_the_host_filtered_annotations(cuda, case):
    from pointrcnn_b200.datasets import kitti_eval as KE
    gts, dts = OK.synth_split(31, 60, 12, 16)
    first = next(k for k, d in enumerate(dts) if len(d["name"]))
    t = 0.5
    if case == "first_image_removed":
        # the first image with detections loses them all, and its first alpha (-10) would have switched AOS off
        dts[first]["score"][:] = 0.05
        dts[first]["alpha"][0] = -10.0
        t = 0.1
    if case == "all_removed":
        t = 2.0
    if case == "tie":
        for d in dts[::3]:
            d["score"][::2] = 0.5
    kept = KE.filter_annos_low_score(dts, t)
    if case == "tie":
        assert sum(int((d["score"] == t).sum()) for d in kept) > 10
    for coco in (False, True):
        dev = KE.evaluate_annos(gts, dts, [0, 1, 2], coco=coco, score_thresh=t)
        host = KE.evaluate_annos(gts, kept, [0, 1, 2], coco=coco)
        _same(dev, host)
        assert dev.min_overlaps.shape[0] == (10 if coco else 2)
    unfiltered = KE.evaluate_annos(gts, dts, [0, 1, 2])
    if case == "first_image_removed":
        assert not unfiltered.compute_aos and dev.compute_aos
    if case == "all_removed":
        assert np.all(dev.precision == 0) and dev.counts[..., 0].sum() == 0 and not dev.compute_aos
    else:
        assert dev.precision.max() > 0
    # a threshold <= 0 filters nothing, as in the reference's evaluate
    _same(KE.evaluate_annos(gts, dts, [0, 1, 2], score_thresh=0.0), unfiltered)


@pytest.mark.gpu
def test_in_memory_coco_evaluation_equals_the_result_files(cuda, tmp_path):
    import torch
    from test_kitti_eval import _scenes
    from pointrcnn_b200.datasets import kitti_eval as KE
    from pointrcnn_b200.datasets import kitti_output as KW
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import Calibration
    n_img, m, B = 32, 24, 8
    gt, names, det, scores, select, calib, shapes, torch = _scenes(13, n_img, m)
    texts = KW.write_kitti_batch(range(n_img), calib, shapes, torch.from_numpy(gt).cuda(), torch.ones(gt.shape[:2], device="cuda"),
                                 torch.ones(gt.shape[:2], dtype=torch.bool, device="cuda"))
    labels = []
    for k, t in enumerate(texts):
        rows = [line.split(" ") for line in t.splitlines()]
        labels.append("".join(" ".join([names[k, i]] + r[1:15]) + "\n" for i, r in enumerate(rows)))
    _write(tmp_path / "label", labels)
    _split_file(tmp_path / "split.txt", n_img)
    gt_annos = KE.read_label_annos(tmp_path / "label", list(range(n_img)))

    ev = KE.KittiEvaluator(gt_annos, [0, 1], "cuda")
    os.makedirs(tmp_path / "result")
    P2 = np.stack([Calibration(c).P2 for c in calib]).astype(np.float32)
    hw = np.array([s[:2] for s in shapes], np.float32)
    batches = []
    for b0 in range(0, n_img, B):
        sl = slice(b0, b0 + B)
        batches.append((list(range(b0, b0 + B)), torch.from_numpy(det[sl]).cuda(), torch.from_numpy(scores[sl]).cuda(),
                        torch.from_numpy(select[sl]).cuda(), torch.from_numpy(P2[sl]).cuda(), torch.from_numpy(hw[sl]).cuda()))
        KW.write_kitti_batch(range(b0, b0 + B), calib[sl], shapes[sl], *batches[-1][1:4], str(tmp_path / "result"))
    t = 0.5
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for b in batches:
            ev.add_batch(*b)
        ev._evaluate_on_device(coco=True, score_thresh=t)            # the filter and the statistics, nothing copied back
    finally:
        torch.cuda.set_sync_debug_mode(0)
    mem = ev.result(coco=True, score_thresh=t)
    dt_files = KE.read_label_annos(tmp_path / "result")
    assert 0 < sum(len(d["name"]) for d in KE.filter_annos_low_score(dt_files, t)) < sum(len(d["name"]) for d in dt_files)
    files = KE.evaluate_annos(gt_annos, dt_files, [0, 1], coco=True, score_thresh=t)
    assert files.precision[0].max() > 0.3, "the fixture must produce matches"
    for k in ("precision", "recall", "orientation", "counts", "thresholds"):
        assert np.array_equal(getattr(mem, k), getattr(files, k)), k
    s = KE.evaluate(tmp_path / "label", tmp_path / "result", tmp_path / "split.txt", [0, 1], coco=True, score_thresh=t)
    assert isinstance(s, str) and mem.result_str == s and s.startswith("Car coco AP@0.50:0.05:0.95:\n")
    # the official table through the same arguments keeps its (result_str, ret_dict)
    off = ev.result(score_thresh=t)
    assert KE.evaluate(tmp_path / "label", tmp_path / "result", tmp_path / "split.txt", [0, 1], score_thresh=t) == (off.result_str, off.ret_dict)


@pytest.mark.gpu
def test_dropin_reference_coco_import_and_call_reach_the_device(cuda, gold, tmp_path):
    from pointrcnn_b200 import _cabi as C
    assert not any(p.rstrip("/").endswith("reference") for p in sys.path)
    saved = {k: v for k, v in sys.modules.items() if k == "tools" or k.startswith("tools.")}
    try:
        from pointrcnn_b200 import dropin
        from pointrcnn_b200.datasets import kitti_eval as KE
        dropin.activate()
        # evaluate.py:5's import line
        from tools.kitti_object_eval_python.eval import get_official_eval_result, get_coco_eval_result  # noqa: F401
        from tools.kitti_object_eval_python.evaluate import evaluate
        assert get_coco_eval_result is KE.get_coco_eval_result
        _write(tmp_path / "label", gold["gt_text"])
        _write(tmp_path / "result", gold["dt_text"])
        _split_file(tmp_path / "val.txt", len(gold["gt_text"]))
        l0 = C.launch_count()
        s = evaluate(str(tmp_path / "label"), str(tmp_path / "result"), str(tmp_path / "val.txt"), current_class=[0, 1, 2], coco=True,
                     score_thresh=0.3)
        assert C.launch_count() - l0 >= 7
        want = KE.evaluate_annos(_annos(gold, "gt"), KE.filter_annos_low_score(_annos(gold, "dt"), 0.3), [0, 1, 2], coco=True)
        assert s == want.result_str and s.startswith("Car coco AP@0.50:0.05:0.95:\n")
        assert get_coco_eval_result(_annos(gold, "gt"), _annos(gold, "dt"), [0, 1, 2]) == str(gold["coco_str"])
    finally:
        for k in [k for k in sys.modules if k == "tools" or k.startswith("tools.")]:
            del sys.modules[k]
        sys.modules.update(saved)


@pytest.mark.gpu
@pytest.mark.parametrize("sets", ["none", "eleven", "overlap_one"])
def test_bad_overlap_sets_are_refused(cuda, sets):
    from pointrcnn_b200.datasets import kitti_eval as KE
    gts, dts = OK.synth_split(41, 4, 6, 6)
    mo = {"none": np.full((0, 3, 1), 0.5), "eleven": np.full((11, 3, 1), 0.5),
          "overlap_one": np.array([[[0.7]] * 3, [[0.5], [1.0], [0.5]]])}[sets]
    with pytest.raises(RuntimeError, match="overlap"):
        KE.evaluate_annos(gts, dts, [0], min_overlaps=mo)

"""The RCNN sampling decisions of oracle/rcnn_offline.py::sample_scene on crafted IoU matrices (tests/rcnn_sample_reference.py)
against what the reference's own loader and target layer decided on the same matrices (oracle/make_golden_rcnn_sample_edges.py):
max_overlaps and the GT assignment (ties, NaN, +-inf, -0.0), the fg / easy / hard lists, the branch, the fg and bg row
counts and the sampled sources.  The draws are the reference's; the candidate checks do not depend on them, and one
replay of the same streams checks the sampled sources in order as well."""
import os

import numpy as np
import pytest
import torch

import rcnn_sample_reference as RS
from oracle import rcnn_offline as RO
from rcnn_sample_reference import bits, run_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "rcnn_sample_edges.npz")
RECIPES = ("loader", "layer")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD, allow_pickle=False)


def test_cases_hit_their_edges():
    by = {c["name"]: c for c in RS.cases()}
    o = {(n, r): run_oracle(c, r) for n, c in by.items() for r in RECIPES}
    branches = {r: {o[n, r]["branch"] for n in by} for r in RECIPES}
    assert branches["layer"] == {"fg+bg", "fg", "bg", "none"} and {"fg+bg", "fg", "bg", "none"} <= branches["loader"] | {"fg"}
    statuses = {o[n, r]["status"] for n in by for r in RECIPES}
    assert statuses == {0, 1, 2}
    # every threshold value (and its neighbours) is some row's max IoU
    mo = o["thresholds", "layer"]["candidates"]["max_overlaps"]
    for t in RS.THRESHOLDS:
        assert {RS.dn(t), t, RS.up(t)} <= set(mo.tolist())
    # hard only / easy only / both in the bg rows
    for name, hard, easy in (("hard_only", True, False), ("easy_only", False, True), ("no_fg_both", True, True)):
        c = o[name, "layer"]["candidates"]
        assert (c["hard"].size > 0, c["easy"].size > 0) == (hard, easy), name
    # the loader's GT-max RoIs: row 0 four times on the column ties
    assert o["column_ties", "loader"]["candidates"]["fg"].tolist() == [0, 0, 0, 0]
    # fg counts around the quota of 8, the layer's and the loader's (one GT-max RoI more)
    assert [o["fg_%d" % k, "layer"]["candidates"]["fg"].size for k in (6, 7, 8, 9)] == [6, 7, 8, 9]
    assert [o["fg_%d" % k, "loader"]["candidates"]["fg"].size for k in (6, 7, 8, 9)] == [7, 8, 9, 10]
    # HARD_BG_RATIO products just under an integer: 100 bg rows of the layer
    assert int(100 * 0.29) == 28 and int(100 * 0.57) == 56
    for ratio, hard_n in ((0.0, 0), (1.0, 100), (0.29, 28), (0.57, 56)):
        s = o["ratio_%g" % ratio, "layer"]["sel"][28:, 0]
        hard = set(o["ratio_%g" % ratio, "layer"]["candidates"]["hard"].tolist())
        assert [int(v) in hard for v in s] == [True] * hard_n + [False] * (100 - hard_n), ratio
    # the layer's trimming keeps a zero GT row in the middle and drops the trailing ones
    assert o["zero_gt_rows", "layer"]["candidates"]["n_gt"] == 3 and o["zero_gt_all", "layer"]["status"] == 2


@pytest.mark.parametrize("recipe", RECIPES)
def test_oracle_decides_as_the_reference(gold, recipe):
    """per case: the reference's stop (raise / pdb) against the oracle's status and branch, max_overlaps (bit for bit in
    the layer, whose reference returns it), the GT assignment, the three candidate lists, the fg / bg row counts, and
    the sampled sources drawn from the right lists"""
    for case in RS.cases():
        key = "%s.%s" % (case["name"], recipe)
        g = lambda k: gold["%s.%s" % (key, k)]
        o = run_oracle(case, recipe)
        msg = key
        if bool(g("raises")):
            # the reference stops where the oracle reports status 2 (an empty RoI or GT list) or takes the fg-only branch
            # (the loader's line 923 raises; the oracle implements what it means)
            assert o["status"] == 2 or (recipe == "loader" and o["branch"] == "fg"), msg
            if o["status"] == 2:
                continue
        elif bool(g("pdb")):
            # no fg and no bg: status 1; with no RoI at all (the layer reduces an empty matrix) the device's status 2
            assert o["status"] == 1 or (o["status"] == 2 and case["iou"].shape[0] == 0), msg
            if o["status"] == 2:
                continue
        else:
            assert o["status"] == 0, msg
        c = o["candidates"]
        mo = g("branch.max_overlaps")
        np.testing.assert_array_equal(c["max_overlaps"], mo, err_msg=msg)
        if recipe == "layer":
            np.testing.assert_array_equal(bits(c["max_overlaps"]), bits(mo), err_msg=msg)
            assert c["n_gt"] == len(g("branch.cur_gt")), msg
        np.testing.assert_array_equal(c["gt_assignment"], g("branch.gt_assignment"), err_msg=msg)
        np.testing.assert_array_equal(c["fg"], g("branch.fg_inds"), err_msg=msg)
        np.testing.assert_array_equal(c["easy"], g("branch.easy_bg_inds"), err_msg=msg)
        np.testing.assert_array_equal(c["hard"], g("branch.hard_bg_inds"), err_msg=msg)
        if o["status"] != 0 or bool(g("raises")):
            continue
        fg_n, bg_n = int(g("jitter.fg_rois_per_this_image")), int(g("jitter.bg_rois_per_this_image"))
        assert fg_n + bg_n == case["R"], msg
        src = o["sel"][:, 0]
        assert set(src[:fg_n].tolist()) <= set(c["fg"].tolist()) and set(g("jitter.fg_inds").tolist()) <= set(c["fg"].tolist()), msg
        hard, easy = set(c["hard"].tolist()), set(c["easy"].tolist())
        ref_bg = g("jitter.bg_inds") if bg_n else np.zeros(0, np.int64)
        # the hard rows come first in both; their count is the reference's
        n_hard_ref = sum(int(v) in hard for v in ref_bg)
        assert all(int(v) in hard for v in ref_bg[:n_hard_ref]) and all(int(v) in easy for v in ref_bg[n_hard_ref:]), msg
        assert all(int(v) in hard for v in src[fg_n:fg_n + n_hard_ref]) and all(int(v) in easy for v in src[fg_n + n_hard_ref:]), msg
        np.testing.assert_array_equal(o["sel"][:, 1], c["gt_assignment"][src], err_msg=msg)


def test_oracle_replays_the_reference_draws(gold):
    """the golden maker's order of cases and recipes on the same seeded streams: the oracle's numpy / torch draws give the
    reference's sampled sources in order, and the layer's reported IoUs (the source's max_overlaps) bit for bit"""
    from oracle import make_golden_rcnn_sample_edges as MG
    np.random.seed(MG.SEED)
    torch.manual_seed(MG.SEED)
    compared = 0
    for case in RS.cases():
        for recipe, draw in (("loader", "numpy"), ("layer", "ref")):
            key = "%s.%s" % (case["name"], recipe)
            o = run_oracle(case, recipe, draw=draw)
            if bool(gold[key + ".raises"]) or bool(gold[key + ".pdb"]):
                continue
            fg_n = int(gold[key + ".jitter.fg_rois_per_this_image"])
            ref = [gold[key + ".jitter.fg_inds"]] if fg_n else []
            if fg_n < case["R"]:
                ref.append(gold[key + ".jitter.bg_inds"])
            np.testing.assert_array_equal(o["sel"][:, 0], np.concatenate(ref), err_msg=key)
            if recipe == "layer":
                np.testing.assert_array_equal(bits(o["iou"]), bits(gold[key + ".iou"]), err_msg=key)
                np.testing.assert_array_equal(o["rois"], gold[key + ".rois"], err_msg=key)
            compared += 1
    assert compared > 50


def test_layer_trims_sum_zero_gt_rows_the_oracle_keeps():
    """a documented deviation: the reference layer trims trailing GT rows whose sum is 0 (`while cur_gt[k].sum() == 0`),
    the device and the oracle only all-zero rows.  A row [1, -1, 0, 0, 0, 0, 0] is a GT box to the device"""
    gt = np.zeros((3, 7), np.float32)
    gt[0] = RS.gts(1)[0]
    gt[1, :2] = [1.0, -1.0]
    assert len(RO.trimmed_gt(gt)) == 2
    k = len(gt) - 1
    while gt[k].sum() == 0:
        k -= 1
    assert k + 1 == 1

"""The RPN proposal edge families of proposal_reference.py on the CPU: every family hits its edge, oracle/proposal.py
reproduces the reference's own Python on them (tests/golden/proposal_edges.npz, oracle/make_golden_proposal_edges.py),
and a host restatement of the kernel's structure (csrc/proposal.cu: capped candidate lists, the far range's fallback
slice, greedy NMS in 32-candidate chunks that stops at post_nms_top_n, the pack) equals the oracle, while each plausible
kernel mistake restated on the host gives a different output on at least one family."""
import os
import sys

import numpy as np
import pytest

import proposal_reference as PR
from oracle import oracle as O
from oracle import proposal as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.append(os.path.join(ROOT, "oracle"))
from make_golden_proposal_edges import DECODE_ROWS, GOLDEN, cases  # noqa: E402

CASES = cases()
F = np.float32


def bits(a):
    a = np.array(a, dtype=F)
    a[np.isnan(a)] = F("nan")
    return a.view(np.int32)


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def scenes():
    return {c[0]: PR.scene(c[1], c[2], c[3], c[4]) for c in CASES}


def _decoded(reg, xyz):
    return P.decode_bbox_target(xyz, reg, PR.ANCHOR, 3.0, 0.5, 12, True)


# ------------------------------------------------------------------------------------------------ the oracle is the reference
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_the_reference_python(gold, scenes, case):
    name, f, v, n, seed, modes = case
    scores, reg, xyz = scenes[name]
    if name + ".decode" in gold:
        assert np.array_equal(bits(_decoded(reg[:DECODE_ROWS], xyz[:DECODE_ROWS])), bits(gold[name + ".decode"]))
    for mode in modes:
        kw = PR.MODES[mode]
        if gold["%s.%s_raises" % (name, mode)]:
            with pytest.raises(AssertionError):
                P.proposal_layer(scores[None], reg[None], xyz[None], PR.ANCHOR, **kw)
            continue
        b, s = P.proposal_layer(scores[None], reg[None], xyz[None], PR.ANCHOR, **kw)
        assert np.array_equal(bits(b[0]), bits(gold["%s.%s_boxes" % (name, mode)])), mode
        assert np.array_equal(bits(s[0]), bits(gold["%s.%s_scores" % (name, mode)])), mode


def test_only_the_empty_near_range_raises(gold):
    raised = sorted(k for k in gold.files if k.endswith("_raises") and gold[k])
    assert raised == ["quota_edges.near_empty.test_normal_raises", "quota_edges.near_empty.train_normal_raises"]


# ------------------------------------------------------------------------------------------------ the families hit their edges
def test_range_edges_decode_onto_every_boundary():
    scores, reg, xyz = PR.scene("range_edges", n=2048, seed=1)
    z = _decoded(reg, xyz)[:, 2]
    for v in PR.RANGE_VALUES:
        assert (z.view(np.int32) == np.array(v, F).view(np.int32)).sum() >= 10, "no decoded z equal to %r" % v


def test_argmax_edges_hold_every_kind():
    _, reg, _ = PR.scene("argmax_edges", n=2048, seed=1)
    for lo in (PR.XB, PR.ZB, PR.HB):
        g = reg[:, lo:lo + PR.NB]
        nan = np.isnan(g)
        first_nan = np.where(nan.any(1), np.argmax(nan, 1), -1)
        assert (first_nan > 0).sum() > 0 and (first_nan == 0).sum() > 0, "NaN at position 0 and later"
        fin = np.where(nan, -np.inf, g)
        top = (fin == fin.max(1, keepdims=True)) & ~nan.any(1, keepdims=True)
        assert (top.sum(1) >= 2).sum() > 0, "tied maxima"
        assert (g == 0).all(1).sum() > 0 and (g == -np.inf).all(1).sum() > 0 and (g == np.inf).any(1).sum() > 0


def test_heading_wrap_lands_on_every_target():
    _, reg, _ = PR.scene("heading_wrap", n=2048, seed=1)
    ry = PR.pre_wrap_ry(reg)
    for t in PR.wrap_targets():
        assert (ry == t).sum() >= 16, "pre-wrap heading %r not hit" % t


def test_degenerate_sizes_are_exact():
    _, reg, xyz = PR.scene("degenerate_sizes", n=2048, seed=1)
    d = _decoded(reg, xyz)
    for c in (3, 4, 5):
        assert (d[:, c] == 0).sum() >= 16 and (d[:, c] < 0).sum() + (c == 3) * 16 >= 16
    assert (d[:, 4] >= 999).sum() >= 32 and (d[:, 5] >= 999).sum() >= 32


def test_non_finite_reaches_scores_boxes_and_headings():
    scores, reg, xyz = PR.scene("non_finite", n=2048, seed=1)
    d = _decoded(reg, xyz)
    assert np.isnan(scores).sum() == 1 and (scores == np.inf).sum() == 1 and (scores == -np.inf).sum() == 1
    for c in range(7):
        assert (~np.isfinite(d[:, c])).sum() > 0, "column %d never non-finite" % c


@pytest.mark.parametrize("variant", list(PR.QUOTA))
def test_quota_edges_have_their_counts(variant):
    scores, reg, xyz = PR.scene("quota_edges", variant, PR.N, seed=1)
    z = _decoded(reg, xyz)[:, 2]
    near, far, far_top = PR.QUOTA[variant]
    assert ((z > 0) & (z <= 40)).sum() == near and ((z > 40) & (z <= 80)).sum() == far
    if far_top:
        o = P.descending(scores)
        assert ((z[o[:far]] > 40) & (z[o[:far]] <= 80)).all()


def test_threshold_pairs_straddle_both_thresholds_within_ulps():
    _, reg, xyz = PR.scene("nms_clusters", "thresh", 2048, seed=1)
    d = _decoded(reg, xyz)[:28]
    bev = O.boxes3d_to_bev(d)
    a, b = bev[0::2], bev[1::2]
    inter = (np.minimum(a[:, 2], b[:, 2]) - np.maximum(a[:, 0], b[:, 0])) * (np.minimum(a[:, 3], b[:, 3]) - np.maximum(a[:, 1], b[:, 1]))
    union = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1]) + (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1]) - inter
    iou = (inter / union).astype(F)
    for t in (F(0.8), F(0.85)):
        steps = iou.view(np.int32).astype(np.int64) - np.int64(t.view(np.int32))
        assert ((steps < 0) & (steps >= -4)).any() and ((steps > 0) & (steps <= 4)).any(), t


# ------------------------------------------------------------------------------------------------ the kernel's structure
def _hits(bev, thresh):
    """hit[i, j] (i < j): the axis-aligned IoU of candidate i over candidate j exceeds the threshold (the NMS mask)"""
    n = bev.shape[0]
    if n == 0:
        return np.zeros((0, 0), bool)
    m = O.nms_mask(bev, thresh, normal=True)
    return np.unpackbits(m.view(np.uint8), axis=1, bitorder="little")[:, :n].astype(bool)


def _chunked_nms(bev, thresh, post, mutant, reached):
    """proposal_select_nms_kernel's phase 2: 32 candidates at a time, each tested against the kept boxes and then against
    the earlier survivors of its chunk, stopping once `post` boxes are kept"""
    hit = _hits(bev, thresh)
    kept = []
    for c0 in range(0, bev.shape[0], 32):
        if len(kept) >= post:
            break
        c1 = min(c0 + 32, bev.shape[0])
        dead = hit[kept, c0:c1].any(0) if kept else np.zeros(c1 - c0, bool)
        new = []
        for c in range(c0, c1):
            if not dead[c - c0] and (mutant == "no_in_chunk_suppression" or not hit[new, c].any()):
                new.append(c)
        if len(kept) < post <= len(kept) + len(new):
            reached.append(new[post - len(kept) - 1])
        kept += new
    return kept if mutant == "keeps_past_post" else kept[:post]


def restated(scores, reg, xyz, mode, mutant=None, info=None):
    """one scene through the kernel's selection, NMS and pack, with the axis-aligned NMS"""
    m = PR.MODES[mode]
    pre, post, thresh = m["pre_nms_top_n"], m["post_nms_top_n"], m["nms_thresh"]
    boxes = _decoded(reg, xyz)
    boxes[:, 1] = boxes[:, 1] + boxes[:, 3] / F(2)
    order = P.descending(scores)
    info = {} if info is None else info
    info.setdefault("reached", [])
    if not m["distance_based"]:
        lists, posts = [order[:pre]], [post]
    else:
        pre0, post0 = int(pre * 0.7), int(post * 0.7)
        z = boxes[order, 2]
        near = order[(z > 0) & ((z < 40) if mutant == "near_range_open" else (z <= 40))]
        far = order[(z > 40) & (z <= 80)]
        if far.size:
            second = far[:pre - pre0]
        else:
            start = 0 if mutant == "fallback_from_0" else pre0
            second = near[start:start + pre - pre0]
            info["fallback_first"] = int(np.nonzero(order[np.isin(order, near)] == second[0])[0][0]) if second.size else None
        lists, posts = [near[:pre0], second], [post0, post - post0]
    rows = []
    for cand, p in zip(lists, posts):
        keep = _chunked_nms(O.boxes3d_to_bev(boxes[cand]), thresh, p, mutant, info["reached"])
        rows.append(cand[np.asarray(keep, np.int64)])
    ret_b, ret_s = np.zeros((post, 7), F), np.zeros(post, F)
    at = 0
    for a, r in enumerate(rows):
        if a == 1 and mutant == "pack_area1_at_post0":
            at = posts[0]
        r = r[:max(0, post - at)]
        ret_b[at:at + len(r)], ret_s[at:at + len(r)] = boxes[r], scores[r]
        at += len(r)
    return ret_b, ret_s


def _argmax_last(a):
    return a.shape[1] - 1 - np.argmax(a[:, ::-1], axis=1)


def _argmax_skipping_nan(a):
    """the loop `if (v > bv) best = k`: a NaN after position 0 never wins"""
    best, bv = np.zeros(a.shape[0], np.int64), a[:, 0].copy()
    for k in range(1, a.shape[1]):
        up = a[:, k] > bv
        best[up], bv[up] = k, a[up, k]
    return best


MUTANTS = {"argmax_last_maximum": _argmax_last, "argmax_skips_nan": _argmax_skipping_nan, "near_range_open": None,
           "fallback_from_0": None, "no_in_chunk_suppression": None, "pack_area1_at_post0": None, "keeps_past_post": None}
AXIS_MODES = ("test_normal", "train_normal")


@pytest.fixture(scope="module")
def oracle_outputs(scenes):
    out = {}
    for name, f, v, n, seed, modes in CASES:
        for mode in AXIS_MODES:
            s, r, x = scenes[name]
            b, sc = P.proposal_layer(s[None], r[None], x[None], PR.ANCHOR, near_empty="far_only", **PR.MODES[mode])
            out[name, mode] = (b[0], sc[0])
    return out


def test_restatement_equals_the_oracle_and_hits_the_chunk_edges(scenes, oracle_outputs):
    reached, fallback = [], []
    for name, f, v, n, seed, modes in CASES:
        for mode in AXIS_MODES:
            info = {}
            b, s = restated(*scenes[name], mode, info=info)
            want_b, want_s = oracle_outputs[name, mode]
            assert np.array_equal(bits(b), bits(want_b)) and np.array_equal(bits(s), bits(want_s)), (name, mode)
            reached += info["reached"]
            if info.get("fallback_first") is not None:
                fallback.append(info["fallback_first"])
    reached = np.array(reached)
    print("post reached at candidates:", sorted(set(reached.tolist()))[:40], "fallback starts:", sorted(set(fallback)))
    assert ((reached + 1) % 32 == 0).sum() > 0, "post never reached at a chunk boundary"
    assert ((reached + 1) % 32 != 0).sum() > 0, "post never reached mid-chunk"
    assert fallback and set(fallback) == {PR.PRE0}, "the fallback slice starts at pre0"


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_kernel_mistakes_are_caught(scenes, oracle_outputs, mutant, monkeypatch):
    if MUTANTS[mutant] is not None:
        monkeypatch.setattr(P, "_argmax", MUTANTS[mutant])
    caught = []
    for name, f, v, n, seed, modes in CASES:
        for mode in AXIS_MODES:
            b, s = restated(*scenes[name], mode, mutant=mutant)
            want_b, want_s = oracle_outputs[name, mode]
            if not (np.array_equal(bits(b), bits(want_b)) and np.array_equal(bits(s), bits(want_s))):
                caught.append("%s/%s" % (name, mode))
    print("mutant %s caught by %d of %d: %s" % (mutant, len(caught), 2 * len(CASES), ", ".join(caught[:6])))
    assert caught, "mutant %s gives the oracle's output on every family" % mutant

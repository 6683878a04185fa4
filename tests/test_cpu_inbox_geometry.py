"""CPU suite: the float64 point-in-box reference (tests/inbox_reference.py), its band, and the host predicates against it."""
import os

import numpy as np
import pytest

import inbox_reference as IR
from oracle import gt_paste as GP
from oracle import kitti_io as KO
from oracle import oracle as O

SEEDS = (3, 4)


def _box(x=0.0, y=1.0, z=10.0, h=1.5, w=1.6, l=4.0, ry=0.0):
    return IR.f32([[x, y, z, h, w, l, ry]])


def test_closed_form_cases():
    b = _box()
    pts = IR.f32([[0.0, 0.25, 10.0],        # centre: y bottom 1.0, h 1.5 -> centre at 0.25
                  [2.0, 0.25, 10.0],        # on the +l/2 face
                  [2.5, 0.25, 10.0],        # 0.5 m past it
                  [0.0, 1.0, 10.0],         # on the bottom face
                  [0.0, -0.5, 10.0],        # on the top face
                  [0.0, 1.25, 10.0]])       # 0.25 m below the bottom
    for rule in ("pool", "label"):
        inside, margin = IR.membership(pts, b, rule)
        assert inside[0].tolist() == [True, True, False, True, True, False]
        np.testing.assert_allclose(margin[0], [0.75, 0.0, -0.5, 0.0, 0.0, -0.25], atol=1e-7)
    # a 30 m long box: the pool rule's cap keeps |dx| <= 10, the label rule has none
    long_ = _box(l=30.0)
    p = IR.f32([[9.5, 0.25, 10.0], [10.5, 0.25, 10.0]])
    assert IR.membership(p, long_, "pool")[0][0].tolist() == [True, False]
    assert IR.membership(p, long_, "label")[0][0].tolist() == [True, True]
    np.testing.assert_allclose(IR.membership(p, long_, "pool")[1][0], [0.5, -0.5], atol=1e-6)
    # turned by pi/2: l lies along z
    t = _box(ry=np.pi / 2)
    assert IR.membership(IR.f32([[0.0, 0.25, 11.9], [1.9, 0.25, 10.0]]), t, "pool")[0][0].tolist() == [True, False]
    # negative or zero sizes hold nothing but an exact face point; a NaN height lets the y test pass (as on the device)
    for rule in IR.RULES:
        assert not IR.membership(pts, _box(w=-1.6), rule)[0].any()
    assert IR.membership(pts[:1], _box(h=np.nan), "pool")[0].all()
    assert not IR.membership(pts[:1], _box(l=np.nan), "pool")[0].any()
    # the paste rule is the pool rule on the box with h + 2
    assert IR.membership(IR.f32([[0.0, -2.0, 10.0]]), b, "paste")[0].all() and not IR.membership(IR.f32([[0.0, -2.0, 10.0]]), b, "pool")[0].any()


# ------------------------------------------------------------------------------------------------ fp32 restatements
def fp32_rule(pts, boxes, rule, mistake=None):
    """the kernels' predicate in numpy fp32 (host cos / sin), with an optional planted mistake"""
    p = IR.f32(pts)
    b = IR.rule_boxes(boxes, rule)
    x, y, z = (p[None, :, k] for k in range(3))
    cx, by, cz, h, w, l, ry = (b[:, k, None] for k in range(7))
    if mistake == "swap_wl":
        w, l = l, w
    c, s = np.cos(ry), np.sin(ry)
    if mistake == "sin_sign":
        s = -s
    with np.errstate(invalid="ignore", over="ignore"):
        dx, dz = x - cx, z - cz
        xr, zr = dx * c - dz * s, dx * s + dz * c
        ok = (np.abs(xr) <= l * np.float32(0.5)) & (np.abs(zr) <= w * np.float32(0.5))
        if rule == "label":
            dy = y - (by - h * np.float32(0.5) if mistake == "y_centre" else by)
            lo = -h * np.float32(0.5) if mistake == "h_not_half" else -h
            return ok & ~((dy > 0) | (dy < lo))
        hh = h.astype(np.float64) / (1.0 if mistake == "h_not_half" else 2.0)
        cy = by if mistake == "y_centre" else (by.astype(np.float64) - h.astype(np.float64) / 2).astype(np.float32)
        ok &= ~(np.abs(y - cy).astype(np.float64) > hh)          # rejecting tests, as in the kernels: NaN keeps
        if mistake == "cap_after_rotation":
            ok &= ~((np.abs(xr) > 10) | (np.abs(zr) > 10))
        elif mistake != "no_cap":
            ok &= ~((np.abs(dx) > 10) | (np.abs(dz) > 10))
    return ok


def _host_predicates():
    from pointrcnn_b200.ext import roipool3d_cuda
    return {
        "oracle": ("pool", lambda p, b: O.pts_in_boxes3d(p, b).astype(bool)),
        "roipool3d_cpu twin": ("pool", lambda p, b: np.stack([roipool3d_cuda._in_box_np(p, q) for q in b])),
        "label oracle": ("label", lambda p, b: np.stack([KO.in_box(p, q) for q in b])),
        "paste oracle": ("paste", lambda p, b: np.stack([GP.paste_in_box(p, q) for q in IR.rule_boxes(b, "paste")])),
        "fp32 pool": ("pool", lambda p, b: fp32_rule(p, b, "pool")),
        "fp32 label": ("label", lambda p, b: fp32_rule(p, b, "label")),
        "fp32 paste": ("paste", lambda p, b: fp32_rule(p, b, "paste")),
    }


@pytest.mark.parametrize("family", IR.FAMILIES)
def test_host_predicates_agree_outside_the_band(family):
    for seed in SEEDS:
        pts, boxes = IR.family(family, seed)
        cls = {r: IR.classify(pts, boxes, r) for r in IR.RULES}
        for name, (rule, fn) in _host_predicates().items():
            with np.errstate(invalid="ignore", over="ignore"):
                got = fn(pts, boxes)
            _, cin, cout = cls[rule]
            assert not (got & cout).any(), "%s (%s rule) takes certainly-outside pairs on %s" % (name, rule, family)
            assert not (~got & cin).any(), "%s (%s rule) drops certainly-inside pairs on %s" % (name, rule, family)


# measured in-band fractions of all point-box pairs of the pool rule, seeds 3 and 4 (see test_band_is_neither_vacuous_nor_huge)
INBAND_LIMIT = {"faces": 4e-3, "edges": 4e-3, "corners": 4e-3, "headings": 2e-3, "cap": 6e-3, "far": 1e-3}


def test_band_is_neither_vacuous_nor_huge():
    for family in ("faces", "edges", "corners", "headings", "cap", "far"):
        fuzzy_in = fuzzy_out = pairs = fuzzy = 0
        for seed in SEEDS:
            pts, boxes = IR.family(family, seed)
            inside, cin, cout = IR.classify(pts, boxes, "pool")
            fz = ~cin & ~cout
            fuzzy_in += int((fz & inside).sum())
            fuzzy_out += int((fz & ~inside).sum())
            fuzzy += int(fz.sum())
            pairs += fz.size
        assert fuzzy_in > 0 and fuzzy_out > 0, "%s: the band must hold pairs on both sides of a face" % family
        assert fuzzy / pairs <= INBAND_LIMIT[family], "%s: in-band fraction %.2e" % (family, fuzzy / pairs)
    for seed in SEEDS:
        pts, boxes = IR.family("random", seed)
        for rule in IR.RULES:
            inside, cin, cout = IR.classify(pts, boxes, rule)
            assert inside.sum() > 100 and (~cin & ~cout).sum() == 0, "random scope: no pair may fall in the band"
    # the band is a few ulp of the differences and box coordinates: about 1e-5 m at 3e4 m as near the sensor, since the
    # fp32 inputs are exact and the differences of nearby points are small
    for family in ("faces", "far"):
        assert 1e-7 < np.median(IR.band(*IR.family(family, 3), "pool")) < 5e-5


MISTAKES = {
    "swap_wl": ("pool", "label"),
    "sin_sign": ("pool", "label"),
    "y_centre": ("pool", "label"),
    "h_not_half": ("pool", "label"),
    "no_cap": ("pool", "paste"),
    "cap_after_rotation": ("pool", "paste"),
}


@pytest.mark.parametrize("mistake", sorted(MISTAKES))
def test_planted_mistakes_are_caught(mistake):
    for rule in MISTAKES[mistake]:
        caught = []
        for family in IR.FAMILIES:
            pts, boxes = IR.family(family, SEEDS[0])
            _, cin, cout = IR.classify(pts, boxes, rule)
            with np.errstate(invalid="ignore", over="ignore"):
                got = fp32_rule(pts, boxes, rule, mistake)
            if ((got & cout) | (~got & cin)).any():
                caught.append(family)
        assert caught, "planted mistake %s in the %s rule passes every family" % (mistake, rule)


def test_reference_labels_lie_in_the_band():
    """the reference's own labels (its Delaunay hull of the fp32 corners): a label that differs from the float64 replay of
    generate_rpn_training_labels' loop is one the replay allows when in-band decisions go the other way, and where every
    decision is certain the regression targets are those of the last box the point is in"""
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti_io.npz"))
    gt = KO.synth_scan(11, 30000, 6)[1]
    cls = gold["probe_cls"]
    fuzzy = IR.check_labels(cls, gold["probe_reg"], gold["probe_pts"], gt, delaunay=True, where="reference probe")
    assert fuzzy < 0.01 * len(cls) and (cls == 1).sum() > 500 and (cls == -1).sum() > 200

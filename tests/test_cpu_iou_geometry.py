"""The rotated BEV overlap of the CPU oracle (a statement-by-statement restatement of the reference kernel) against the
float64 clip of iou_reference.py, on every seeded pair family: the error bound on well-conditioned pairs, its power to
catch planted mistakes, the conditioning classifier, the polygon vertex count, and the pinned far-range behaviour of
identical boxes."""
import numpy as np
import pytest

import iou_reference as I
from oracle import oracle as O

N = 3000
SEED = 2024
CASES = [(f, p) for f in I.FAMILIES for p in I.PLACES] + [("generic", "off1000")]


@pytest.fixture(scope="module")
def pairs():
    out = {}
    for f, p in CASES:
        a7, b7 = I.family(f, p, N, SEED)
        a, b = I.to_bev(a7), I.to_bev(b7)
        got, cnt = O.box_overlap_pairs(a, b)
        out[(f, p)] = dict(a=a, b=b, got=got, cnt=cnt, exact=I.exact_overlap(a, b), cond=I.conditioning(a, b))
    return out


def test_clip_is_exact_on_known_shapes():
    """the float64 clip on shapes with a closed-form overlap: a box with itself, nested boxes, a half-shifted box, a
    square turned by 45 degrees inside a larger one, disjoint and touching boxes"""
    a = np.array([[0, 0, 4, 2, 0.3]] * 6, np.float32)
    b = np.array([[0, 0, 4, 2, 0.3], [1, 0.5, 3, 1.5, 0.3], [2, 0, 6, 2, 0.0], [10, 10, 11, 11, 0.7], [4, 0, 5, 2, 0.0],
                  [1.5, 0.5, 2.5, 1.5, np.pi / 4]], np.float32)
    a[2, 4] = a[4, 4] = 0.0
    ov = I.exact_overlap(a, b)
    np.testing.assert_allclose(ov, [8.0, 2.0, 4.0, 0.0, 0.0, 1.0], rtol=1e-12, atol=1e-12)


def test_well_conditioned_pairs_are_within_the_bound(pairs):
    worst = 0.0
    for (f, p), d in pairs.items():
        w = ~d["cond"]["ill"]
        if not w.any():
            continue
        ok, ratio, bad = I.check(d["got"][w], d["exact"][w], I.bound(d["a"][w], d["b"][w], d["cond"]["R"][w]))
        print("%-12s %-8s well-conditioned %5d  max err/bound %.4f" % (f, p, w.sum(), ratio))
        assert ok, "%s@%s: %d well-conditioned pairs outside the bound (max err/bound %.3g)" % (f, p, bad, ratio)
        assert ratio < 0.25, "%s@%s: the oracle uses %.3g of the bound" % (f, p, ratio)
        worst = max(worst, ratio)
    assert worst > 0, "no rounding error seen: the bound was not exercised"


def test_generic_families_are_mostly_well_conditioned(pairs):
    for f in ("generic", "nested", "pedestrian", "big"):
        for p in I.PLACES:
            assert (~pairs[(f, p)]["cond"]["ill"]).mean() > 0.9, (f, p)


@pytest.mark.parametrize("family", I.ILL)
def test_fragile_families_are_classified_ill_conditioned(pairs, family):
    """guards the classifier: every pair of a family built on a fragile configuration is flagged, at both placements"""
    for p in I.PLACES:
        d = pairs[(family, p)]
        ill = d["cond"]["ill"]
        print("%-12s %-8s ill-conditioned %d/%d  oracle overlap range [%.4g, %.4g]" % (
            family, p, ill.sum(), len(ill), np.nanmin(d["got"]), np.nanmax(d["got"])))
        assert ill.all(), "%s@%s: %d pairs classified well-conditioned" % (family, p, (~ill).sum())


def test_polygon_never_exceeds_sixteen_vertices(pairs):
    """the kernels keep the intersection polygon in 16 slots (cp[16], 16-slot shared-memory columns)"""
    worst = {k: int(d["cnt"].max()) for k, d in pairs.items()}
    print("largest vertex count per family:", worst)
    assert max(worst.values()) <= 16
    assert max(worst.values()) == 16, "no family reaches the 16-vertex edge case any more"


def test_identical_boxes_can_overlap_less_than_themselves_at_far_range(pairs):
    """pinned reference behaviour, not a truth claim: the corners of a box rotated there and back miss the box's own
    MARGIN at far range, so IoU(a, a) < 1 for some seeded identical pairs (never near the origin)"""
    for p in I.PLACES:
        d = pairs[("identical", p)]
        area = I.bev_area(d["a"])
        short = d["got"] < area * (1 - 1e-3)
        print("identical@%s: %d of %d pairs overlap less than their area, smallest ratio %.3g" % (
            p, short.sum(), len(short), (d["got"] / area).min()))
        if p == "far":
            assert short.any()
        else:
            assert not short.any()


# ------------------------------------------------------------------------------------------------ sensitivity
MUTANTS = {1: "last corner of b never tested", 2: "sin of the heading negated", 4: "sort stops one pass early"}


@pytest.mark.parametrize("mutant", sorted(MUTANTS), ids=[MUTANTS[m].replace(" ", "_") for m in sorted(MUTANTS)])
@pytest.mark.parametrize("place", I.PLACES)
def test_bound_catches_a_planted_mistake(pairs, mutant, place):
    d = pairs[("generic", place)]
    w = ~d["cond"]["ill"]
    got, _ = O.box_overlap_pairs(d["a"], d["b"], mutant)
    ok, ratio, bad = I.check(got[w], d["exact"][w], I.bound(d["a"][w], d["b"][w], d["cond"]["R"][w]))
    print("mutant %-32s %s: %d pairs outside the bound, max err/bound %.3g" % (MUTANTS[mutant], place, bad, ratio))
    assert not ok


def test_reversed_sort_is_not_a_mistake(pairs):
    """sorting the polygon by decreasing angle walks it clockwise; the fan area takes fabs, so the overlap is unchanged --
    the bound must not (and does not) flag it"""
    d = pairs[("generic", "far")]
    got, _ = O.box_overlap_pairs(d["a"], d["b"], 3)
    w = ~d["cond"]["ill"]
    assert I.check(got[w], d["exact"][w], I.bound(d["a"][w], d["b"][w], d["cond"]["R"][w]))[0]

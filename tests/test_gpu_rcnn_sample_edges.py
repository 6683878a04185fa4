"""prb_rcnn_sample_rois and prb_rcnn_roi_targets at their edges.

The sampler is called directly with the crafted IoU matrices of tests/rcnn_sample_reference.py and 0 jitter tries, so
every row keeps its source box and IoU; status, sel, iou_out, rois_out, gt_out and pool_boxes must equal
oracle/rcnn_offline.py::sample_scene(draw="hash", iou3d=M) bit for bit, under the loader's and the layer's recipe, with
every output prefilled with a sentinel and followed by guard words.  Simulated mistakes (last-max, `>` for fg, the hard /
easy count off by one) must fail that comparison.  The jitter loop's inline IoU is checked against prb_boxes_iou3d on
real box families; the targets kernel's labels exactly and its canonical transform within a derived fp32 bound."""
import numpy as np
import pytest
import torch

import iou_reference as IR
import rcnn_sample_reference as RS
from oracle import rcnn_offline as RO
from rcnn_sample_reference import bits, run_oracle

pytestmark = pytest.mark.gpu
RECIPES = ("loader", "layer")
SENT = 0x7fc0dead                 # a NaN pattern no kernel writes
GUARD = 1024
SEED = 0x2026


def _C():
    from pointrcnn_b200 import _cabi as C
    return C


def recipe(which, case_cfg, R, tries=0):
    from pointrcnn_b200.rcnn import targets as TG
    d = {k: v for k, v in TG.DEFAULT_CFG.items() if k != "RCNN"}
    d["RCNN"] = dict(TG.DEFAULT_CFG["RCNN"], ROI_PER_IMAGE=R, **case_cfg)
    cfg = TG.ns(d)
    rc = TG.loader_recipe(cfg, "TRAIN") if which == "loader" else TG.layer_recipe(cfg)
    return rc._replace(fg_aug_times=tries, bg_aug_times=min(tries, 1))


def _buf(cuda, n, dtype):
    t = torch.empty(n + GUARD, dtype=torch.int32, device=cuda).fill_(SENT)
    return t if dtype == torch.int32 else t.view(dtype)


def device_sample(cuda, rc, rois, gts, iou, roi_count=None, gt_count=None, seed=SEED):
    """rois (B,m,7), gts (B,g,7), iou (B,m,g) numpy -> dict of numpy outputs; asserts every output word was written and
    no guard word behind an output was"""
    C = _C()
    B, m, g = iou.shape
    R = rc.roi_per_image
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    d_iou, d_rois, d_gts = T(iou), T(rois), T(gts)
    counts = None
    if rc.counts:
        counts = T(np.stack([np.full(B, m) if roi_count is None else roi_count, np.full(B, g) if gt_count is None else gt_count]).astype(np.int32))
    out = dict(rois=_buf(cuda, B * R * 7, torch.float32), gts=_buf(cuda, B * R * 7, torch.float32), iou=_buf(cuda, B * R, torch.float32),
               pool=_buf(cuda, B * R * 7, torch.float32), sel=_buf(cuda, B * R * 3, torch.int32), status=_buf(cuda, B, torch.int32))
    rc_ = C.lib().prb_rcnn_sample_rois(
        B, m, g, C.ptr(d_iou), C.ptr(d_rois), C.ptr(counts[0]) if counts is not None else None, C.ptr(d_gts),
        C.ptr(counts[1]) if counts is not None else None, R, rc.fg_per_image, rc.reg_fg_thresh, rc.cls_fg_thresh, rc.cls_bg_thresh,
        rc.cls_bg_thresh_lo, rc.hard_bg_ratio, rc.aug_method, rc.gt_max_fg, rc.fg_aug_times, rc.bg_aug_times, rc.kept_src_iou,
        rc.pool_extra_width, seed, C.ptr(out["rois"]), C.ptr(out["gts"]), C.ptr(out["iou"]), C.ptr(out["pool"]), C.ptr(out["sel"]),
        C.ptr(out["status"]), C.stream())
    C.check(rc_, "rcnn_sample_rois")
    sizes = dict(rois=B * R * 7, gts=B * R * 7, iou=B * R, pool=B * R * 7, sel=B * R * 3, status=B)
    res = {}
    for k, n in sizes.items():
        w = out[k].view(torch.int32).cpu().numpy()
        assert (w[:n] != SENT).all(), "%s: %d words never written" % (k, (w[:n] == SENT).sum())
        assert (w[n:] == SENT).all(), "%s: %d guard words overwritten" % (k, (w[n:] != SENT).sum())
        res[k] = out[k].cpu().numpy()[:n]
    shp = dict(rois=(B, R, 7), gts=(B, R, 7), iou=(B, R), pool=(B, R, 7), sel=(B, R, 3), status=(B,))
    return {k: v.reshape(shp[k]) for k, v in res.items()}


def expected(o, rc):
    """the device's outputs of one scene from the oracle's"""
    R = rc.roi_per_image
    if o["status"] != 0:
        pool = np.tile(np.array([0, 0, 0, -1, -1, -1, 0], np.float32), (R, 1))
    else:
        pool = RO.enlarge_box3d(o["rois"], rc.pool_extra_width)
    return dict(status=o["status"], sel=o["sel"], iou=o["iou"], rois=o["rois"], gts=o["gt_of_rois"], pool=pool)


def compare(dev, b, exp, what):
    assert int(dev["status"][b]) == exp["status"], (what, "status", int(dev["status"][b]), exp["status"])
    np.testing.assert_array_equal(dev["sel"][b], exp["sel"], err_msg="%s sel" % what)
    for k in ("iou", "rois", "gts", "pool"):
        np.testing.assert_array_equal(bits(dev[k][b]), bits(exp[k]), err_msg="%s %s" % (what, k))


def run_case(cuda, case, which, seed=SEED):
    rc = recipe(which, case["cfg"], case["R"])
    r, t, M = RS.scene(case)
    rc_count = None if case["roi_count"] is None else np.array([case["roi_count"]])
    gt_count = None if case["gt_count"] is None else np.array([case["gt_count"]])
    dev = device_sample(cuda, rc, r[None], t[None], M[None], rc_count, gt_count, seed)
    return dev, rc


@pytest.mark.parametrize("which", RECIPES)
def test_crafted_matrices_bit_exact(cuda, which):
    for case in RS.cases():
        dev, rc = run_case(cuda, case, which)
        o = run_oracle(case, which, seed=SEED)
        compare(dev, 0, expected(o, rc), "%s.%s" % (case["name"], which))


@pytest.mark.parametrize("which", RECIPES)
def test_limit_sizes_bit_exact(cuda, which):
    """m = 4096 RoIs, g = 256 GT boxes, R = 1024 rows: ~101 KB of dynamic shared memory; fg lists of n + ng candidates"""
    fg = []
    for case in RS.big_cases():
        dev, rc = run_case(cuda, case, which)
        o = run_oracle(case, which, seed=SEED)
        compare(dev, 0, expected(o, rc), "%s.%s" % (case["name"], which))
        fg.append(o["candidates"]["fg"].size)
    if which == "loader":
        assert fg[1] == 4096 + 256


@pytest.mark.parametrize("which", RECIPES)
def test_batch_of_branches(cuda, which):
    cs = RS.batch_cases()
    rc = recipe(which, {}, cs[0]["R"])
    sc = [RS.scene(c, i) for i, c in enumerate(cs)]
    dev = device_sample(cuda, rc, np.stack([s[0] for s in sc]), np.stack([s[1] for s in sc]), np.stack([s[2] for s in sc]))
    branches = set()
    for i, c in enumerate(cs):
        o = run_oracle(c, which, seed=SEED, index=i)
        compare(dev, i, expected(o, rc), "%s.%s" % (c["name"], which))
        branches.add(o["branch"])
    assert branches >= {"fg+bg", "fg", "bg"}
    assert which == "loader" or "none" in branches


def _case(name):
    return next(c for c in RS.cases() if c["name"] == name)


def _rejects(dev, exp, what):
    with pytest.raises(AssertionError):
        compare(dev, 0, exp, what)


@pytest.mark.parametrize("which", RECIPES)
def test_catches_last_max(cuda, which):
    """simulated: the GT of a tied row is the last maximum, not the first"""
    case = _case("row_ties")
    dev, rc = run_case(cuda, case, which)
    o = run_oracle(case, which, seed=SEED)
    exp = expected(o, rc)
    M, t = case["iou"], RS.scene(case)[1]
    last = M.shape[1] - 1 - M[:, ::-1].argmax(1)
    src = exp["sel"][:, 0]
    assert (last[src] != exp["sel"][:, 1]).any()
    exp["sel"] = exp["sel"].copy()
    exp["sel"][:, 1] = last[src]
    exp["gts"] = t[last[src]]
    _rejects(dev, exp, "last max")


@pytest.mark.parametrize("which", RECIPES)
def test_catches_strict_fg_threshold(cuda, which):
    """simulated: fg is max_overlaps > fg_thresh (the oracle's threshold one ulp up)"""
    case = _case("thresholds")
    dev, rc = run_case(cuda, case, which)
    bad = dict(case, cfg=dict(case["cfg"], REG_FG_THRESH=float(RS.up(RS.FG))))
    _rejects(dev, expected(run_oracle(bad, which, seed=SEED), rc), "> for fg")


@pytest.mark.parametrize("which", RECIPES)
def test_catches_hard_easy_split_off_by_one(cuda, which):
    """simulated: one hard bg row more than int(bg_rows * HARD_BG_RATIO)"""
    case = _case("ratio_0.29")
    dev, rc = run_case(cuda, case, which)
    rows = 100 if which == "layer" else 99           # R = 128 less 28 fg rows (29 with the loader's GT-max RoI)
    assert int((run_oracle(case, which, seed=SEED)["sel"][:, 0] < 28).sum()) == 128 - rows
    # the ratio that makes int(rows * ratio) one larger
    bad = dict(case, cfg=dict(case["cfg"], HARD_BG_RATIO=(int(rows * 0.29) + 1.5) / rows))
    _rejects(dev, expected(run_oracle(bad, which, seed=SEED), rc), "hard / easy split")


def test_refusals_leave_outputs_untouched(cuda):
    """sizes past the kernel's limits and out-of-range recipe values are refused before a launch: rc != 0, nothing written"""
    C = _C()
    rc = recipe("loader", {}, 16)
    for m, g, R, fg, ratio in ((4097, 4, 16, 8, 0.8), (4, 257, 16, 8, 0.8), (4, 4, 1025, 8, 0.8), (4, 4, 0, 0, 0.8), (4, 4, 16, 17, 0.8),
                               (4, 4, 16, 8, 1.5), (4, 4, 16, 8, -0.1)):
        iou = torch.zeros((1, m, g), device=cuda)
        rois, gts = torch.zeros((1, m, 7), device=cuda), torch.zeros((1, g, 7), device=cuda)
        outs = [_buf(cuda, max(R, 1) * 7, torch.float32) for _ in range(4)] + [_buf(cuda, max(R, 1) * 3, torch.int32), _buf(cuda, 1, torch.int32)]
        r = C.lib().prb_rcnn_sample_rois(1, m, g, C.ptr(iou), C.ptr(rois), None, C.ptr(gts), None, R, fg, rc.reg_fg_thresh, rc.cls_fg_thresh,
                                         rc.cls_bg_thresh, rc.cls_bg_thresh_lo, ratio, rc.aug_method, 1, 0, 0, 0, 1.0, 1,
                                         *[C.ptr(o) for o in outs], C.stream())
        assert r != 0, (m, g, R, fg, ratio)
        torch.cuda.synchronize()
        for o in outs:
            assert (o.view(torch.int32) == SENT).all().item(), (m, g, R, fg, ratio)


# ------------------------------------------------------------------------------------------------ the jitter loop's IoU
JITTER_FAMILIES = (("shifted", "near"), ("rotated", "far"), ("generic", "far"), ("nested", "near"), ("zero", "near"))


def _pair_iou(cuda, a, b):
    """prb_boxes_iou3d of aligned rows: (n,7), (n,7) -> (n,)"""
    C = _C()
    n = a.shape[0]
    A, Bx = (torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(cuda).view(n, 1, 7) for x in (a, b))
    out = torch.empty((n, 1, 1), device=cuda)
    C.check(C.lib().prb_boxes_iou3d(n, 1, C.ptr(A), 1, C.ptr(Bx), C.ptr(out), C.stream()), "boxes_iou3d")
    return out.view(n).cpu().numpy()


@pytest.mark.parametrize("which", RECIPES)
def test_jitter_loop_iou_equals_boxes_iou3d(cuda, which):
    """real boxes, the IoU matrix from prb_boxes_iou3d, the recipe's default tries: a row whose last try jittered the box
    (or, in the loader, any row that tried) reports prb_boxes_iou3d of its output box and GT bit for bit; a row that
    kept its source box under the layer reports the source's max_overlaps"""
    C = _C()
    n, R = 48, 64
    fam = [IR.family(f, p, n, 700 + i) for i, (f, p) in enumerate(JITTER_FAMILIES)]
    gts = np.stack([a for a, _ in fam])
    rois = np.stack([b for _, b in fam])
    B = len(fam)
    T = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(cuda)
    iou = torch.empty((B, n, n), device=cuda)
    d_rois, d_gts = T(rois), T(gts)                  # held: a freed temporary's block is reused by the next allocation
    C.check(C.lib().prb_boxes_iou3d(B, n, C.ptr(d_rois), n, C.ptr(d_gts), C.ptr(iou), C.stream()), "boxes_iou3d")
    M = iou.cpu().numpy()
    assert (M.max(2) >= RS.FG).sum() > n and (M.max(2) < RS.LO).sum() > n // 2      # fg rows with 10 tries, bg rows with 1
    rc = recipe(which, {}, R, tries=10)
    assert rc.fg_aug_times == 10 and rc.bg_aug_times == 1
    dev = device_sample(cuda, rc, rois, gts, M)
    pair = _pair_iou(cuda, dev["rois"].reshape(-1, 7), dev["gts"].reshape(-1, 7)).reshape(B, R)
    jittered = kept = 0
    assert (dev["status"] == 0).sum() >= B - 1
    for b in range(B):
        if dev["status"][b] != 0:
            continue
        arg = M[b].argmax(1)
        mo = M[b][np.arange(n), arg]
        hd = RO.HashDraws(SEED, b)
        for r in range(R):
            src, ga, tries = (int(v) for v in dev["sel"][b, r])
            assert ga == arg[src]
            np.testing.assert_array_equal(dev["gts"][b, r], gts[b, ga])
            keep = tries > 0 and hd.keep(r, tries - 1)
            if tries > 0 and not (which == "layer" and keep):
                assert bits(dev["iou"][b, r]) == bits(pair[b, r]), (b, r, dev["iou"][b, r], pair[b, r])
                jittered += not keep
            else:
                assert bits(dev["iou"][b, r]) == bits(mo[src]), (b, r, dev["iou"][b, r], mo[src])
                np.testing.assert_array_equal(dev["rois"][b, r], rois[b, src])
                kept += 1
    assert jittered > B * R // 4 and (which == "loader" or kept > 0), (jittered, kept)


# ------------------------------------------------------------------------------------------------ prb_rcnn_roi_targets
U = 2.0 ** -24
TWO_PI32 = float(np.float32(2 * np.pi))        # the reference's `% (2 * np.pi)` on fp32 values divides by this
RYS = [0.0, -0.0, np.pi, -np.pi, 2 * np.pi, -2 * np.pi, 2 * np.pi * 1000, -2 * np.pi * 999, -1e-8, -3e-6, 1.0, -2.5, 7.0]
IOUS = [v for t in (RS.BG, RS.FG, RS.CLS) for v in (RS.dn(t), t, RS.up(t))] + [RS.LO, np.float32(0), np.float32(-0.0), np.float32(1),
                                                                              RS.NAN]


def _targets_inputs(S=64, W=5, seed=3):
    """one row per (ry, IoU, empty) combination: RoIs at 70 m, GT boxes beside them, S points within 3 m of the RoI"""
    rng = np.random.default_rng(seed)
    rows = [(ry, v, e) for ry in RYS for v in IOUS for e in (0, 1)]
    K = len(rows)
    phi = rng.uniform(np.radians(25), np.radians(155), K)
    roi = np.zeros((K, 7), np.float32)
    roi[:, 0], roi[:, 2], roi[:, 1] = 70 * np.cos(phi), 70 * np.sin(phi), 1.6
    roi[:, 3:6] = [1.5, 1.6, 3.9]
    roi[:, 6] = [r[0] for r in rows]
    gt = roi.copy()
    gt[:, [0, 1, 2]] += rng.uniform(-0.4, 0.4, (K, 3)).astype(np.float32)
    gt[:, 3:6] *= np.float32(1.05)
    gt[:, 6] = roi[:, 6] + np.float32(0.05)
    pts = np.zeros((K, S, W), np.float32)
    pts[:, :, 0:3] = roi[:, None, 0:3] + rng.uniform(-3, 3, (K, S, 3)).astype(np.float32)
    pts[:, :, 3:] = rng.standard_normal((K, S, W - 3)).astype(np.float32)
    iou = np.array([r[1] for r in rows], np.float32)
    empty = np.array([r[2] for r in rows], np.int32)
    return pts, roi, gt, iou, empty


def _restate(pts, roi, gt, rc, k, R):
    """float64: stage-2 augmentation with the device's draws (oracle/rcnn_offline.py), then the canonical transform with
    the fp32 2 pi modulus; -> points (S,3), roi, gt, gt_ct and the per-row bound terms"""
    p, rb, gb = pts[:, 0:3].astype(np.float64), roi.astype(np.float64), gt.astype(np.float64)
    if rc.aug_data:
        c = dict(AUG_METHOD_LIST=["rotation", "scaling", "flip"], AUG_METHOD_PROB=[1.0, 1.0, rc.flip_prob], AUG_ROT_RANGE=18)
        en, angle, scale = RO.HashDraws(SEED, k // R, None if rc.rot_hi != 0.0 else 0.0).aug(k % R, c)
        p, rb, gb = RO._augment_f64(p, roi, gt, en, angle, scale, c)
    roi_ry = np.fmod(rb[6], TWO_PI32)
    roi_ry = roi_ry + TWO_PI32 if roi_ry < 0 else roi_ry
    a = rb[6] if rc.pts_raw_ry else roi_ry
    q = p - rb[0:3]
    x, z = q[:, 0] * np.cos(a) - q[:, 2] * np.sin(a), q[:, 0] * np.sin(a) + q[:, 2] * np.cos(a)
    q[:, 0], q[:, 2] = x, z
    g = gb.copy()
    g[0:3] -= rb[0:3]
    g[0], g[2] = g[0] * np.cos(roi_ry) - g[2] * np.sin(roi_ry), g[0] * np.sin(roi_ry) + g[2] * np.cos(roi_ry)
    g[6] -= roi_ry
    return q, rb, gb, g


def _bounds(rc, A, D, ry):
    """fp32 error bounds (u = 2^-24, sinf / cosf / atan2f within 2 ulp): A the coordinates' magnitude before centring, D
    after, ry the heading's.  Without augmentation a point is one subtraction (u D) and one rotation (3 roundings and two
    2-ulp sines, 11 u D), rotated by an angle off by delta: half an ulp of 2 pi from the + 2 pi of a negative heading.
    Augmentation first rotates (11 u A), scales (u A) and flips (exact) points and boxes at magnitude A, and moves the
    heading through two atan2f (4 ulp of pi) and five roundings at |ry| + 2 pi, plus the fp32 pi of the flip."""
    delta = 2.0 ** -22 if not rc.pts_raw_ry else 0.0
    pos = 16 * U * D + D * delta
    head = 2 * U * (abs(ry) + 2 * np.pi) + delta
    if rc.aug_data:
        d_aug = 4 * 2.0 ** -22 + 10 * U * (abs(ry) + 2 * np.pi) + 1e-7
        pos += 2 * 16 * U * A + D * (d_aug + 2.0 ** -22)
        head += 2 * d_aug + 2.0 ** -22
    return pos, head


@pytest.mark.parametrize("which", RECIPES)
@pytest.mark.parametrize("aug", [0, 1])
def test_roi_targets_labels_exact_transform_bounded(cuda, which, aug):
    C = _C()
    rc = recipe(which, {}, 1)._replace(aug_data=aug)
    pts, roi, gt, iou, empty = _targets_inputs()
    K, S, W = pts.shape
    R = K                                      # one scene: the draws are keyed by row
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    d_pts, d_roi, d_gt, d_iou, d_empty = T(pts), T(roi), T(gt), T(iou), T(empty)
    gt_ct, cls, reg = (torch.empty((K, 7), device=cuda), torch.empty(K, dtype=torch.int32, device=cuda),
                       torch.empty(K, dtype=torch.int32, device=cuda))
    C.check(C.lib().prb_rcnn_roi_targets(1, R, S, W, C.ptr(d_pts), C.ptr(d_roi), C.ptr(d_gt), C.ptr(d_iou), C.ptr(d_empty), rc.aug_data,
                                         rc.aug_rotation, rc.aug_scaling, rc.aug_flip, rc.rot_lo, rc.rot_hi, rc.flip_prob, rc.pts_raw_ry,
                                         rc.reg_fg_thresh, rc.cls_fg_thresh, rc.cls_bg_thresh, SEED, C.ptr(gt_ct), C.ptr(cls), C.ptr(reg),
                                         C.stream()), "rcnn_roi_targets")
    o_pts, o_roi, o_gt, o_ct, o_cls, o_reg = (x.cpu().numpy() for x in (d_pts, d_roi, d_gt, gt_ct, cls, reg))
    # labels: float64 comparisons against the fp32 thresholds; NaN is neither fg nor ignored
    v = iou.astype(np.float64)
    fg, bg, reg_t = float(np.float32(rc.cls_fg_thresh)), float(np.float32(rc.cls_bg_thresh)), float(np.float32(rc.reg_fg_thresh))
    want_cls = np.where((v > bg) & (v < fg) | (empty != 0), -1, (v > fg).astype(np.int32))
    want_reg = ((v > reg_t) & (empty == 0)).astype(np.int32)
    np.testing.assert_array_equal(o_cls, want_cls)
    np.testing.assert_array_equal(o_reg, want_reg)
    assert set(o_cls.tolist()) == {-1, 0, 1} and set(o_reg.tolist()) == {0, 1}
    # the feature columns are not touched
    np.testing.assert_array_equal(o_pts[:, :, 3:], pts[:, :, 3:])
    worst = 0.0
    for k in range(K):
        q, rb, gb, g = _restate(pts[k], roi[k], gt[k], rc, k, R)
        A = max(np.abs(pts[k, :, 0:3]).max(), np.abs(roi[k, 0:3]).max(), np.abs(gt[k, 0:3]).max())
        D = max(np.abs(q).max(), np.abs(g[0:3]).max())
        pos, head = _bounds(rc, A, D, max(abs(float(roi[k, 6])), abs(float(gt[k, 6]))))
        err = np.abs(o_pts[k, :, 0:3] - q).max()
        assert err <= pos, (k, roi[k, 6], err, pos)
        assert np.abs(o_ct[k, 0:6] - g[0:6]).max() <= pos, (k, roi[k, 6], o_ct[k], g, pos)
        assert abs(o_ct[k, 6] - g[6]) <= head, (k, roi[k, 6], o_ct[k, 6], g[6], head)
        box_tol = np.array([pos] * 3 + [4 * U * 4] * 3 + [head])
        assert (np.abs(o_roi[k] - rb) <= box_tol).all(), (k, o_roi[k], rb)
        assert (np.abs(o_gt[k] - gb) <= box_tol).all(), (k, o_gt[k], gb)
        worst = max(worst, err / pos)
    assert worst > 0 or not aug

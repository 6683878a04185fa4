"""The rotated BEV overlap on the device, on the seeded pair families of iou_reference.py (generic, near-duplicate,
touching, degenerate and non-finite pairs, near the origin and at KITTI far range).

The anchor is the overlap / IoU matrix kernel (prb_boxes_overlap_bev / prb_boxes_iou_bev): within the float64 bound on
well-conditioned pairs, and bit-identical to the reference's own kernel (oracle/_ref) on every pair when that library
is present.  The consumers must equal the anchor bit for bit on every pair, ill-conditioned and non-finite ones
included, because a divergence flips NMS keeps and recall counts: the NMS mask, the proposal kernel's NMS, the fused 3D
IoU (against boxes_iou3d_gpu's torch op sequence on the anchor) and the recall statistics."""
import numpy as np
import pytest
import torch

import iou_reference as I
from oracle import oracle as O
from oracle import refgpu as R

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200.ext import iou3d_cuda  # noqa: E402
from pointrcnn_b200.iou3d import iou3d_utils  # noqa: E402

HAVE_REF = R.available()
N = 256                       # pairs per family and placement
SEED = 7
CASES = [(f, p) for f in I.FAMILIES for p in I.PLACES] + [("generic", "off1000")]
IDS = ["%s@%s" % c for c in CASES]


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def anchor_overlap(a_bev, b_bev):
    out = torch.zeros((a_bev.shape[0], b_bev.shape[0]), dtype=torch.float32, device=a_bev.device)
    iou3d_cuda.boxes_overlap_bev_gpu(a_bev.contiguous(), b_bev.contiguous(), out)
    return out


def anchor_iou(a_bev, b_bev):
    out = torch.zeros((a_bev.shape[0], b_bev.shape[0]), dtype=torch.float32, device=a_bev.device)
    iou3d_cuda.boxes_iou_bev_gpu(a_bev.contiguous(), b_bev.contiguous(), out)
    return out


def same(x, y):
    """bit-identical, NaN payloads aside"""
    x, y = x.cpu().numpy(), y.cpu().numpy()
    return x.shape == y.shape and bool(((x == y) | (np.isnan(x) & np.isnan(y))).all())


def _differing(x, y):
    x, y = x.cpu().numpy(), y.cpu().numpy()
    return int((~((x == y) | (np.isnan(x) & np.isnan(y)))).sum())


@pytest.fixture(scope="module")
def fams():
    return {c: I.family(c[0], c[1], N, SEED) for c in CASES}


# ------------------------------------------------------------------------------------------------ the anchor
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_anchor_bound_and_reference_parity(cuda, fams, case):
    a7, b7 = fams[case]
    a, b = I.to_bev(a7), I.to_bev(b7)
    ta, tb = T(a, cuda), T(b, cuda)
    ov, iou = anchor_overlap(ta, tb), anchor_iou(ta, tb)
    diag = ov.diagonal().cpu().numpy()
    cond = I.conditioning(a, b)
    w = ~cond["ill"]
    if w.any():
        ok, ratio, bad = I.check(diag[w], I.exact_overlap(a, b)[w], I.bound(a[w], b[w], cond["R"][w]))
        print("%s@%s: %d well-conditioned pairs, max err/bound %.4f" % (case + (w.sum(), ratio)))
        assert ok, "%d well-conditioned pairs outside the bound (max err/bound %.3g)" % (bad, ratio)
    if case[0] not in I.ILL:
        assert w.mean() > 0.9
    if HAVE_REF:
        ref_ov, ref_iou = R.boxes_overlap_bev(ta, tb), R.boxes_iou_bev(ta, tb)
        assert _differing(ov, ref_ov) == 0, "%d overlap entries differ from the reference kernel" % _differing(ov, ref_ov)
        assert _differing(iou, ref_iou) == 0, "%d IoU entries differ from the reference kernel" % _differing(iou, ref_iou)


def test_identical_boxes_at_far_range_pin(cuda):
    """as in the reference: some identical boxes overlap themselves by less than their area at far range, none near the
    origin (20000 seeded boxes per placement, aligned 3D IoU of each box with itself)"""
    for place in I.PLACES:
        a7 = I.family("identical", place, 20000, SEED)[0]
        ta = T(a7, cuda)
        iou = iou3d_cuda.boxes_iou3d_aligned(ta, ta).cpu().numpy()
        short = iou < 1 - 1e-3
        print("identical@%s on the device: %d of %d boxes with IoU(a, a) < 1, smallest %.3g" % (place, short.sum(), len(iou), iou.min()))
        assert short.any() == (place == "far")
        if HAVE_REF:
            bev = T(I.to_bev(a7[:2048]), cuda)
            assert same(anchor_overlap(bev, bev), R.boxes_overlap_bev(bev, bev))


# ------------------------------------------------------------------------------------------------ fused 3D IoU
@pytest.mark.parametrize("place", I.PLACES)
def test_iou3d_matrix_batched_aligned_equal_the_anchor_formula(cuda, fams, place):
    names = [f for f in I.FAMILIES if f != "nonfinite"]
    A = np.stack([fams[(f, place)][0] for f in names])             # (families, N, 7): one batch entry per family
    B = np.stack([fams[(f, place)][1] for f in names])
    ta, tb = T(A, cuda), T(B, cuda)
    batched = iou3d_cuda.boxes_iou3d(ta, tb)
    for k, f in enumerate(names):
        mirror = iou3d_utils.boxes_iou3d_gpu(ta[k], tb[k])         # the anchor overlap + boxes_iou3d_gpu's torch ops
        single = iou3d_cuda.boxes_iou3d(ta[k], tb[k])
        aligned = iou3d_cuda.boxes_iou3d_aligned(ta[k], tb[k])
        assert same(batched[k], single) and same(aligned, single.diagonal()), f
        assert same(single, mirror), "%s@%s: fused 3D IoU differs from the anchor formula on %d of %d entries" % (
            f, place, _differing(single, mirror), N * N)
    a7, b7 = fams[("nonfinite", place)]                           # a NaN or Inf field: NaN where torch gives NaN
    ta, tb = T(a7, cuda), T(b7, cuda)
    mirror = iou3d_utils.boxes_iou3d_gpu(ta, tb)
    assert torch.isnan(mirror.diagonal()).any()
    assert same(iou3d_cuda.boxes_iou3d(ta, tb), mirror)
    assert same(iou3d_cuda.boxes_iou3d_aligned(ta, tb), mirror.diagonal())


# ------------------------------------------------------------------------------------------------ bitmask NMS
def _interleaved(fams, place, names):
    """a box set where each box is followed by its pair partner: duplicates and near-duplicates sit next to each other"""
    out = []
    for f in names:
        a7, b7 = fams[(f, place)]
        out.append(np.stack([I.to_bev(a7)[:64], I.to_bev(b7)[:64]], 1).reshape(-1, 5))
    return np.ascontiguousarray(np.concatenate(out))


def _expected_mask(iou, thresh):
    n = iou.shape[0]
    hit = np.triu(iou > np.float32(thresh), 1)
    cb = (n + 63) // 64
    pad = np.zeros((n, cb * 64), bool)
    pad[:, :n] = hit
    bits = pad.reshape(n, cb, 64).astype(np.uint64) << np.arange(64, dtype=np.uint64)
    return np.bitwise_or.reduce(bits, axis=2)


@pytest.mark.parametrize("thresh", [0.1, 0.7, 0.8, 0.85])
@pytest.mark.parametrize("normal", [0, 1])
def test_nms_mask_is_the_anchor_iou_over_the_threshold(cuda, fams, thresh, normal):
    names = [f for f in I.FAMILIES if f != "nonfinite"]
    for place in I.PLACES:
        boxes = _interleaved(fams, place, names)
        tb = T(boxes, cuda)
        n = boxes.shape[0]
        mask = torch.zeros((n, (n + 63) // 64), dtype=torch.int64, device=cuda)
        C.check(C.lib().prb_nms_mask(C.ptr(tb), n, C.c_float(thresh), normal, C.ptr(mask), C.stream()), "nms_mask")
        got = mask.cpu().numpy().view(np.uint64)
        if normal:      # the axis-aligned IoU has no transcendental: the CPU oracle is the anchor
            want = O.nms_mask(boxes, thresh, normal=True)
            rows = np.arange(n)[:, None] // 64
            upper = np.arange(got.shape[1])[None, :] >= rows
            assert np.array_equal(got[upper], want[upper])
        else:
            want = _expected_mask(anchor_iou(tb, tb).cpu().numpy(), thresh)
            assert np.array_equal(got, want), "%s: %d mask words differ from the anchor IoU" % (place, (got != want).sum())
        keep = torch.zeros(n, dtype=torch.int64)
        num = (iou3d_cuda.nms_normal_gpu if normal else iou3d_cuda.nms_gpu)(tb, keep, thresh)
        assert np.array_equal(keep[:num].numpy(), O.nms_scan(got))


# ------------------------------------------------------------------------------------------------ proposal NMS
def _greedy(iou, thresh):
    kept = []
    for i in range(iou.shape[0]):
        if all(iou[k, i] <= np.float32(thresh) for k in kept):
            kept.append(i)
    return kept


@pytest.mark.parametrize("thresh", [0.1, 0.7, 0.85])
def test_proposal_nms_keeps_the_greedy_scan_over_the_anchor(cuda, fams, thresh):
    """the proposal kernel's in-kernel NMS goes through the plain box_overlap (iou_bev), not the precomputed one: its keep
    list must still be the greedy scan over the anchor IoU, on exact duplicates with distinct scores and near-duplicates"""
    names = ["identical", "shifted", "rotated", "flipped", "square90", "nested", "generic"]
    scenes = []
    for place in I.PLACES:
        rows = [np.stack([fams[(f, place)][0][:48], fams[(f, place)][1][:48]], 1).reshape(-1, 7) for f in names]
        scenes.append(np.concatenate(rows))
    boxes = np.ascontiguousarray(np.stack(scenes))                    # (2, n, 7)
    b, n = boxes.shape[:2]
    rng = np.random.default_rng(3)
    scores = np.stack([1.0 + rng.permutation(n) / n for _ in range(b)]).astype(np.float32)
    tbx, tsc = T(boxes, cuda), T(scores, cuda)
    order = torch.sort(tsc, dim=1, descending=True)[1].contiguous()
    out_b = torch.zeros((b, n, 7), device=cuda)
    out_s = torch.zeros((b, n), device=cuda)
    ws = torch.empty(C.lib().prb_rpn_proposals_workspace_bytes(b, n), dtype=torch.uint8, device=cuda)
    C.check(C.lib().prb_rpn_proposals(b, n, C.ptr(tbx), C.ptr(tsc), C.ptr(order), 0, n, n, C.c_float(thresh), 0, C.ptr(out_b),
                                      C.ptr(out_s), C.ptr(ws), C.c_size_t(ws.numel()), C.stream()), "rpn_proposals")
    got_s = out_s.cpu().numpy()
    for s in range(b):
        o = order[s].cpu().numpy()
        bev = T(I.to_bev(boxes[s][o]), cuda)
        want = _greedy(anchor_iou(bev, bev).cpu().numpy(), thresh)
        pos = {float(v): k for k, v in enumerate(scores[s][o])}
        got = [pos[float(v)] for v in got_s[s] if v != 0]
        assert got == want, "scene %d: keep list of %d differs from the anchor's greedy scan of %d" % (s, len(got), len(want))


# ------------------------------------------------------------------------------------------------ recall statistics
@pytest.mark.parametrize("place", I.PLACES)
def test_eval_recall_equals_the_anchor_iou3d(cuda, fams, place):
    """one scene per pair (box a, GT b): each box's max IoU is the anchor's 3D IoU, and the recall count at every
    threshold is the number of anchor IoUs above it (a NaN IoU, from a non-finite box, is the max and recalls nothing)"""
    a7 = np.concatenate([fams[(f, place)][0] for f in I.FAMILIES])
    b7 = np.concatenate([fams[(f, place)][1] for f in I.FAMILIES])
    n = len(a7)
    ta, tb = T(a7, cuda), T(b7, cuda)
    want = iou3d_utils.boxes_iou3d_gpu(ta, tb).diagonal().contiguous()
    thresh = np.array([0.1, 0.25, 0.5, 0.7, 0.9, 0.99], np.float32)
    recalled = torch.zeros(len(thresh), dtype=torch.int64, device=cuda)
    total = torch.zeros(1, dtype=torch.int64, device=cuda)
    box_max = torch.full((n,), float("nan"), device=cuda)
    ones = torch.ones(n, dtype=torch.int32, device=cuda)
    C.check(C.lib().prb_eval_box_recall(n, 1, C.ptr(ta), None, 1, C.ptr(tb), C.ptr(ones), len(thresh),
                                        thresh.ctypes.data_as(C.ctypes.POINTER(C.c_float)), C.ptr(recalled), C.ptr(total),
                                        C.ptr(box_max), C.stream()), "eval_box_recall")
    assert same(box_max, want)
    w = want.cpu().numpy()
    assert recalled.cpu().tolist() == [int((w > t).sum()) for t in thresh]
    assert int(total.item()) == n


# ------------------------------------------------------------------------------------------------ scratch isolation
def test_sentinel_outputs_and_neighbour_independence(cuda, fams):
    """NaN-prefilled outputs with a guard behind them: nothing is written out of range, and a pair's value is the same
    alone as in a 128 x 128 tile of ill-conditioned neighbours (the polygon scratch columns are per thread)"""
    ill = [f for f in I.ILL if f != "nonfinite"]
    a7 = np.concatenate([fams[(f, "far")][0][:16] for f in ill])[:128]
    b7 = np.concatenate([fams[(f, "far")][1][:16] for f in ill])[:128]
    a, b = I.to_bev(a7), I.to_bev(b7)
    ta, tb = T(a, cuda), T(b, cuda)
    n, G = 128, 4096
    for fn in (C.lib().prb_boxes_overlap_bev, C.lib().prb_boxes_iou_bev):
        buf = torch.full((n * n + G,), float("nan"), device=cuda)
        C.check(fn(n, C.ptr(ta), n, C.ptr(tb), C.ptr(buf), C.stream()), "pair matrix")
        tile = buf[: n * n].view(n, n)
        assert not torch.isnan(tile).any() and torch.isnan(buf[n * n:]).all()
        one = torch.full((1 + G,), float("nan"), device=cuda)
        for i in range(0, n, 9):
            C.check(fn(1, C.ptr(ta[i:i + 1]), 1, C.ptr(tb[i:i + 1]), C.ptr(one), C.stream()), "pair matrix")
            assert same(one[:1], tile[i, i:i + 1]) and torch.isnan(one[1:]).all()
    t7a, t7b = T(a7, cuda), T(b7, cuda)
    buf = torch.full((n * n + G,), float("nan"), device=cuda)
    C.check(C.lib().prb_boxes_iou3d(1, n, C.ptr(t7a), n, C.ptr(t7b), C.ptr(buf), C.stream()), "boxes_iou3d")
    assert torch.isnan(buf[n * n:]).all() and not torch.isnan(buf[: n * n]).any()
    al = torch.full((n + G,), float("nan"), device=cuda)
    C.check(C.lib().prb_boxes_iou3d_aligned(n, C.ptr(t7a), C.ptr(t7b), C.ptr(al), C.stream()), "boxes_iou3d_aligned")
    assert torch.isnan(al[n:]).all() and same(al[:n], buf[: n * n].view(n, n).diagonal())

"""The RPN proposal layer on the device (csrc/proposal.cu) on the edge families of proposal_reference.py, bit for bit
against oracle/proposal.py, at B = 16 x 16384 with every scene from another family, and at small sizes and quotas.

The oracle is fed the device's own torch.sort order, so tied scores test the kernel and not the sort.  Its NMS is the
CPU oracle's for the axis-aligned IoU (plain fp32 arithmetic) and, for the rotated one, the greedy scan over the
device's BEV IoU matrix kernel (the anchor that test_gpu_iou_geometry.py pins to the reference's own kernel) or, when
oracle/_ref is built, the reference's own NMS kernel and host scan."""
import numpy as np
import pytest
import torch

import iou_reference as I
import proposal_reference as PR
from oracle import oracle as O
from oracle import proposal as P
from oracle import refgpu as R

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200.rpn.proposal_layer import ProposalLayer, decode_rpn_proposals  # noqa: E402

SERVERS = ["anchor", "reference"]
SENTINEL = np.array([0x7fa5a5a5], np.int32).view(np.float32)[0]        # a NaN payload no kernel produces


def T(a, dev="cuda:0"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def bits(a):
    """int32 patterns with every NaN mapped to one canonical NaN (device and numpy NaN payloads differ)"""
    a = np.array(a.cpu().numpy() if torch.is_tensor(a) else a, dtype=np.float32)
    a[np.isnan(a)] = np.float32("nan")
    return a.view(np.int32)


def _differing_rows(got, want):
    g, w = bits(got), bits(want)
    return int((g != w).reshape(g.shape[0], -1).any(1).sum()) if g.ndim > 1 else int((g != w).sum())


def _cfg(mode):
    import types
    m = PR.MODES[mode]
    ns = types.SimpleNamespace
    stage = ns(RPN_PRE_NMS_TOP_N=m["pre_nms_top_n"], RPN_POST_NMS_TOP_N=m["post_nms_top_n"], RPN_NMS_THRESH=m["nms_thresh"],
               RPN_DISTANCE_BASED_PROPOSE=m["distance_based"])

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    c = Cfg(TEST=stage, TRAIN=stage)
    c["CLS_MEAN_SIZE"] = PR.ANCHOR[None]
    c["RPN"] = ns(LOC_SCOPE=3.0, LOC_BIN_SIZE=0.5, NUM_HEAD_BIN=12, LOC_XZ_FINE=True, NMS_TYPE=m["nms_type"])
    return c


def _nms_server(server):
    def nms(boxes_bev, scores, thresh, nms_type):
        order = P.descending(scores)
        b = np.ascontiguousarray(boxes_bev[order])
        if b.shape[0] == 0:
            return order
        if nms_type == "normal":
            keep = O.nms(b, thresh, normal=True)
        elif server == "anchor":
            t = T(b)
            keep = I.greedy(I.anchor_iou(t, t).cpu().numpy(), thresh)
        else:
            keep = R.nms(T(b), float(thresh), normal=False).numpy()
        return order[np.asarray(keep, np.int64)]
    return nms


def _device(scores, reg, xyz, mode, **quota):
    cfg = _cfg(mode)
    for k, v in quota.items():
        setattr(cfg.TEST, k, v)
    layer = ProposalLayer(mode="TEST", cfg=cfg)
    ts = T(scores)
    b, s = layer(ts, T(reg), T(xyz))
    order = torch.sort(ts, dim=1, descending=True)[1].cpu().numpy()        # the layer's own call (proposal_layer.py:36)
    return b, s, order


def _oracle(scores, reg, xyz, mode, order, **over):
    kw = dict(PR.MODES[mode], **over)
    return P.proposal_layer(scores, reg, xyz, PR.ANCHOR, order=order, near_empty="far_only", **kw)


def _check(got_b, got_s, want_b, want_s, what):
    assert tuple(got_b.shape) == want_b.shape and tuple(got_s.shape) == want_s.shape
    for s in range(want_s.shape[0]):
        nb, ns = _differing_rows(got_b[s], want_b[s]), _differing_rows(got_s[s], want_s[s])
        assert nb == 0 and ns == 0, "%s scene %d: %d box rows and %d scores differ from the oracle" % (what, s, nb, ns)


@pytest.fixture(scope="module")
def batches():
    return [PR.batch(k) for k in range(len(PR.BATCHES))]


# ------------------------------------------------------------------------------------------------ decode
@pytest.mark.parametrize("k", range(len(PR.BATCHES)))
def test_decode_bit_exact_on_every_family(cuda, batches, k):
    scores, reg, xyz = batches[k]
    got = decode_rpn_proposals(T(xyz), T(reg), PR.ANCHOR, 3.0, 0.5, 12, True).reshape(-1, 7)
    want = P.decode_bbox_target(xyz.reshape(-1, 3), reg.reshape(-1, PR.C), PR.ANCHOR, 3.0, 0.5, 12, True)
    want[:, 1] = want[:, 1] + want[:, 3] / np.float32(2)                   # proposal_layer.py:32, fused into the kernel
    bad = (bits(got) != bits(want)).any(1).reshape(len(PR.BATCHES[k]), -1)
    for s, (f, v) in enumerate(PR.BATCHES[k]):
        assert not bad[s].any(), "%s/%s: %d decoded boxes differ from the oracle, first row %d" % (
            f, v, bad[s].sum(), int(np.argmax(bad[s])))


def test_cuda_argmax_picks_the_oracles_bins(cuda):
    """torch.argmax on CUDA takes the first NaN, as torch on the CPU and np.argmax do: the rule the decode follows"""
    _, reg, _ = PR.scene("argmax_edges", n=2048, seed=5)
    for lo in (PR.XB, PR.ZB, PR.HB):
        g = reg[:, lo:lo + PR.NB]
        assert np.array_equal(torch.argmax(T(g), dim=1).cpu().numpy(), np.argmax(g, axis=1))


# ------------------------------------------------------------------------------------------------ the whole layer
@pytest.mark.parametrize("server", SERVERS)
@pytest.mark.parametrize("mode", list(PR.MODES))
@pytest.mark.parametrize("k", range(len(PR.BATCHES)))
def test_layer_bit_exact_at_batch_16(cuda, batches, k, mode, server, monkeypatch):
    if server == "reference" and (PR.MODES[mode]["nms_type"] == "normal" or not R.available()):
        pytest.skip("the reference's NMS kernel serves the rotated modes, where oracle/_ref is built")
    scores, reg, xyz = batches[k]
    b, s, order = _device(scores, reg, xyz, mode)
    monkeypatch.setattr(P, "_nms", _nms_server(server))
    want_b, want_s = _oracle(scores, reg, xyz, mode, order)
    _check(b, s, want_b, want_s, "%s batch %d" % (mode, k))


SIZE_SCENES = [("nms_clusters", "dense"), ("non_finite", ""), ("range_edges", "")]


@pytest.mark.parametrize("n", [1, 33, 1000, 16383, 16384])
@pytest.mark.parametrize("mode", ["test_normal", "score_based"])
def test_layer_bit_exact_at_small_sizes(cuda, n, mode, monkeypatch):
    rows = [PR.scene(f, v, n, 40 + i) for i, (f, v) in enumerate(SIZE_SCENES)]
    scores, reg, xyz = (np.stack([r[i] for r in rows]) for i in range(3))
    monkeypatch.setattr(P, "_nms", _nms_server("anchor"))
    b, s, order = _device(scores, reg, xyz, mode)
    _check(b, s, *_oracle(scores, reg, xyz, mode, order), "%s n=%d" % (mode, n))


@pytest.mark.parametrize("pre,post", [(20000, 100), (1, 1), (2, 2), (1, 2), (2, 1), (3, 7)])
@pytest.mark.parametrize("mode", ["test_normal", "test_rotate", "score_based"])
def test_layer_bit_exact_at_small_quotas(cuda, batches, pre, post, mode, monkeypatch):
    """pre_nms_top_n above N, and quotas where int(post * 0.7) or int(pre * 0.7) is 0"""
    scores, reg, xyz = batches[1]
    monkeypatch.setattr(P, "_nms", _nms_server("anchor"))
    b, s, order = _device(scores, reg, xyz, mode, RPN_PRE_NMS_TOP_N=pre, RPN_POST_NMS_TOP_N=post)
    _check(b, s, *_oracle(scores, reg, xyz, mode, order, pre_nms_top_n=pre, post_nms_top_n=post), "%s %d/%d" % (mode, pre, post))


# ------------------------------------------------------------------------------------------------ the C ABI
def _abi(b, n, boxes, scores, order, dist, pre, post, out_b, out_s, ws, wsb, normal=1):
    return C.lib().prb_rpn_proposals(b, n, C.ptr(boxes), C.ptr(scores), C.ptr(order), dist, pre, post, C.c_float(0.8), normal,
                                     C.ptr(out_b), C.ptr(out_s), C.ptr(ws), C.c_size_t(wsb), C.stream())


def _decoded(batches, k=0):
    scores, reg, xyz = batches[k]
    ts = T(scores)
    boxes = decode_rpn_proposals(T(xyz), T(reg), PR.ANCHOR, 3.0, 0.5, 12, True)
    return boxes, ts, torch.sort(ts, dim=1, descending=True)[1].contiguous()


@pytest.mark.parametrize("dist,pre,post", [(1, 9000, 100), (1, 9000, 512), (0, 9000, 100), (1, 3, 1)])
def test_abi_writes_every_row_and_nothing_past_the_end(cuda, batches, dist, pre, post):
    """outputs prefilled with a NaN sentinel and followed by guard words; the workspace exactly
    prb_rpn_proposals_workspace_bytes.  Every row is written (survivors, then zeros), nothing behind the last"""
    boxes, scores, order = _decoded(batches)
    B, n = scores.shape
    G = 4096
    out_b = torch.full((B * post * 7 + G,), float(SENTINEL), device=cuda)
    out_s = torch.full((B * post + G,), float(SENTINEL), device=cuda)
    out_b.view(torch.int32).fill_(int(np.float32(SENTINEL).view(np.int32)))
    out_s.view(torch.int32).fill_(int(np.float32(SENTINEL).view(np.int32)))
    wsb = C.lib().prb_rpn_proposals_workspace_bytes(B, post)
    ws = torch.empty(wsb, dtype=torch.uint8, device=cuda)
    C.check(_abi(B, n, boxes, scores, order, dist, pre, post, out_b, out_s, ws, wsb), "rpn_proposals")
    sent = int(np.float32(SENTINEL).view(np.int32))
    for out, rows in ((out_b, B * post * 7), (out_s, B * post)):
        w = out.view(torch.int32).cpu().numpy()
        assert (w[:rows] != sent).all(), "%d output words never written" % (w[:rows] == sent).sum()
        assert (w[rows:] == sent).all(), "%d guard words overwritten" % (w[rows:] != sent).sum()


def test_abi_batch_zero_and_shared_memory_refusal(cuda, batches):
    """b = 0 returns without a launch; quotas whose lists need more than 200 KB of shared memory (4 bytes per candidate,
    8 in the far range, 68 per kept box, 48 KB of polygon scratch) are refused before anything is written; the largest
    accepted ones run and equal the oracle"""
    boxes, scores, order = _decoded(batches, 1)
    B, n = scores.shape
    sent = int(np.float32(SENTINEL).view(np.int32))
    out_b = torch.empty((B * 100 * 7,), dtype=torch.int32, device=cuda).fill_(sent).view(torch.float32)
    out_s = torch.empty((B * 100,), dtype=torch.int32, device=cuda).fill_(sent).view(torch.float32)
    wsb = C.lib().prb_rpn_proposals_workspace_bytes(B, 100)
    ws = torch.empty(wsb, dtype=torch.uint8, device=cuda)
    assert _abi(0, n, boxes, scores, order, 1, 9000, 100, out_b, out_s, ws, wsb) == 0
    # score based: 4 pre + 68 * 100 + 49152 <= 204800 up to pre 37212; distance based: area 0 (int(0.7 pre) candidates)
    # is the larger, up to pre 53889
    for dist, last in ((0, 37212), (1, 53889)):
        assert _abi(B, n, boxes, scores, order, dist, last + 1, 100, out_b, out_s, ws, wsb) != 0
        assert "shared memory" in C.lib().prb_last_error().decode()
        torch.cuda.synchronize()
        assert (out_b.view(torch.int32) == sent).all() and (out_s.view(torch.int32) == sent).all(), "a refused call wrote"
    C.check(_abi(B, n, boxes, scores, order, 1, 53889, 100, out_b, out_s, ws, wsb), "rpn_proposals")
    s_np, r_np, x_np = batches[1]
    want_b, want_s = P.proposal_layer(s_np, r_np, x_np, PR.ANCHOR, pre_nms_top_n=53889, post_nms_top_n=100, nms_thresh=0.8,
                                      nms_type="normal", order=order.cpu().numpy(), near_empty="far_only")
    _check(out_b.view(B, 100, 7), out_s.view(B, 100), want_b, want_s, "pre 53889")


# ------------------------------------------------------------------------------------------------ determinism, no host sync
@pytest.mark.parametrize("mode", ["test_rotate", "train_normal"])
def test_repeatable_and_free_of_host_synchronisation_on_a_side_stream(cuda, batches, mode):
    scores, reg, xyz = batches[0]
    ts, tr, tx = T(scores), T(reg), T(xyz)
    layer = ProposalLayer(mode="TEST", cfg=_cfg(mode))
    ref_b, ref_s = layer(ts, tr, tx)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda.set_sync_debug_mode("error")
        try:
            b1, s1 = layer(ts, tr, tx)
            b2, s2 = layer(ts, tr, tx)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    side.synchronize()
    for got in (b1, b2):
        assert np.array_equal(bits(got), bits(ref_b))
    for got in (s1, s2):
        assert np.array_equal(bits(got), bits(ref_s))

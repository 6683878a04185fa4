"""The device SA training path (csrc/sa_train.cu) bit for bit on integer-valued inputs, at every row split it has.

On the cases of sa_train_reference.integer_case every TF32 conversion and every fp32 product and partial sum is exact in
any order (check_exact asserts it per case), so Z, the outputs, the chosen samples, dW, dbias and the atomically
scattered feature gradient each have exactly one right answer, and the float64 reference computes it -- on the GPU at
the training sizes.  Floats are compared as int32 bit patterns after adding +0.0 (which maps -0.0 to +0.0 and leaves
every other value, NaN included, as it is): the sign of an exact zero is not part of the answer.

- the C ABI directly on bias-only chains (the RCNN layout) over a matrix of widths, feature counts, depths, sample counts
  and row counts around the 32-wide K chunks, the 64-column tiles and the 128-row tiles, with the output buffers'
  channel slice, guard words, a NULL out_pm, an accumulated feature gradient and a skipped scatter;
- the training shapes: RPN SA1 (16 x 4096 centres, 16 and 32 samples: 16384 row tiles, the statistics parts at their cap
  of 1024 with 64 groups each, about 525 weight-gradient chunks), as bias chains and as the BN chains it trains with
  (layer 0's statistics against a float64 replay of its exact sums), RCNN SA1 at 32768 groups, 32770 groups (a last
  statistics part of one group), RCNN SA3 (GroupAll);
- the module path (PointnetSAModuleMSG through _forward_train, both scales into one output and one feature gradient);
- non-finite features against the torch path: NaN and +-Inf reach the same outputs and running statistics."""
import copy
import ctypes
import time

import pytest
import torch

import sa_train_reference as R
from pointrcnn_b200 import _cabi as C
from pointrcnn_b200 import config
from pointrcnn_b200.pointnet2 import sa_train
from pointrcnn_b200.pointnet2.pointnet2_modules import PointnetSAModule, PointnetSAModuleMSG

pytestmark = pytest.mark.gpu

SENTINEL = -7.0     # every word of out / out_pm outside the channel slice keeps it
GUARD = 64          # words behind each output buffer
OTHER_GRAD = 1000.0  # grad_out outside the channel slice: a read of it would change the gradients


def _bits(t):
    return (t.float() + 0.0).view(torch.int32)


def _assert_bits(got, want, what):
    g, w = _bits(got.contiguous()), _bits(want.to(got.device).float().contiguous())
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = int((g != w).sum())
    assert bad == 0, "%s differs in %d of %d words (first at %s)" % (what, bad, g.numel(), (g != w).nonzero()[0].tolist())


def _ptrs(ts):
    return (ctypes.c_void_p * 3)(*[None if t is None else t.data_ptr() for t in ts] + [None] * (3 - len(ts)))


def run_cabi(case, cuda, stride_extra=5, c_off=3, with_pm=True, grad_feats="prefill", backward=True):
    """prb_sa_train_forward + prb_sa_train_backward on `case` (integer_case's form) -> dict of the device results.
    out / out_pm have stride_extra channels more than the chain writes, at offset c_off, sentinel-filled, with GUARD
    words behind; grad_out carries OTHER_GRAD outside the slice.  grad_feats: "prefill" (integers the backward must add
    to), "null" (NULL: no scatter), or None (c_feat = 0)."""
    L = C.lib()
    layers = case["layers"]
    bn = "gamma" in layers[0]
    xyz, centres = case["xyz"].to(cuda), case["centres"].to(cuda)
    idx = case["idx"].to(cuda)
    B, N, _ = xyz.shape
    _, P, ns = idx.shape
    feats = case["feats"]
    c_feat = 0 if feats is None else feats.shape[1]
    feats_pm = None if feats is None else feats.to(cuda).transpose(1, 2).contiguous()
    widths = [d["w"].shape[0] for d in layers]
    Cl = widths[-1]
    stride = Cl + stride_extra
    dev_layers = []
    d = C.SATrainDesc()
    d.num_layers, d.c_in, d.bn = len(layers), 3 + c_feat, int(bn)
    for l, lay in enumerate(layers):
        t = dict(w=lay["w"].float().to(cuda).contiguous())
        d.c_out[l] = widths[l]
        d.weight[l] = t["w"].data_ptr()
        if bn:
            t.update(gamma=lay["gamma"].float().to(cuda), beta=lay["beta"].float().to(cuda), rm=lay["rm"].float().to(cuda),
                     rv=lay["rv"].float().to(cuda), nbt=torch.full((1,), lay["nbt"], dtype=torch.int64, device=cuda))
            d.eps, d.momentum = lay["eps"], lay["momentum"]
            d.gamma[l], d.beta[l] = t["gamma"].data_ptr(), t["beta"].data_ptr()
            d.running_mean[l], d.running_var[l] = t["rm"].data_ptr(), t["rv"].data_ptr()
            d.num_batches_tracked[l] = t["nbt"].data_ptr()
        else:
            t["b"] = lay["b"].float().to(cuda)
            d.bias[l] = t["b"].data_ptr()
        dev_layers.append(t)
    rows = B * P * ns
    z = [torch.empty((rows, c), dtype=torch.float32, device=cuda) for c in widths]
    stats = torch.empty((len(widths), sa_train.STAT_ROWS, sa_train.MAX_WIDTH), dtype=torch.float32, device=cuda)
    chosen = torch.empty((B * P, Cl), dtype=torch.uint8, device=cuda)
    out_buf = torch.full((B * stride * P + GUARD,), SENTINEL, device=cuda)
    pm_buf = torch.full((B * P * stride + GUARD,), SENTINEL, device=cuda) if with_pm else None
    out = out_buf[:B * stride * P].view(B, stride, P)
    out_pm = pm_buf[:B * P * stride].view(B, P, stride) if with_pm else None
    stream = C.stream()
    ws = torch.empty(max(L.prb_sa_train_workspace_bytes(B, P, ns, c_feat, ctypes.byref(d), int(backward)), 1), dtype=torch.uint8, device=cuda)
    C.check(L.prb_sa_train_forward(ctypes.byref(d), B, N, P, ns, c_feat, C.ptr(xyz), C.ptr(centres), C.ptr(feats_pm), C.ptr(idx),
                                   _ptrs(z), C.ptr(stats), C.ptr(chosen), C.ptr(out), C.ptr(out_pm), stride, c_off, C.ptr(ws),
                                   ws.numel(), stream), "sa_train_forward")
    res = dict(z=z, stats=stats, chosen=chosen, out_buf=out_buf, pm_buf=pm_buf, out=out, out_pm=out_pm, stride=stride,
               c_off=c_off, layers=dev_layers)
    if not backward:
        return res
    gout = torch.full((B, stride, P), OTHER_GRAD, device=cuda)
    gout[:, c_off:c_off + Cl] = case["grad_out"].to(cuda)
    gw = [torch.full_like(t["w"], SENTINEL) for t in dev_layers]
    gb = [torch.full_like(t["b"], SENTINEL) if "b" in t else None for t in dev_layers]
    gf = prefill = None
    if grad_feats == "prefill":
        prefill = torch.randint(-50, 51, (B, c_feat, N), generator=torch.Generator().manual_seed(5)).float()
        gf = prefill.to(cuda)
    C.check(L.prb_sa_train_backward(ctypes.byref(d), B, N, P, ns, c_feat, C.ptr(xyz), C.ptr(centres), C.ptr(feats_pm), C.ptr(idx),
                                    _ptrs(z), C.ptr(stats), C.ptr(chosen), C.ptr(gout), stride, c_off, _ptrs(gw),
                                    _ptrs(gb) if not bn else None, None, None, C.ptr(gf), C.ptr(ws), ws.numel(), stream),
            "sa_train_backward")
    res.update(gw=gw, gb=gb, gf=gf, prefill=prefill)
    return res


def first_max(pre, groups):
    """the sample the device records: the first maximal pre-activation of every (group, channel)"""
    return pre.view(groups, -1, pre.shape[1]).argmax(1)


def ties_among_distinct_points(case, pre, cuda):
    """(group, channel) pairs whose maximum is reached by two or more different points"""
    idx = case["idx"].to(cuda).long()
    G = idx.shape[0] * idx.shape[1]
    y = pre.view(G, -1, pre.shape[1])
    at_max = y == y.max(1, keepdim=True).values
    pts = idx.view(G, -1, 1).expand_as(y)
    lo = torch.where(at_max, pts, torch.full_like(pts, 1 << 30)).min(1).values
    hi = torch.where(at_max, pts, torch.full_like(pts, -1)).max(1).values
    return int((lo != hi).sum())


def check_bias_chain(case, got, cuda):
    """every result of run_cabi on a bias chain against the float64 reference, bit for bit; returns a short summary"""
    ref = R.scale(case["xyz"], case["centres"], case["feats"], case["idx"], case["layers"], case["grad_out"], device=cuda)
    prefill = got.get("prefill")
    R.check_exact(case, ref, grad_feats_prefill=prefill)
    layers = case["layers"]
    B, P = case["idx"].shape[:2]
    Cl, stride, off = layers[-1]["w"].shape[0], got["stride"], got["c_off"]
    for l, lay in enumerate(layers):
        _assert_bits(got["z"][l], ref["pre"][l] - lay["b"].to(cuda), "Z%d" % l)
    want_chosen = first_max(ref["pre"][-1], B * P)
    assert torch.equal(got["chosen"].long(), want_chosen), "chosen differs in %d places" % int((got["chosen"].long() != want_chosen).sum())
    out = got["out"]
    _assert_bits(out[:, off:off + Cl], ref["out"], "out")
    assert (_bits(out[:, :off]) == _bits(torch.tensor(SENTINEL))).all() and (_bits(out[:, off + Cl:]) == _bits(torch.tensor(SENTINEL))).all(), \
        "out written outside its channel slice"
    assert (got["out_buf"][-GUARD:] == SENTINEL).all(), "out written past its end"
    if got["out_pm"] is not None:
        pm = got["out_pm"]
        _assert_bits(pm[:, :, off:off + Cl], ref["out"].transpose(1, 2), "out_pm")
        assert (pm[:, :, :off] == SENTINEL).all() and (pm[:, :, off + Cl:] == SENTINEL).all(), "out_pm written outside its slice"
        assert (got["pm_buf"][-GUARD:] == SENTINEL).all(), "out_pm written past its end"
    if "gw" not in got:
        return ""
    # the reference routes the gradient by the first maximum of the ReLU outputs; where that differs from the device's
    # first maximum of the pre-activations, the maximum is <= 0 and the ReLU drops the gradient either way
    for l in range(len(layers)):
        _assert_bits(got["gw"][l], ref["w"][l], "grad_weight%d" % l)
        _assert_bits(got["gb"][l], ref["b"][l], "grad_bias%d" % l)
    if got["gf"] is not None:
        _assert_bits(got["gf"], ref["feats"] + prefill.to(cuda).double(), "grad_feats")
    flowing = [int((dz != 0).any(1).sum()) for dz in ref["dz"]]
    assert flowing[0] > 0, "no gradient reaches layer 0: the case tests nothing"
    return "rows with gradient per layer %s, ties among distinct points %d" % (flowing, ties_among_distinct_points(case, ref["pre"][-1], cuda))


# ------------------------------------------------------------------------------------------ a. the C ABI, bias chains
CABI_CASES = [
    # B, N, npoint, ns, c_feat, widths
    (1, 40, 3, 4, 0, [1]),                        # 12 rows, under one 128-row tile; no features
    (1, 64, 8, 16, 1, [8, 24]),                   # exactly one row tile
    (2, 300, 37, 8, 29, [40, 63, 64]),            # 592 rows; c_in 32: exactly one K chunk
    (2, 200, 19, 32, 61, [65, 128]),              # c_in 64: two K chunks, one 64-column tile
    (2, 200, 9, 64, 62, [196]),                   # c_in 65: a K tail of one, a second 64-column tile of one
    (1, 300, 5, 128, 125, [384, 8]),              # c_in 128; 128 samples per centre
    (1, 600, 6, 16, 509, [512, 1, 24]),           # c_in 512; a one-wide inner layer
    (2, 100, 11, 4, 128, [64, 65, 40]),           # c_in 131
    (3, 500, 41, 32, 1, [16, 16, 32]),            # RPN SA1's narrow chain, 3936 rows
]


@pytest.mark.parametrize("B,N,npoint,ns,c_feat,widths", CABI_CASES)
def test_cabi_bias_chain_bits(cuda, B, N, npoint, ns, c_feat, widths):
    case = R.integer_case(B, N, npoint, ns, c_feat, widths, seed=B * 7 + ns + c_feat)
    got = run_cabi(case, cuda, grad_feats="prefill" if c_feat else None)
    print(check_bias_chain(case, got, cuda))


def test_cabi_null_out_pm_and_null_feature_gradient(cuda):
    """out_pm = NULL is accepted; grad_feats = NULL skips the scatter and leaves every other result unchanged"""
    case = R.integer_case(2, 300, 37, 8, 29, [40, 63, 64], seed=11)
    got = run_cabi(case, cuda, stride_extra=0, c_off=0, with_pm=False, grad_feats="null")
    assert got["gf"] is None
    check_bias_chain(case, got, cuda)


# ------------------------------------------------------------------------------------------ b. the training shapes
TRAIN_CASES = {
    # name: (B, N, npoint, ns, c_feat, widths, group_all)
    "rpn_sa1_ns16": (16, 16384, 4096, 16, 1, [16, 16, 32], False),
    "rpn_sa1_ns32": (16, 16384, 4096, 32, 1, [32, 32, 64], False),
    "rcnn_sa1_32768_groups": (256, 512, 128, 64, 128, [128, 128, 128], False),
    "32770_groups": (2, 20000, 16385, 4, 3, [24, 40], False),
    "rcnn_sa3_group_all": (256, 32, 1, 32, 256, [256, 256, 512], True),
}


@pytest.mark.parametrize("name", list(TRAIN_CASES))
def test_training_shape_bias_chain_bits(cuda, name):
    B, N, npoint, ns, c_feat, widths, group_all = TRAIN_CASES[name]
    t0 = time.time()
    case = R.integer_case(B, N, npoint, ns, c_feat, widths, seed=len(name), group_all=group_all)
    got = run_cabi(case, cuda)
    summary = check_bias_chain(case, got, cuda)
    torch.cuda.synchronize()
    print("%s: %s; %.1f s" % (name, summary, time.time() - t0))


def _ulps(got, want):
    """|got - want| in units of the fp32 spacing at want (float64 want)"""
    w32 = want.float()
    spacing = (torch.nextafter(w32.abs(), torch.tensor(float("inf"), device=w32.device)) - w32.abs()).double()
    return ((got.double() - want).abs() / spacing).max().item()


@pytest.mark.parametrize("name", ["rpn_sa1_ns16", "rpn_sa1_ns32"])
def test_training_shape_bn_chain_layer0_statistics(cuda, name):
    """the chains RPN SA1 trains with: Z0 is exact; layer 0's mean, invstd, a, b and running statistics are within one
    fp32 ulp of a float64 replay of its exact column sums; num_batches_tracked of every layer goes up by one"""
    B, N, npoint, ns, c_feat, widths, _ = TRAIN_CASES[name]
    case = R.integer_case(B, N, npoint, ns, c_feat, widths, seed=len(name), bn=True)
    ref = R.scale(case["xyz"], case["centres"], case["feats"], case["idx"], case["layers"][:1], device=cuda)
    R.check_exact(case, ref, layers_exact=1)
    got = run_cabi(case, cuda, backward=False)
    a0 = R.rows0(case["xyz"], case["centres"], case["feats"], case["idx"], cuda)
    lay = case["layers"][0]
    z = a0 @ lay["w"].to(cuda).t()
    _assert_bits(got["z"][0], z, "Z0")
    n = z.shape[0]
    s1, s2 = z.sum(0), (z * z).sum(0)                   # exact: integers below 2^53
    mean = s1 / n
    var = (s2 / n - mean * mean).clamp_min(0)
    invstd = 1.0 / torch.sqrt(var + lay["eps"])
    gamma, beta, rm, rv = (lay[k].float().double().to(cuda) for k in ("gamma", "beta", "rm", "rv"))   # what the device reads
    m = lay["momentum"]
    c = z.shape[1]
    st = got["stats"][0, :, :c]
    ulps = {"mean": _ulps(st[0], mean), "invstd": _ulps(st[1], invstd), "a": _ulps(st[2], gamma * invstd),
            "b": _ulps(st[3], beta - mean * gamma * invstd),
            "running_mean": _ulps(got["layers"][0]["rm"], (1 - m) * rm + m * mean),
            "running_var": _ulps(got["layers"][0]["rv"], (1 - m) * rv + m * var * n / (n - 1))}
    print("%s layer 0: largest distance in fp32 ulps %s" % (name, " ".join("%s=%.2f" % kv for kv in ulps.items())))
    assert max(ulps.values()) <= 1.0, ulps
    for t, l in zip(got["layers"], case["layers"]):
        assert int(t["nbt"]) == l["nbt"] + 1


# ------------------------------------------------------------------------------------------ c. the module path
def test_module_msg_bias_chains_bits(cuda):
    """PointnetSAModuleMSG(bn=False) with integer weights on an integer grid through _forward_train: both scales write
    one output and accumulate one feature gradient; bit for bit against the reference on the device's own indices"""
    B, N, P, c_feat = 2, 2048, 256, 2
    widths = [[16, 16, 32], [32, 32, 64]]
    m = PointnetSAModuleMSG(npoint=P, radii=[1.5, 2.5], nsamples=[16, 32], mlps=[[c_feat] + w for w in widths], bn=False).to(cuda).train()
    proto = R.integer_case(B, N, P, 16, c_feat, widths[0], seed=21)
    xyz = proto["xyz"].to(cuda)
    feats = proto["feats"].to(cuda).requires_grad_(True)
    cases, gouts = [], []
    for k, w in enumerate(widths):
        cs = R.integer_case(B, N, P, 16, c_feat, w, seed=22 + k)
        with torch.no_grad():
            for layer, lay in zip(m.mlps[k].children(), cs["layers"]):
                layer.conv.weight.copy_(lay["w"].view_as(layer.conv.weight))
                layer.conv.bias.copy_(lay["b"])
        cases.append(cs)
        gouts.append(cs["grad_out"])
    new_xyz, out = m._forward_train(xyz, feats, None)
    assert type(out.grad_fn).__name__.startswith("_SATrain")
    gout = torch.cat(gouts, 1).to(cuda)
    out.backward(gout)
    centres, idxs = m.fused_geometry(xyz, new_xyz)[1:3]
    off, gf_ref, scatter = 0, 0, 0
    for k, cs in enumerate(cases):
        case = dict(cs, xyz=xyz.cpu(), centres=centres.cpu(), feats=feats.detach().cpu(), idx=idxs[k].cpu())
        ref = R.scale(case["xyz"], case["centres"], case["feats"], case["idx"], case["layers"], case["grad_out"], device=cuda)
        scatter = scatter + R.check_exact(case, ref)
        c = widths[k][-1]
        _assert_bits(out[:, off:off + c].detach(), ref["out"], "scale %d out" % k)
        _assert_bits(out._prb_pm[0][:, :, off:off + c], ref["out"].transpose(1, 2), "scale %d out_pm" % k)
        for l, layer in enumerate(m.mlps[k].children()):
            _assert_bits(layer.conv.weight.grad.flatten(1), ref["w"][l], "scale %d grad_weight%d" % (k, l))
            _assert_bits(layer.conv.bias.grad, ref["b"][l], "scale %d grad_bias%d" % (k, l))
        gf_ref = gf_ref + ref["feats"]
        off += c
    assert scatter.max() < R.FP32_EXACT, "the two scales' feature scatters reach 2^24 together"
    _assert_bits(feats.grad, gf_ref, "grad_feats (both scales)")


# ------------------------------------------------------------------------------------------ d. non-finite features
@pytest.mark.parametrize("bn", [False, True])
@pytest.mark.parametrize("value", [float("nan"), float("inf"), float("-inf")])
def test_non_finite_features_propagate_as_on_the_torch_path(cuda, value, bn):
    """one point's features set to NaN / +-Inf: the device path's outputs and running statistics are non-finite exactly
    where the torch path's are; on a bias chain, exactly in the groups that gather that point"""
    torch.manual_seed(3)
    m = PointnetSAModuleMSG(npoint=64, radii=[0.2, 0.4], nsamples=[16, 32], mlps=[[2, 16, 32], [2, 32, 64]], bn=bn).to(cuda).train()
    g = torch.Generator().manual_seed(4)
    xyz = torch.rand(2, 1024, 3, generator=g).to(cuda)
    feats = torch.randn(2, 2, 1024, generator=g).to(cuda)
    feats[0, :, 0] = value                                 # point 0 of scene 0: the first centre of the sampling
    res = {}
    for impl in ("device", "torch"):
        mm = copy.deepcopy(m)
        f = feats.clone().requires_grad_(True)
        with config.override(sa_train=impl):
            new_xyz, out = mm(xyz, f)
        assert type(out.grad_fn).__name__.startswith("_SATrain") == (impl == "device"), impl
        running = [(layer.bn.bn.running_mean.clone(), layer.bn.bn.running_var.clone()) for mlp in mm.mlps for layer in mlp.children()] if bn else []
        res[impl] = (out.detach(), running, mm, new_xyz)
    out_d, run_d, md, new_xyz = res["device"]
    out_t, run_t, _, _ = res["torch"]
    assert not torch.isfinite(out_t).all(), "the torch path swallowed the value: the case tests nothing"
    assert torch.equal(torch.isfinite(out_d), torch.isfinite(out_t)), \
        "non-finite outputs differ in %d places" % int((torch.isfinite(out_d) != torch.isfinite(out_t)).sum())
    for l, ((dm, dv), (tm, tv)) in enumerate(zip(run_d, run_t)):
        assert torch.equal(torch.isfinite(dm), torch.isfinite(tm)), ("running_mean", l)
        assert torch.equal(torch.isfinite(dv), torch.isfinite(tv)), ("running_var", l)
    if not bn:
        idxs = md.fused_geometry(xyz, new_xyz)[2]
        off = 0
        for k, idx in enumerate(idxs):
            c = md.mlps[k][-1].conv.out_channels
            gathers = torch.zeros(2, idx.shape[1], dtype=torch.bool, device=cuda)
            gathers[0] = (idx[0] == 0).any(-1)
            assert gathers.any()
            assert torch.equal((~torch.isfinite(out_d[:, off:off + c])).any(1), gathers), k
            off += c

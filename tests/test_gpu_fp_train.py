"""The device training path of PointnetFPModule (pointnet2/fp_train.py, prb_fp_train_* in csrc/sa_train.cu) against the
float64 reference (tests/fp_train_reference.py), bit for bit on integer cases, across calls, and in a whole RPN step."""
import pytest
import torch

import fp_train_reference as R

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import config  # noqa: E402
from pointrcnn_b200.pointnet2 import fp_train  # noqa: E402
from pointrcnn_b200.pointnet2.pointnet2_modules import PointnetFPModule  # noqa: E402
from pointrcnn_b200.pointnet2 import pointnet2_utils  # noqa: E402

DEV = torch.device("cuda")
# (c_known, c_skip, widths, n, m) per RPN FP level (n, m per scene)
RPN_LEVELS = {"fp3": (1024, 512, (512, 512), 256, 64), "fp2": (512, 256, (512, 512), 1024, 256),
              "fp1": (512, 96, (256, 256), 4096, 1024), "fp0": (256, 1, (128, 128), 16384, 4096)}


def _module(c_known, c_skip, widths, bn=True, seed=0):
    torch.manual_seed(seed)
    m = PointnetFPModule(mlp=[c_known + c_skip] + list(widths), bn=bn).to(DEV).train()
    with torch.no_grad():
        for layer in m.mlp.children():
            if bn:
                layer.bn.bn.weight.uniform_(0.5, 1.5)
                layer.bn.bn.bias.uniform_(-0.2, 0.2)
            elif layer.conv.bias is not None:
                layer.conv.bias.uniform_(-0.2, 0.2)
    return m


def _inputs(B, n, m, c_known, c_skip, seed=1, skip_grad=True):
    g = torch.Generator(device=DEV).manual_seed(seed)
    unknown = torch.rand(B, n, 3, generator=g, device=DEV) * 10
    known = torch.rand(B, m, 3, generator=g, device=DEV) * 10
    kf = torch.randn(B, c_known, m, generator=g, device=DEV).requires_grad_(True)
    skip = torch.randn(B, c_skip, n, generator=g, device=DEV).requires_grad_(skip_grad) if c_skip else None
    gout_seed = torch.Generator(device=DEV).manual_seed(seed + 7)
    return unknown, known, kf, skip, gout_seed


def _layers(mod, bn):
    out = []
    for layer in mod.mlp.children():
        L = dict(W=layer.conv.weight.detach().double().cpu().view(layer.conv.out_channels, -1))
        if bn:
            L.update(gamma=layer.bn.bn.weight.detach().cpu(), beta=layer.bn.bn.bias.detach().cpu())
        else:
            L["bias"] = layer.conv.bias.detach().cpu() if layer.conv.bias is not None else None
        out.append(L)
    return out


def _device(mod, unknown, known, kf, skip, gout=None):
    mod.zero_grad(set_to_none=True)
    kf.grad = None
    if skip is not None:
        skip.grad = None
    out = mod._forward_train(unknown, known, skip, kf)
    if gout is None:
        gout = torch.randn(out.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    out.backward(gout)
    return out.detach(), gout


def _device_masks(out):
    """the ReLU decisions behind `out`: the sign of fma(a, z, b), exact in float64"""
    dec = fp_train.decisions(out)
    return [(s[2, :z.size(1)].double() * z.double() + s[3, :z.size(1)].double()) > 0 for z, s in zip(dec["z"], dec["stats"])]


def _check_against_reference(mod, unknown, known, kf, skip, bn):
    _, idx, w = pointnet2_utils.three_nn_weights(unknown.contiguous(), known.contiguous())
    mod.zero_grad(set_to_none=True)
    out = mod._forward_train(unknown, known, skip, kf)
    gout = torch.randn(out.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    masks = _device_masks(out)
    out.backward(gout)
    out = out.detach()
    ref_out, cache = R.forward(kf.detach().cpu(), skip.detach().cpu() if skip is not None else None, idx.cpu(), w.cpu(), _layers(mod, bn), bn,
                               order="projected")
    ref = R.backward(cache, gout.cpu(), masks=masks)
    bad = []
    ok, msg = R.compare(ref_out, out, "fwd")
    bad += [] if ok else ["out: " + msg]
    for l, layer in enumerate(mod.mlp.children()):
        ok, msg = R.compare(ref["W"][l], layer.conv.weight.grad.view(layer.conv.out_channels, -1), "grad")
        bad += [] if ok else ["W%d: %s" % (l, msg)]
        if bn:
            for k, p in (("gamma", layer.bn.bn.weight), ("beta", layer.bn.bn.bias)):
                ok, msg = R.compare(ref[k][l], p.grad, "grad")
                bad += [] if ok else ["%s%d: %s" % (k, l, msg)]
        elif layer.conv.bias is not None:
            ok, msg = R.compare(ref["bias"][l], layer.conv.bias.grad, "grad")
            bad += [] if ok else ["bias%d: %s" % (l, msg)]
    ok, msg = R.compare(ref["known"], kf.grad, "grad")
    bad += [] if ok else ["known: " + msg]
    if skip is not None and skip.requires_grad:
        ok, msg = R.compare(ref["skip"], skip.grad, "grad")
        bad += [] if ok else ["skip: " + msg]
    elif skip is not None:
        assert skip.grad is None
    assert not bad, bad


@pytest.mark.parametrize("level", sorted(RPN_LEVELS))
def test_rpn_levels_match_the_reference(level):
    c_known, c_skip, widths, n, m = RPN_LEVELS[level]
    mod = _module(c_known, c_skip, widths)
    unknown, known, kf, skip, _ = _inputs(2, n, m, c_known, c_skip, skip_grad=level != "fp0")
    _check_against_reference(mod, unknown, known, kf, skip, True)


@pytest.mark.parametrize("c_skip,widths,bn,B,n,m", [
    (0, (32,), True, 2, 200, 50),               # no skip, one layer
    (7, (48, 24, 16), True, 2, 300, 75),        # three layers
    (7, (48, 24, 16), False, 2, 300, 75),       # bias chain
    (3, (40, 70), False, 1, 50, 13),            # fewer rows than one row tile
    (5, (64, 64), True, 1, 90, 3),              # three known points
])
def test_shapes_match_the_reference(c_skip, widths, bn, B, n, m):
    mod = _module(20, c_skip, widths, bn=bn)
    unknown, known, kf, skip, _ = _inputs(B, n, m, 20, c_skip)
    _check_against_reference(mod, unknown, known, kf, skip, bn)


def test_two_calls_are_the_same_bits():
    c_known, c_skip, widths, n, m = RPN_LEVELS["fp1"]
    mod = _module(c_known, c_skip, widths)
    unknown, known, kf, skip, _ = _inputs(2, n, m, c_known, c_skip)
    res = []
    for _ in range(2):
        bns = [layer.bn.bn for layer in mod.mlp.children()]
        saved = [(b.running_mean.clone(), b.running_var.clone()) for b in bns]
        out, _ = _device(mod, unknown, known, kf, skip)
        stats = [(b.running_mean.clone(), b.running_var.clone()) for b in bns]
        for b, (rm, rv) in zip(bns, saved):
            b.running_mean.copy_(rm)
            b.running_var.copy_(rv)
        res.append([out, kf.grad.clone(), skip.grad.clone()] + [p.grad.clone() for p in mod.parameters()] + [t for s in stats for t in s])
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_no_host_synchronisation():
    c_known, c_skip, widths, n, m = RPN_LEVELS["fp0"]
    mod = _module(c_known, c_skip, widths)
    unknown, known, kf, skip, _ = _inputs(2, n, m, c_known, c_skip, skip_grad=False)
    _device(mod, unknown, known, kf, skip)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _device(mod, unknown, known, kf, skip)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_nan_in_known_features_propagates_as_on_the_torch_path():
    c_known, c_skip, widths, n, m = 16, 4, (32, 16), 256, 64
    mod = _module(c_known, c_skip, widths)
    unknown, known, kf, skip, _ = _inputs(2, n, m, c_known, c_skip)
    with torch.no_grad():
        kf[0, 3, 5] = float("nan")
    out, _ = _device(mod, unknown, known, kf, skip)
    with config.override(fp_train="torch"):
        ref = mod(unknown, known, skip, kf)
    assert torch.equal(torch.isnan(out), torch.isnan(ref.detach()))
    assert torch.isnan(kf.grad).any()


def test_peak_memory_at_fp0_is_not_above_the_torch_path():
    c_known, c_skip, widths, n, m = RPN_LEVELS["fp0"]
    mod = _module(c_known, c_skip, widths)
    mod.emit_point_major = False      # as the backbone's FP0: nothing gathers from the finest level
    unknown, known, kf, skip, _ = _inputs(16, n, m, c_known, c_skip, skip_grad=False)
    peaks = {}
    for impl in ("torch", "device", "torch", "device"):
        with config.override(fp_train=impl):
            mod.zero_grad(set_to_none=True)
            kf.grad = None
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            out = mod(unknown, known, skip, kf)
            out.backward(torch.ones_like(out))
            torch.cuda.synchronize()
            peaks[impl] = torch.cuda.max_memory_allocated() - base
            del out
    assert peaks["device"] <= peaks["torch"], peaks


def test_the_rule_selects_the_measured_levels():
    from pointrcnn_b200.backbone import Pointnet2MSG
    bb = Pointnet2MSG(input_channels=1)
    skips = [1, 96, 256, 512]
    chosen = {}
    for k, mod in enumerate(bb.FP_modules):
        c_in = mod.mlp[0].conv.in_channels
        chosen["fp%d" % k] = fp_train.faster_on_device(mod, c_in - skips[k], skips[k])
    assert chosen == {"fp0": True, "fp1": False, "fp2": False, "fp3": True}


@pytest.mark.parametrize("B,level,taps", [(2, "fp1", "onehot"), (2, "fp3", "onehot"), (16, "fp0", "onehot"), (16, "fp0", "half")])
def test_integer_cases_are_bit_exact(B, level, taps):
    c_known, c_skip, widths, n, m = RPN_LEVELS[level]
    if taps == "half":
        widths = widths[:1]
    c = R.integer_case(B, n, m, c_known, c_skip, widths, seed=B, taps=taps)
    out_ref, cache = R.forward(c["known"], c["skip"], c["idx"], c["w"], c["layers"], False)
    ref = R.backward(cache, c["gout"])
    R.check_exact(c, cache, out_ref, ref)
    mod = _module(c_known, c_skip, widths, bn=False)
    with torch.no_grad():
        for layer, L in zip(mod.mlp.children(), c["layers"]):
            layer.conv.weight.copy_(L["W"].view_as(layer.conv.weight))
            layer.conv.bias.copy_(L["bias"])
    kf = c["known"].to(DEV).requires_grad_(True)
    skip = c["skip"].to(DEV).requires_grad_(True)
    known_pm = kf.detach().transpose(1, 2).contiguous()
    out, _ = fp_train.forward(mod, c["idx"].to(DEV), c["w"].to(DEV), known_pm, kf, skip, False)
    out.backward(c["gout"].to(DEV))
    assert torch.equal(out.detach().cpu().double(), out_ref)
    assert torch.equal(kf.grad.cpu().double(), ref["known"])
    assert torch.equal(skip.grad.cpu().double(), ref["skip"])
    for layer, gw, gb in zip(mod.mlp.children(), ref["W"], ref["bias"]):
        assert torch.equal(layer.conv.weight.grad.view_as(gw).cpu().double(), gw)
        assert torch.equal(layer.conv.bias.grad.cpu().double(), gb)


def test_trainer_agrees_with_the_torch_path():
    import synth
    from pointrcnn_b200.train.step import RPNTrainer, synthetic_labels
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 7, channels=4)).to(DEV)
    cls, reg = synthetic_labels(pc, seed=2)

    def grads(fp, tf32=True):
        tr = RPNTrainer(input_channels=1, device=DEV, seed=3, loss_impl="device", sa_train="device", fp_train=fp)
        old = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = tf32
        try:
            loss, _ = tr.forward_loss(pc, cls, reg)
            loss.backward()
        finally:
            torch.backends.cudnn.allow_tf32 = old
        return float(loss), torch.cat([p.grad.flatten() for p in tr.params if p.grad is not None])

    l_t, g_t = grads("torch")
    l_d, g_d = grads("device")
    _, g_t32off = grads("torch", tf32=False)
    assert abs(l_d - l_t) <= 1e-4 * abs(l_t)
    base = float(torch.linalg.norm(g_t32off - g_t) / torch.linalg.norm(g_t))
    diff = float(torch.linalg.norm(g_d - g_t) / torch.linalg.norm(g_t))
    print("grad diff device %.3g, torch TF32 on/off %.3g" % (diff, base))
    assert diff <= max(base, 1e-6) * 1.5


def test_whole_rpn_step_does_not_synchronise():
    import synth
    from pointrcnn_b200.train.step import RPNTrainer, synthetic_labels
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 9, channels=4)).to(DEV)
    cls, reg = synthetic_labels(pc, seed=2)
    tr = RPNTrainer(input_channels=1, device=DEV, seed=3, loss_impl="device", sa_train="device", fp_train="device")
    tr.step(pc, cls, reg)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        tr.step(pc, cls, reg)
    finally:
        torch.cuda.set_sync_debug_mode(0)

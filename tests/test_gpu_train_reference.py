"""The SA and FP training kernels at the batch-16 training shapes against the per-element bound of tests/train_bound.py,
replayed in float64 on the device: every Z, statistic, running statistic, output and gradient element has
error / bound <= 1.  BN parameters are set so that some channels have gamma near 1e-3, one channel is constant (zero
variance) and one input channel is offset so that |mean| >> std.  Then one device RPN training step with hooks on every
SA / FP module and both heads: each device module's replay from what it received, the gradient at every junction
against the sum of what its consumers returned, and the gradient reaching the heads against the device loss.  Each
case prints the worst error / bound per tensor, the peak device memory and the wall time."""
import time

import numpy as np
import pytest
import torch

import train_bound as TB
from neighbour_reference import lidar
from pointrcnn_b200 import config
from pointrcnn_b200.pointnet2 import fp_train, sa_train
from pointrcnn_b200.pointnet2.pointnet2_modules import PointnetFPModule, PointnetSAModule, PointnetSAModuleMSG
from sa_train_reference import layer_params
from pointrcnn_b200.train.losses import rpn_loss

pytestmark = pytest.mark.gpu


def _harden(mod, seed):
    """gamma near 1e-3 on channels 0 and 1 of every BN layer, layer 0's channel 3 constant (zero weight row)"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for mlp in (mod.mlps if hasattr(mod, "mlps") else [mod.mlp]):
            for l, layer in enumerate(mlp.children()):
                if hasattr(layer, "bn"):
                    bn = layer.bn.bn
                    bn.weight.copy_(torch.rand(bn.weight.shape, generator=g) + 0.5)
                    bn.weight[0], bn.weight[1] = 1e-3, -2e-3
                    bn.bias.copy_(torch.rand(bn.bias.shape, generator=g) * 0.4 - 0.2)
                    bn.running_mean.copy_(torch.randn(bn.running_mean.shape, generator=g))
                    bn.running_var.copy_(torch.rand(bn.running_var.shape, generator=g) + 0.5)
                elif layer.conv.bias is not None:
                    layer.conv.bias.copy_(torch.rand(layer.conv.bias.shape, generator=g) * 0.2 - 0.1)
                if l == 0:
                    layer.conv.weight[3] = 0


def _report(name, worst, t0):
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    top = max(worst, key=worst.get)
    print("%s: worst error / bound %.3g (%s), peak %.1f GiB, %.1f s\n  %s" % (
        name, worst[top], top, peak, time.time() - t0, " ".join("%s=%.3g" % kv for kv in sorted(worst.items()))))
    assert worst[top] <= 1.0, (top, worst[top])


def _sa_case(cuda, kind):
    if kind == "rpn_sa1":
        B, N = 16, 16384
        xyz = torch.from_numpy(np.stack([lidar(N, 100 + b) for b in range(B)])).to(cuda)
        g = torch.Generator(device=cuda).manual_seed(1)
        feats = (torch.rand(B, 1, N, generator=g, device=cuda) + 8.0).requires_grad_(True)   # |mean| >> std
        torch.manual_seed(0)
        mod = PointnetSAModuleMSG(npoint=4096, radii=[0.1, 0.5], nsamples=[16, 32], mlps=[[1, 16, 16, 32], [1, 32, 32, 64]]).to(cuda)
    else:
        B, N = 256, 512                 # RoIs x pooled points, RCNN SA1 / SA2 settings (bias chains)
        g = torch.Generator(device=cuda).manual_seed(2)
        xyz = (torch.rand(B, N, 3, generator=g, device=cuda) - 0.5) * 3.0
        c_feat, npoint, radius, mlp = (128, 128, 0.2, [128, 128, 128, 128]) if kind == "rcnn_sa1" else (128, 32, 0.4, [128, 128, 128, 256])
        if kind == "rcnn_sa2":
            xyz = xyz[:, :128].contiguous()
            N = 128
        feats = torch.randn(B, c_feat, N, generator=g, device=cuda).requires_grad_(True)
        torch.manual_seed(0)
        mod = PointnetSAModule(npoint=npoint, radius=radius, nsample=64, mlp=mlp, bn=False).to(cuda)
    mod.train()
    _harden(mod, 3)
    return mod, xyz, feats


def _param_grads(mlp, grads):
    """{w|b|gamma|beta l: error / bound} of a SharedMLP's parameter gradients against replayed ones"""
    out = {}
    for l, c in enumerate(mlp.children()):
        got = dict(w=c.conv.weight.grad, b=c.conv.bias.grad if c.conv.bias is not None else None,
                   gamma=c.bn.bn.weight.grad if hasattr(c, "bn") else None, beta=c.bn.bn.bias.grad if hasattr(c, "bn") else None)
        for k, g in got.items():
            r = grads.get(k, [None] * (l + 1))[l]
            if g is not None or r is not None:
                out["%s%d" % (k, l)] = TB.ratio(g.reshape(r[0].shape), r[0], r[1])
    return out


def _replay_sa(mod, xyz, feats, new_xyz, layers, dec, out, gout, g_feats, chunk=None):
    """{quantity: worst error / bound} of one SA module's device forward and backward, replayed from its inputs (feats:
    the values it read), its decisions, its output and the gradient that reached it.  g_feats: the feature gradient it
    returned.  chunk: replay a bias chain that many scenes at a time (every sum of a bias chain is per scene but the
    parameter gradients', which add over the parts)"""
    B = xyz.shape[0]
    chunk = chunk or B
    assert chunk == B or len(mod.mlps) == 1
    centres, idxs = mod.fused_geometry(xyz, new_xyz)[1:3]
    worst, feat_parts, off = {}, {}, 0

    def put(name, r):
        worst[name] = max(worst.get(name, 0.0), r)

    for k, mlp in enumerate(mod.mlps):
        d = dec[k]
        C = d["z"][-1].shape[1]
        stats = [d["stats"][l, :, :z.shape[1]] for l, z in enumerate(d["z"])]
        P, ns = idxs[k].shape[1:]
        children = list(mlp.children())
        running = [(c.bn.bn.running_mean, c.bn.bn.running_var) if hasattr(c, "bn") else None for c in children]
        parts = []
        for b0 in range(0, B, chunk):
            b1, r0, r1 = min(B, b0 + chunk), b0 * P * ns, min(B, b0 + chunk) * P * ns
            st = TB.sa_scale(xyz[b0:b1], centres[b0:b1], None if feats is None else feats[b0:b1], idxs[k][b0:b1], layers[k],
                             [z[r0:r1] for z in d["z"]], stats, d["chosen"][b0 * P:b1 * P], gout[b0:b1, off:off + C],
                             dev=xyz.device, rows_total=None if chunk == B else B * P * ns, store=chunk == B)
            for q, r in TB.ratios(dict(out=out[b0:b1, off:off + C], running=running), st).items():
                put("s%d.%s" % (k, q), r)
            pool_ratio, not_first = st.pool
            put("s%d.pool" % k, pool_ratio if not not_first else float("inf"))
            put("s%d.relu" % k, st.flips)
            parts.append(st.grads)
            if st.feats is not None:
                feat_parts.setdefault(b0, []).append(st.feats)
            del st
        grads = parts[0] if chunk == B else TB.finish_grads(parts)
        for q, r in _param_grads(mlp, grads).items():
            put("s%d.%s" % (k, q), r)
        off += C
    for b0, fp in feat_parts.items():
        v, e = TB.feats_grad(fp)
        put("feats", TB.ratio(g_feats[b0:b0 + v.shape[0]], v, e))
    return worst


def _replay_fp(mod, unknown, known, kf, skip, layers, dec, out, gout, g_known, g_skip):
    """{quantity: worst error / bound} of one FP module's device forward and backward, replayed from its inputs, its saved
    state, its output and the gradient that reached it; g_known / g_skip: the input gradients it returned"""
    idx, w = mod.fused_geometry(unknown, known)
    st = TB.fp_module(kf, skip, idx, w, layers, dec["z"], [dec["stats"][l, :, :z.shape[1]] for l, z in enumerate(dec["z"])],
                      gout, dev=unknown.device)
    children = list(mod.mlp.children())
    got = dict(out=out, running=[(c.bn.bn.running_mean, c.bn.bn.running_var) for c in children], known=g_known, skip=g_skip)
    worst = TB.ratios(got, st)
    worst.update(_param_grads(mod.mlp, st.grads))
    worst["relu"] = st.flips
    return worst


@pytest.mark.parametrize("kind,entry", [("rpn_sa1", "atomic"), ("rpn_sa1", "ordered"), ("rcnn_sa1", "atomic"), ("rcnn_sa2", "ordered")])
def test_sa_training_kernels_stay_inside_the_bound(kind, entry, cuda, monkeypatch):
    if kind != "rpn_sa1":
        monkeypatch.setattr(sa_train, "FAST_MAX_WIDTH", 512)      # the width rule keeps the RCNN levels on the torch path
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    mod, xyz, feats = _sa_case(cuda, kind)
    layers = [layer_params(mlp) for mlp in mod.mlps]
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(entry == "ordered")
    try:
        with config.override(sa_train="device"):
            new_xyz, out = mod(xyz, feats)
        assert type(out.grad_fn).__name__.startswith("_SATrain"), "the dispatch did not take the device path"
        dec = sa_train.decisions(out)
        gout = torch.randn(out.shape, generator=torch.Generator(device=cuda).manual_seed(7), device=cuda)
        out.backward(gout)
    finally:
        torch.use_deterministic_algorithms(old)
    with torch.no_grad():
        worst = _replay_sa(mod, xyz, feats.detach(), new_xyz, layers, dec, out.detach(), gout, feats.grad,
                           chunk=None if kind == "rpn_sa1" else 32)
    _report("%s %s" % (kind, entry), worst, t0)


# (c_known, c_skip, widths, n, m) per RPN FP level at B = 16 (n, m per scene)
RPN_FP = {"fp3": (1024, 512, (512, 512), 256, 64), "fp2": (512, 256, (512, 512), 1024, 256),
          "fp1": (512, 96, (256, 256), 4096, 1024), "fp0": (256, 1, (128, 128), 16384, 4096)}


@pytest.mark.parametrize("level", sorted(RPN_FP))
def test_fp_training_kernels_stay_inside_the_bound(level, cuda, monkeypatch):
    c_known, c_skip, widths, n, m = RPN_FP[level]
    monkeypatch.setattr(fp_train, "FAST_LEVELS", {(c_known, c_skip, widths)})   # the rule selects FP0 and FP3 only
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    B = 16
    torch.manual_seed(0)
    mod = PointnetFPModule(mlp=[c_known + c_skip] + list(widths)).to(cuda).train()
    _harden(mod, 4)
    g = torch.Generator(device=cuda).manual_seed(5)
    unknown = torch.from_numpy(np.stack([lidar(n, 200 + b) for b in range(B)])).to(cuda)
    known = unknown[:, torch.randperm(n, generator=torch.Generator().manual_seed(6))[:m].to(cuda)].contiguous()
    kf = torch.relu(torch.randn(B, c_known, m, generator=g, device=cuda))
    kf[:, 0] += 8.0                                                   # |mean| >> std
    kf.requires_grad_(True)
    skip = torch.randn(B, c_skip, n, generator=g, device=cuda).requires_grad_(True)
    layers = layer_params(mod.mlp)
    with config.override(fp_train="device"):
        out = mod(unknown, known, skip, kf)
    assert type(out.grad_fn).__name__.startswith("_FPTrain"), "the dispatch did not take the device path"
    dec = fp_train.decisions(out)
    gout = torch.randn(out.shape, generator=torch.Generator(device=cuda).manual_seed(7), device=cuda)
    out.backward(gout)
    with torch.no_grad():
        worst = _replay_fp(mod, unknown, known, kf.detach(), skip.detach(), layers, dec, out.detach(), gout, kf.grad, skip.grad)
    _report("RPN %s at B = 16" % level, worst, t0)


# ------------------------------------------------------------------------------------------------ one device RPN step
def _sum_ratio(total, parts):
    """largest |total - sum(parts)| over the fp32 rounding of adding len(parts) tensors, (k - 1) u sum |part|; with one
    part the two must be the same bits (inf otherwise)"""
    s = sum(p.double() for p in parts)
    bound = (len(parts) - 1) * TB.U * sum(p.double().abs() for p in parts)
    return TB.ratio(total, s, bound)


def test_device_rpn_step_hands_off_every_gradient(cuda):
    """one RPNTrainer step at B = 16 with the device SA, FP and loss paths, the input intensity given a gradient.  Hooks
    capture every SA / FP module's inputs, output, decisions, the gradient reaching its output and the gradients it
    returns (each input passes through an alias of its own, which keeps the point-major twin).  Then:
    (a) every module that took a device path stays inside the bound when replayed from what it was given;
    (b) at every junction the gradient on the tensor equals the sum of what its consumers returned: the intensity (SA1
        grouping + FP0 skip), SA_k's output (SA_k+1 grouping + FP_k skip; SA4: FP3's known features), FP_k's output
        (FP_k-1's known features; FP0: both heads);
    (c) the gradients reaching the head outputs are the device loss backward's, bit for bit."""
    import synth
    from pointrcnn_b200.train.step import RPNTrainer, synthetic_labels
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    pc = torch.from_numpy(synth.u_kitti(16, 16384, 123, channels=4)).to(cuda)
    cls_label, reg_label = synthetic_labels(pc, seed=1)
    tr = RPNTrainer(input_channels=1, device=cuda, world=1, seed=3, loss_impl="device", sa_train="device", fp_train="device")
    m = tr.model
    bb = m.backbone_net
    cap, ret, tot, hooks, given = {}, {}, {}, [], {}

    def keep(store, key):
        def hook(g):
            store[key] = g.detach().clone()
        return hook

    def alias(t, key):
        if t is None or not t.requires_grad:
            return t
        a = t.view_as(t)
        if hasattr(t, "_prb_pm"):
            a._prb_pm = t._prb_pm              # the producer's point-major twin: the alias shares t's version counter
        a.register_hook(keep(ret, key))
        return a

    def pre(name, slots):
        def hook(mod, args):
            args = list(args)
            cap[name] = dict(args=[a.detach() if torch.is_tensor(a) else a for a in args],
                             layers=[layer_params(x) for x in mod.mlps] if hasattr(mod, "mlps") else
                             layer_params(mod.mlp) if hasattr(mod, "mlp") else None)
            for i, slot in slots.items():
                args[i] = alias(args[i], "%s.%s" % (name, slot))
            return tuple(args)
        return hook

    def post(name, index=None):
        def hook(mod, args, out):
            t = out if index is None else out[index]
            cap[name]["out"] = t.detach()
            if index is not None:
                cap[name]["new_xyz"] = out[0]
            kind = type(t.grad_fn).__name__
            if kind.startswith("_SATrain"):
                cap[name]["dec"] = sa_train.decisions(t)
            elif kind.startswith("_FPTrain"):
                cap[name]["dec"] = fp_train.decisions(t)
            t.register_hook(keep(tot, name))
        return hook

    for k, sa in enumerate(bb.SA_modules):
        hooks += [sa.register_forward_pre_hook(pre("sa%d" % k, {1: "features"})), sa.register_forward_hook(post("sa%d" % k, 1))]
    for k, fp in enumerate(bb.FP_modules):
        hooks += [fp.register_forward_pre_hook(pre("fp%d" % k, {2: "skip", 3: "known"})), fp.register_forward_hook(post("fp%d" % k))]
    for name in ("rpn_cls_layer", "rpn_reg_layer"):
        hooks += [getattr(m, name).register_forward_pre_hook(pre(name, {0: "in"})), getattr(m, name).register_forward_hook(post(name))]
    split = bb._break_up_pc

    def break_up(p):
        xyz, f = split(p)
        given["intensity"] = f.requires_grad_(True)
        return xyz, f

    bb._break_up_pc = break_up
    grads = {}
    step = tr.opt.step

    def snapshot_then_step(*a, **kw):
        grads.update({n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None})
        return step(*a, **kw)

    tr.opt.step = snapshot_then_step
    try:
        loss, _ = tr.step(pc, cls_label, reg_label)
    finally:
        for h in hooks:
            h.remove()
        del bb._break_up_pc
        tr.opt.step = step
    device = sorted(n for n, c in cap.items() if "dec" in c)
    assert device == ["fp0", "fp3", "sa0"], device

    worst = {}
    with torch.no_grad():
        # (a) the device modules' replays, their parameter gradients as they were before the optimizer step
        for p in m.parameters():
            p.grad = None
        for n, p in m.named_parameters():
            if n in grads:
                p.grad = grads[n]
        c = cap["sa0"]
        w = _replay_sa(bb.SA_modules[0], c["args"][0].contiguous(), c["args"][1], c["new_xyz"], c["layers"], c["dec"], c["out"],
                       tot["sa0"], ret["sa0.features"])
        worst.update({"sa0." + q: r for q, r in w.items()})
        for k in (0, 3):
            c = cap["fp%d" % k]
            unknown, known, skip, kf = c["args"]
            w = _replay_fp(bb.FP_modules[k], unknown, known, kf, skip, c["layers"], c["dec"], c["out"], tot["fp%d" % k],
                           ret["fp%d.known" % k], ret["fp%d.skip" % k])
            worst.update({"fp%d.%s" % (k, q): r for q, r in w.items()})
        # (b) the junctions
        junctions = {"intensity": (given["intensity"].grad, ["sa0.features", "fp0.skip"])}
        for k in range(3):
            junctions["sa%d" % k] = (tot["sa%d" % k], ["sa%d.features" % (k + 1), "fp%d.skip" % (k + 1)])
        junctions["sa3"] = (tot["sa3"], ["fp3.known"])
        for k in (3, 2, 1):
            junctions["fp%d" % k] = (tot["fp%d" % k], ["fp%d.known" % (k - 1)])
        junctions["fp0"] = (tot["fp0"], ["rpn_cls_layer.in", "rpn_reg_layer.in"])
        for name, (total, parts) in junctions.items():
            worst["junction." + name] = _sum_ratio(total, [ret[p] for p in parts])
        # (c) the device loss backward from the head outputs the step produced
        heads = [cap[n]["out"].transpose(1, 2).contiguous().requires_grad_(True) for n in ("rpn_cls_layer", "rpn_reg_layer")]
        with torch.enable_grad():
            again, _ = rpn_loss(heads[0], heads[1], cls_label, reg_label, tr.mean_size, impl="device")
            g_cls, g_reg = torch.autograd.grad(again, heads)
        assert torch.equal(again, loss)
        for n, g in (("rpn_cls_layer", g_cls), ("rpn_reg_layer", g_reg)):
            worst["heads." + n] = 0.0 if torch.equal(tot[n], g.transpose(1, 2)) else float("inf")
    _report("device RPN step at B = 16", worst, t0)

"""The device SA training path (csrc/sa_train.cu through pointnet2/sa_train.py, config.sa_train="device") against the
float64 reference of tests/sa_train_reference.py: forward output and running statistics with the reference's own
decisions, every gradient with the device's decisions (ReLU masks from the saved Z, the chosen samples), the decisions
themselves within the forward bound of a tie or of zero, determinism, no host synchronisation, the trainers against the
torch path, and peak memory."""
import copy

import numpy as np
import pytest
import torch

import sa_train_reference as R
from pointrcnn_b200 import config
from pointrcnn_b200.pointnet2 import sa_train
from pointrcnn_b200.pointnet2.pointnet2_modules import PointnetSAModule, PointnetSAModuleMSG

pytestmark = pytest.mark.gpu


def _cloud(B, N, seed, spread=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, N, 3, generator=g) * spread


# name: (module factory, B, N, c_feat, features need grad)
CASES = {
    "rpn_sa1": (lambda: PointnetSAModuleMSG(npoint=64, radii=[0.1, 0.5], nsamples=[16, 32], mlps=[[1, 16, 16, 32], [1, 32, 32, 64]]),
                2, 1024, 1, False),
    "rpn_sa2_96": (lambda: PointnetSAModuleMSG(npoint=32, radii=[0.5, 1.0], nsamples=[16, 32], mlps=[[96, 64, 64, 128], [96, 64, 96, 128]]),
                   2, 256, 96, True),
    "rpn_sa3_196": (lambda: PointnetSAModuleMSG(npoint=16, radii=[1.0, 2.0], nsamples=[16, 32],
                                                mlps=[[256, 128, 196, 256], [256, 128, 196, 256]]), 2, 128, 256, True),
    "rpn_sa4_384": (lambda: PointnetSAModuleMSG(npoint=8, radii=[2.0, 4.0], nsamples=[16, 32],
                                                mlps=[[512, 256, 256, 512], [512, 256, 384, 512]]), 2, 64, 512, True),
    "rcnn_sa1": (lambda: PointnetSAModule(npoint=32, radius=0.2, nsample=64, mlp=[128, 128, 128, 128], bn=False), 2, 256, 128, True),
    "rcnn_sa2": (lambda: PointnetSAModule(npoint=8, radius=0.4, nsample=64, mlp=[128, 128, 128, 256], bn=False), 2, 32, 128, True),
    "rcnn_sa3_group_all": (lambda: PointnetSAModule(mlp=[256, 256, 256, 512], bn=False), 2, 32, 256, True),
    "no_features_1_layer": (lambda: PointnetSAModule(npoint=32, radius=0.3, nsample=16, mlp=[0, 32]), 2, 256, 0, False),
    "two_layers": (lambda: PointnetSAModule(npoint=32, radius=0.3, nsample=32, mlp=[8, 24, 40]), 2, 256, 8, True),
    "sparse_padding": (lambda: PointnetSAModule(npoint=32, radius=0.03, nsample=32, mlp=[4, 16, 32]), 2, 512, 4, True),
    "smaller_than_a_tile": (lambda: PointnetSAModule(npoint=4, radius=0.5, nsample=8, mlp=[4, 16, 16]), 1, 64, 4, True),
}


def _setup(name, cuda, seed=0):
    make, B, N, c_feat, feat_grad = CASES[name]
    torch.manual_seed(seed)
    m = make().to(cuda).train()
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.weight.uniform_(0.5, 1.5)
                mod.bias.uniform_(-0.2, 0.2)
            if isinstance(mod, torch.nn.Conv2d) and mod.bias is not None:
                mod.bias.uniform_(-0.1, 0.1)
    xyz = _cloud(B, N, seed + 1, spread=3.0 if "sparse" in name else 1.0).to(cuda)
    feats = None
    if c_feat:
        feats = torch.randn(B, c_feat, N, generator=torch.Generator().manual_seed(seed + 2)).to(cuda)
        if feat_grad:
            feats.requires_grad_(True)
    return m, xyz, feats


def _run(m, xyz, feats, gout=None):
    """forward (through the device path whatever the width rule says) + backward -> (new_xyz, out, gout, decisions)"""
    with config.override(sa_train="device"):
        assert sa_train.supported(m, xyz, feats, None)
        new_xyz, out = m._forward_train(xyz, feats, None)
    assert type(out.grad_fn).__name__.startswith("_SATrain"), "the device path did not run"
    dec = [{k: [t.clone() for t in v] if isinstance(v, list) else v.clone() for k, v in d.items()} for d in sa_train.decisions(out)]
    if gout is None:
        gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(7)).to(out.device)
    out.backward(gout)
    return new_xyz, out, gout, dec


def _reference(m0, m, xyz, feats, new_xyz, out, gout, dec):
    """per scale: the float64 reference with its own decisions (forward), with the device's decisions (gradients), and the
    largest error-to-tolerance ratio of every quantity; asserts the decision bound"""
    centres, idxs = m.fused_geometry(xyz.contiguous(), new_xyz)[1:3]
    ratios, off = {}, 0
    for k, mlp0 in enumerate(m0.mlps):
        layers = R.layer_params(mlp0)
        d = dec[k]
        c = mlp0[-1].conv.out_channels
        g = gout[:, off:off + c]
        f = None if feats is None else feats.detach()
        own = R.scale(xyz, centres, f, idxs[k], layers)
        masks = [(st[R_A] * z + st[R_B] > 0) for z, st in ((z, d["stats"][l, :, :z.shape[1]]) for l, z in enumerate(d["z"]))]
        dev_dec = R.scale(xyz, centres, f, idxs[k], layers, g, masks=masks, chosen=d["chosen"])
        # the decisions: a flipped ReLU lies within the forward bound of zero, a chosen sample within it of the maximum
        for l, (mk, pre) in enumerate(zip(masks, own["pre"])):
            flip = mk.cpu() != (pre > 0)
            bound = R.FWD_TOL * pre.abs().max()
            assert (pre[flip].abs() <= bound).all(), (k, l, int(flip.sum()), float(pre[flip].abs().max()), float(bound))
        y = torch.relu(own["pre"][-1]).view(d["chosen"].shape[0], -1, c)
        picked = y.gather(1, d["chosen"].long().cpu().unsqueeze(1)).squeeze(1)
        assert (picked >= y.max(1).values - R.FWD_TOL * y.abs().max()).all(), k
        got = dict(out=out[:, off:off + c].detach(), running=[], w=[], b=[], gamma=[], beta=[])
        for layer in mlp_layers(m.mlps[k]):
            if hasattr(layer, "bn"):
                bn = layer.bn.bn
                got["running"].append((bn.running_mean, bn.running_var, int(bn.num_batches_tracked)))
                got["gamma"].append(bn.weight.grad)
                got["beta"].append(bn.bias.grad)
            else:
                got["gamma"].append(None)
                got["beta"].append(None)
            got["w"].append(layer.conv.weight.grad.flatten(1))
            got["b"].append(None if layer.conv.bias is None else layer.conv.bias.grad)
        for q, r in R.all_ratios(dict(out=got["out"], running=got["running"]), own).items():
            ratios["s%d.%s" % (k, q)] = r
        for a, b in zip(got["running"], own["running"]):
            assert a[2] == b[2]
        for q, r in R.all_ratios(dict(got, out=dev_dec["out"], running=[]), dev_dec).items():
            if q != "out":
                ratios["s%d.%s" % (k, q)] = r
        off += c
    return ratios


R_MEAN, R_INVSTD, R_A, R_B = range(4)


def mlp_layers(mlp):
    return list(mlp.children())


def _feature_grad_ratio(m0, m, xyz, feats, new_xyz, gout, dec):
    """d features summed over all scales, with the device's decisions"""
    centres, idxs = m.fused_geometry(xyz.contiguous(), new_xyz)[1:3]
    total, off = None, 0
    for k, mlp0 in enumerate(m0.mlps):
        d = dec[k]
        c = mlp0[-1].conv.out_channels
        masks = [(st[R_A] * z + st[R_B] > 0) for z, st in ((z, d["stats"][l, :, :z.shape[1]]) for l, z in enumerate(d["z"]))]
        r = R.scale(xyz, centres, feats.detach(), idxs[k], R.layer_params(mlp0), gout[:, off:off + c], masks=masks, chosen=d["chosen"])
        total = r["feats"] if total is None else total + r["feats"]
        off += c
    return R.grad_ratio(feats.grad, total)


@pytest.mark.parametrize("name", list(CASES))
def test_device_path_against_the_float64_reference(name, cuda):
    m, xyz, feats = _setup(name, cuda)
    m0 = copy.deepcopy(m)
    new_xyz, out, gout, dec = _run(m, xyz, feats)
    ratios = _reference(m0, m, xyz, feats, new_xyz, out, gout, dec)
    if feats is not None and feats.requires_grad:
        ratios["feats"] = _feature_grad_ratio(m0, m, xyz, feats, new_xyz, gout, dec)
    elif feats is not None:
        assert feats.grad is None
    worst = max(ratios, key=ratios.get)
    print("%s: largest error / tolerance %.3f (%s); %s" % (name, ratios[worst], worst,
                                                           " ".join("%s=%.3f" % kv for kv in sorted(ratios.items()))))
    assert ratios[worst] <= 1.0, (worst, ratios)


def test_forward_and_backward_are_deterministic_and_do_not_synchronise(cuda):
    m, xyz, feats = _setup("rpn_sa2_96", cuda)
    state = copy.deepcopy(m.state_dict())
    runs = []
    _, out0, gout, _ = _run(m, xyz, feats)
    for rep in range(2):
        m.load_state_dict(state)
        m.zero_grad(set_to_none=True)
        feats.grad = None
        torch.cuda.synchronize()
        if rep == 1:
            torch.cuda.set_sync_debug_mode("error")
        try:
            _, out, _, _ = _run(m, xyz, feats, gout)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        runs.append([out.detach().clone()] + [t.detach().clone() for t in m.state_dict().values()]
                    + [p.grad.clone() for p in m.parameters()])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def _rpn_batch(cuda, B):
    import synth
    from pointrcnn_b200.train.step import synthetic_labels
    pc = torch.from_numpy(synth.u_kitti(B, 16384, 123, channels=4)).to(cuda)
    return (pc,) + synthetic_labels(pc, seed=1)


def test_rpn_step_with_device_sa_and_loss_does_not_synchronise(cuda):
    from pointrcnn_b200.train.step import RPNTrainer
    tr = RPNTrainer(input_channels=1, device=cuda, world=1, seed=3, loss_impl="device", sa_train="device")
    batch = _rpn_batch(cuda, 2)
    tr.step(*batch)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss, _ = tr.step(*batch)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(loss).item()


def _rcnn_batch(cuda):
    from oracle import rcnn_offline as RO
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    scenes = [RO.synth_scene(s, k, n_feat=128) for s, k in ((51, "mixed"), (52, "hard"))]
    return RCNNOfflineSampler(device=cuda).prepare_jit_batch(scenes)


def _train_once(kind, cuda, batch, impl, cudnn_tf32=True, capture=False):
    """one forward + backward of a fresh trainer (same seed every time) -> dict(loss, grads {name: grad}, ran [indices of the
    SA modules that took the device path]); capture: also a copy of SA1 from before the forward, its inputs and the
    gradient that reached its output"""
    from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer
    old_tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = cudnn_tf32
    hooks, ran, cap = [], [], {}
    try:
        if kind == "rpn":
            tr = RPNTrainer(input_channels=1, device=cuda, world=1, seed=3, sa_train=impl)
            sas = tr.model.backbone_net.SA_modules
        else:
            tr = RCNNTrainer(device=cuda, seed=5, target_draw="device", sa_train=impl)
            sas = tr.model.SA_modules
        for i, sa in enumerate(sas):
            hooks.append(sa.register_forward_hook(
                lambda mod, args, out, i=i: ran.append(i) if type(out[1].grad_fn).__name__.startswith("_SATrain") else None))
        if capture:
            cap["module"] = copy.deepcopy(sas[0])
            hooks.append(sas[0].register_forward_pre_hook(lambda mod, args: cap.update(
                xyz=args[0].detach().clone(), feats=None if args[1] is None else args[1].detach().clone())))
            def keep_gout(mod, args, out):           # returns None: a forward hook's return value would replace the output
                out[1].register_hook(lambda g: cap.update(gout=g.detach().clone()))
            hooks.append(sas[0].register_forward_hook(keep_gout))
        tr.opt.zero_grad(set_to_none=True)
        loss, _ = tr.forward_loss(*batch) if kind == "rpn" else tr.forward_loss_jit(batch)
        loss.backward()
    finally:
        torch.backends.cudnn.allow_tf32 = old_tf32
        for h in hooks:
            h.remove()
    grads = {n: p.grad.detach().clone() for n, p in tr.model.named_parameters() if p.requires_grad}
    return dict(loss=float(loss), grads=grads, ran=ran, cap=cap, sa1_prefix=("backbone_net." if kind == "rpn" else "") + "SA_modules.0.")


def _spread(run, base):
    """the largest relative Frobenius difference of a parameter gradient, and its name"""
    return max((float((g - base["grads"][n]).norm() / base["grads"][n].norm().clamp_min(1e-30)), n) for n, g in run["grads"].items())


@pytest.mark.parametrize("kind", ["rpn", "rcnn"])
def test_trainer_agrees_with_the_torch_path(kind, cuda, monkeypatch):
    """device vs torch at B = 2 from the same seed and batch.
    - The first loss agrees within 1e-4 relative.
    - Whole-network parameter gradients of an untrained network amplify TF32-level perturbations: the torch path against
      itself with cuDNN's TF32 switched off differs by up to ~0.3 relative Frobenius (RPN).  The device path's difference
      must not exceed that baseline, measured in the same test.
    - The gradients the device backward owns, SA1's parameters, are bounded at 2e-2 relative Frobenius when it is given the
      torch run's SA1 inputs and the upstream gradient that reached SA1's output there."""
    if kind == "rcnn":
        monkeypatch.setattr(sa_train, "FAST_MAX_WIDTH", 512)        # every RCNN level is wider than the rule: force the device path
    batch = _rpn_batch(cuda, 2) if kind == "rpn" else _rcnn_batch(cuda)
    base = _train_once(kind, cuda, batch, "torch", capture=True)
    fp32 = _train_once(kind, cuda, batch, "torch", cudnn_tf32=False)
    dev = _train_once(kind, cuda, batch, "device")
    assert base["ran"] == [] and fp32["ran"] == []
    assert dev["ran"] == ([0] if kind == "rpn" else [0, 1, 2]), dev["ran"]
    rel_loss = abs(dev["loss"] - base["loss"]) / abs(base["loss"])
    s_dev, s_tf32 = _spread(dev, base), _spread(fp32, base)
    print("%s trainer: first loss rel. diff %.2e; worst gradient rel. Frobenius device %.2e (%s), torch with fp32 convolutions "
          "%.2e (%s)" % (kind, rel_loss, s_dev[0], s_dev[1], s_tf32[0], s_tf32[1]))
    assert rel_loss <= 1e-4
    assert s_dev[0] <= s_tf32[0]

    cap = base["cap"]
    sa1 = cap["module"]
    feats = None if cap["feats"] is None else cap["feats"].requires_grad_(True)
    out = sa1._forward_train(cap["xyz"], feats, None)[1]
    assert type(out.grad_fn).__name__.startswith("_SATrain")
    out.backward(cap["gout"])
    own = {n: float((p.grad - base["grads"][base["sa1_prefix"] + n]).norm() / base["grads"][base["sa1_prefix"] + n].norm().clamp_min(1e-30))
           for n, p in sa1.named_parameters()}
    worst = max(own, key=own.get)
    print("  SA1 parameters, same inputs and upstream gradient: worst rel. Frobenius %.2e (%s)" % (own[worst], worst))
    assert own[worst] <= 2e-2, own


def test_the_width_rule_selects_rpn_sa1_only(cuda):
    from pointrcnn_b200.backbone import Pointnet2MSG
    sa = Pointnet2MSG(input_channels=1).to(cuda).train().SA_modules
    assert [sa_train.faster_on_device(m) for m in sa] == [True, False, False, False]
    xyz = _cloud(1, 1024, 3).to(cuda)
    f = torch.rand(1, 1, 1024, device=cuda)
    for impl, want in (("device", "_SATrain"), ("torch", "Cat")):
        with config.override(sa_train=impl):
            _, out = sa[0](xyz, f)
        assert type(out.grad_fn).__name__.startswith(want), (impl, type(out.grad_fn).__name__)


def test_peak_memory_of_rpn_sa1_is_not_above_the_torch_path(cuda):
    import synth
    from pointrcnn_b200.backbone import Pointnet2MSG
    torch.manual_seed(0)
    sa1 = Pointnet2MSG(input_channels=1).to(cuda).train().SA_modules[0]
    pc = torch.from_numpy(synth.u_kitti(4, 16384, 5, channels=4)).to(cuda)
    xyz, feats = pc[..., :3].contiguous(), pc[..., 3:].transpose(1, 2).contiguous()
    peaks = {}
    for impl in ("torch", "device", "torch"):
        sa1.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with config.override(sa_train=impl):
            _, out = sa1(xyz, feats)
        out.backward(torch.ones_like(out))
        del out
        torch.cuda.synchronize()
        peaks[impl] = torch.cuda.max_memory_allocated() - base
    print("RPN SA1 at B = 4: peak MB torch %.1f, device %.1f" % (peaks["torch"] / 2 ** 20, peaks["device"] / 2 ** 20))
    assert peaks["device"] <= peaks["torch"]

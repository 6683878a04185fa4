"""CPU side of the device SA training path: the C ABI exports and descriptor layout, CPU tensors refused, the dispatch rule,
the float64 reference's tolerances shown to catch each of the mistakes they guard against, and the integer-valued cases
of the exact GPU tests: the generator's cases pass the exactness check, which refuses an operand or a sum too large."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn

import sa_train_reference as R
from pointrcnn_b200 import _cabi as C
from pointrcnn_b200 import config
from pointrcnn_b200.pointnet2 import sa_train
from pointrcnn_b200.pointnet2.pointnet2_modules import PointnetSAModule, PointnetSAModuleMSG


def test_sa_train_symbols_resolve_at_abi_11():
    lib = C.lib()
    for name in ("prb_sa_train_workspace_bytes", "prb_sa_train_forward", "prb_sa_train_backward"):
        assert getattr(lib, name) is not None
    assert lib.prb_abi_version() == 11
    d = C.SATrainDesc(num_layers=3, c_in=4)
    d.c_out[:] = [16, 16, 32]
    fwd = lib.prb_sa_train_workspace_bytes(16, 4096, 32, 1, ctypes.byref(d), 0)
    bwd = lib.prb_sa_train_workspace_bytes(16, 4096, 32, 1, ctypes.byref(d), 1)
    rows = 16 * 4096 * 32
    assert fwd > 0 and bwd >= fwd + 2 * rows * 16 * 4    # the forward leaves out the two backward gradient buffers
    d.c_out[2] = 513
    assert lib.prb_sa_train_workspace_bytes(16, 4096, 32, 1, ctypes.byref(d), 0) == 0     # refused: wider than 512
    assert b"512" in lib.prb_last_error()


def test_descriptor_layout_matches_the_header():
    """six ints (num_layers, c_in, c_out[3], bn), eps and momentum, then seven arrays of three pointers"""
    assert ctypes.sizeof(C.SATrainDesc) == 24 + 16 + 7 * 3 * 8
    assert C.SATrainDesc.eps.offset == 24 and C.SATrainDesc.weight.offset == 40
    assert C.SATrainDesc.num_batches_tracked.offset == 40 + 6 * 24


def test_forward_refuses_cpu_tensors():
    m = PointnetSAModuleMSG(npoint=4, radii=[0.5], nsamples=[8], mlps=[[1, 8]]).train()
    xyz, f = torch.rand(1, 32, 3), torch.rand(1, 1, 32)
    idx = torch.zeros(1, 4, 8, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="CUDA"):
        sa_train.forward(m, xyz, f, f.transpose(1, 2).contiguous(), xyz[:, :4].contiguous(), [idx], [8])


def _modules():
    """(name, module, c_feat) of every layout the rule accepts"""
    yield "rpn_sa1", PointnetSAModuleMSG(npoint=8, radii=[0.1, 0.5], nsamples=[16, 32], mlps=[[1, 16, 16, 32], [1, 32, 32, 64]]), 1
    yield "rpn_sa3", PointnetSAModuleMSG(npoint=8, radii=[1.0, 2.0], nsamples=[16, 32], mlps=[[256, 128, 196, 256], [256, 128, 196, 256]]), 256
    yield "rcnn_sa1", PointnetSAModule(npoint=8, radius=0.2, nsample=64, mlp=[128, 128, 128, 128], bn=False), 128
    yield "rcnn_sa3", PointnetSAModule(mlp=[256, 256, 256, 512], bn=False), 256
    yield "no_feats", PointnetSAModule(npoint=8, radius=0.2, nsample=4, mlp=[0, 32]), 0


def test_rule_accepts_the_project_layouts():
    for name, m, c_feat in _modules():
        assert sa_train.layout_ok(m.train(), c_feat, 64), name


def test_rule_rejects_every_unsupported_layout():
    def base():
        return PointnetSAModuleMSG(npoint=8, radii=[0.1, 0.5], nsamples=[16, 32], mlps=[[1, 16, 16, 32], [1, 32, 32, 64]]).train()

    cases = {}
    m = base().eval()
    cases["eval_bn"] = m
    m = base()
    m.mlps[0].layer0.bn.bn.momentum = None
    cases["cumulative_momentum"] = m
    m = base()
    m.mlps[1].layer1.bn.bn.track_running_stats = False
    cases["untracked_stats"] = m
    m = base()
    m.mlps[0].layer2.bn.bn.eps = 1e-3
    cases["mixed_eps"] = m
    m = base()
    m.pool_method = "avg_pool"
    cases["avg_pool"] = m
    cases["instance_norm"] = PointnetSAModule(npoint=8, radius=0.2, nsample=16, mlp=[1, 16], bn=False, instance_norm=True).train()
    cases["no_use_xyz"] = PointnetSAModule(npoint=8, radius=0.2, nsample=16, mlp=[1, 16], use_xyz=False).train()
    cases["nsample_24"] = PointnetSAModule(npoint=8, radius=0.2, nsample=24, mlp=[1, 16]).train()
    cases["nsample_2"] = PointnetSAModule(npoint=8, radius=0.2, nsample=2, mlp=[1, 16]).train()
    cases["nsample_256"] = PointnetSAModule(npoint=8, radius=0.2, nsample=256, mlp=[1, 16]).train()
    cases["four_layers"] = PointnetSAModule(npoint=8, radius=0.2, nsample=16, mlp=[1, 16, 16, 16, 16]).train()
    cases["width_1024"] = PointnetSAModule(npoint=8, radius=0.2, nsample=16, mlp=[1, 1024]).train()
    m = PointnetSAModule(npoint=8, radius=0.2, nsample=16, mlp=[1, 16, 16]).train()
    m.mlps[0].layer0.activation = nn.LeakyReLU()
    cases["leaky_relu"] = m
    m = PointnetSAModule(npoint=8, radius=0.2, nsample=16, mlp=[1, 16]).train()
    m.mlps[0].layer0.conv = nn.Conv2d(4, 16, kernel_size=(1, 3), padding=(0, 1), bias=False)
    cases["conv_1x3"] = m
    for name, m in cases.items():
        assert not sa_train.layout_ok(m, 1, 64), name
    assert not sa_train.layout_ok(PointnetSAModule(mlp=[1, 16]).train(), 1, 48)            # GroupAll over 48 points
    assert not sa_train.layout_ok(base(), 2, 64)                                          # channels do not match


def test_cpu_modules_and_the_torch_switch_keep_the_torch_path():
    torch.manual_seed(0)
    m = PointnetSAModuleMSG(npoint=4, radii=[0.5], nsamples=[8], mlps=[[1, 8]]).train()
    xyz, f = torch.rand(1, 32, 3), torch.rand(1, 1, 32)
    assert config.get("sa_train") in ("torch", "device")
    with config.override(sa_train="device"):
        try:
            _, out = m(xyz, f)
        except RuntimeError as e:              # the torch path's natives need CUDA too; the device path must not be what ran
            assert "sa_train" not in str(e)
        else:
            assert "SATrain" not in type(out.grad_fn).__name__


def test_trainer_refuses_an_unknown_setting():
    from pointrcnn_b200.train.step import RPNTrainer
    with pytest.raises(ValueError, match="sa_train"):
        RPNTrainer(device="cpu", sa_train="cuda")


# ---------------------------------------------------------------------------------------------- the tolerances bite
def _case(n_small=False, bn=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    if n_small:
        B, N, P, ns, widths = 1, 24, 4, 4, [8, 8]           # n = 16 rows: n / (n - 1) is visible
    else:
        B, N, P, ns, widths = 2, 96, 16, 8, [16, 16, 24]
    c_feat = 2
    m = PointnetSAModule(npoint=P, radius=0.45, nsample=ns, mlp=[c_feat] + widths, bn=bn).train()
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (0.6 if p.dim() > 1 else 0.3) + (1.0 if p.dim() == 1 and bn else 0.0))
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.running_mean.copy_(torch.randn(mod.num_features, generator=g) * 0.1)
                mod.running_var.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
    xyz = torch.rand(B, N, 3, generator=g)
    centres = xyz[:, :P].clone()
    feats = torch.randn(B, c_feat, N, generator=g)
    idx = R.ball_query(0.45, ns, xyz, centres)
    gout = torch.randn(B, widths[-1], P, generator=g)
    return m, xyz, centres, feats, idx, gout


@pytest.mark.parametrize("mutant", R.MUTANTS)
def test_each_mutant_of_the_reference_exceeds_a_tolerance(mutant):
    m, xyz, centres, feats, idx, gout = _case(n_small=mutant == "biased_running")
    layers = R.layer_params(m.mlps[0])
    ref = R.scale(xyz, centres, feats, idx, layers, gout)
    bad = R.scale(xyz, centres, feats, idx, copy.deepcopy(layers), gout, mutant=mutant)
    ratios = R.all_ratios(bad, ref)
    assert max(ratios.values()) > 1.0, (mutant, ratios)
    assert max(R.all_ratios(R.scale(xyz, centres, feats, idx, layers, gout), ref).values()) == 0.0


def _integer_bias_case():
    """an integer-valued bias-only chain (sa_train_reference.integer_case) as a torch module and its inputs"""
    B, N, P, ns, c_feat, widths = 2, 96, 16, 8, 2, [16, 16, 24]
    case = R.integer_case(B, N, P, ns, c_feat, widths, seed=4)
    m = PointnetSAModule(npoint=P, radius=1.0, nsample=ns, mlp=[c_feat] + widths, bn=False).train()
    with torch.no_grad():
        for layer, lay in zip(m.mlps[0].children(), case["layers"]):
            layer.conv.weight.copy_(lay["w"].view_as(layer.conv.weight))
            layer.conv.bias.copy_(lay["b"])
    return m, case["xyz"], case["centres"], case["feats"], case["idx"].long(), case["grad_out"]


def _torch_module_run(m, xyz, centres, feats, idx, gout):
    """the torch module itself in float64 on the same grouping, with autograd -> (out, feature gradient, module)"""
    md = copy.deepcopy(m).double()
    f = feats.double().requires_grad_(True)
    bi = torch.arange(xyz.shape[0])[:, None, None]
    rel = (xyz.double()[bi, idx] - centres.double()[:, :, None, :]).permute(0, 3, 1, 2)
    grouped = torch.cat([rel, f.transpose(1, 2)[bi, idx].permute(0, 3, 1, 2)], 1)
    y = md.mlps[0](grouped)
    out = nn.functional.max_pool2d(y, kernel_size=[1, y.size(3)]).squeeze(-1)
    out.backward(gout.double())
    return out, f.grad, md


def test_reference_matches_the_torch_module_in_float64():
    """the float64 reference is the torch module's own math: grouping, conv, train-mode BN, ReLU, max-pool, autograd"""
    m, xyz, centres, feats, idx, gout = _case()
    layers = R.layer_params(m.mlps[0])
    ref = R.scale(xyz, centres, feats, idx, layers, gout)
    out, f_grad, md = _torch_module_run(m, xyz, centres, feats, idx, gout)
    assert torch.allclose(out, ref["out"], rtol=1e-10, atol=1e-12)
    assert torch.allclose(f_grad, ref["feats"], rtol=1e-8, atol=1e-10)
    for l, layer in enumerate(md.mlps[0].children()):
        assert torch.allclose(layer.conv.weight.grad.flatten(1), ref["w"][l], rtol=1e-8, atol=1e-10)
        bn = layer.bn.bn
        assert torch.allclose(bn.weight.grad, ref["gamma"][l], rtol=1e-8, atol=1e-10)
        assert torch.allclose(bn.running_var, ref["running"][l][1], rtol=1e-10)
        assert int(bn.num_batches_tracked) == ref["running"][l][2]


def test_reference_equals_the_torch_module_on_an_integer_bias_chain():
    """on an integer-valued bias-only chain both the reference and the torch module are exact: they agree exactly"""
    m, xyz, centres, feats, idx, gout = _integer_bias_case()
    layers = R.layer_params(m.mlps[0])
    ref = R.scale(xyz, centres, feats, idx, layers, gout)
    R.check_exact(dict(xyz=xyz, centres=centres, feats=feats, idx=idx, layers=layers), ref)
    out, f_grad, md = _torch_module_run(m, xyz, centres, feats, idx, gout)
    assert torch.equal(out, ref["out"]) and torch.equal(f_grad, ref["feats"])
    assert f_grad.abs().max() > 0
    for l, layer in enumerate(md.mlps[0].children()):
        assert torch.equal(layer.conv.weight.grad.flatten(1), ref["w"][l]), l
        assert torch.equal(layer.conv.bias.grad, ref["b"][l]), l


# ---------------------------------------------------------------------------------------------- exact integer cases
EXACT_CASES = [
    # B, N, npoint, ns, c_feat, widths, bn, group_all
    (1, 40, 3, 4, 0, [1], False, False),
    (2, 300, 37, 8, 29, [40, 63, 64], False, False),
    (2, 200, 9, 64, 62, [196], False, False),
    (1, 600, 6, 16, 509, [512, 1, 24], False, False),
    (2, 100, 11, 4, 128, [64, 65, 40], False, False),
    (3, 500, 41, 32, 1, [32, 32, 64], True, False),
    (4, 32, 1, 32, 256, [256, 256, 512], False, True),
]


def _exact_case(B, N, npoint, ns, c_feat, widths, bn, group_all):
    case = R.integer_case(B, N, npoint, ns, c_feat, widths, seed=B * 7 + ns + c_feat, bn=bn, group_all=group_all)
    ref = R.scale(case["xyz"], case["centres"], case["feats"], case["idx"], case["layers"], None if bn else case["grad_out"])
    return case, ref


@pytest.mark.parametrize("B,N,npoint,ns,c_feat,widths,bn,group_all", EXACT_CASES)
def test_exactness_check_accepts_the_generated_cases(B, N, npoint, ns, c_feat, widths, bn, group_all):
    case, ref = _exact_case(B, N, npoint, ns, c_feat, widths, bn, group_all)
    R.check_exact(case, ref, layers_exact=1 if bn else None)
    idx = case["idx"].long()
    assert (idx[:, :, 1:] == idx[:, :, :1]).any() or group_all, "no ball-query padding"
    assert int(idx[-1, -1].max()) == N - 1
    if not bn:
        assert all(int((dz != 0).any(1).sum()) > 0 for dz in ref["dz"]), "a layer without gradient"
    w0 = case["layers"][0]["w"]
    assert (w0 != 0).any(0).all(), "an input column no weight reads"


def test_exactness_check_rejects_a_tf32_operand_of_2049():
    case, _ = _exact_case(2, 300, 37, 8, 29, [40, 63, 64], False, False)
    case["feats"][0, 5, case["idx"][0, 0, 0]] = 2049.0
    ref = R.scale(case["xyz"], case["centres"], case["feats"], case["idx"], case["layers"], case["grad_out"])
    with pytest.raises(AssertionError, match="layer 0 input reaches 2049"):
        R.check_exact(case, ref)


def test_exactness_check_rejects_an_absolute_sum_of_2_to_the_24():
    """four products of 2048 x 2048 in one row of |A| |W|^T: every operand is allowed, their sum is not"""
    case, _ = _exact_case(2, 300, 37, 8, 4, [8], False, False)
    case["feats"][0, :, case["idx"][0, 0, 0]] = 2048.0
    w = case["layers"][0]["w"]
    w[0, 3:7] = 2048.0
    ref = R.scale(case["xyz"], case["centres"], case["feats"], case["idx"], case["layers"], case["grad_out"])
    with pytest.raises(AssertionError, match="layer 0 forward"):
        R.check_exact(case, ref)
    w[0, 6] = 2047.0                                    # one below: 2^24 - 2^11 plus the other columns still passes
    w[0, :3] = 0.0
    ref = R.scale(case["xyz"], case["centres"], case["feats"], case["idx"], case["layers"], case["grad_out"])
    R.check_exact(case, ref)

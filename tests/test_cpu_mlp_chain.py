"""The MLP chains the modules build (pointrcnn_b200/mlp_chain.py), checked on the host: the packed image, scale, shift and
descriptor of every chain of seeded modules are pinned by sha256, and a chain packed for one entry point or width is
refused by the others before anything is launched."""
import hashlib

import numpy as np
import pytest
import torch
import torch.nn as nn

from pointrcnn_b200 import config
from pointrcnn_b200 import mlp_chain as M
from pointrcnn_b200.backbone import Pointnet2MSG
from pointrcnn_b200.pointnet2 import pointnet2_modules as pm
from pointrcnn_b200.pointnet2 import pytorch_utils as pt_utils
from pointrcnn_b200.rcnn.stage import RCNNStage
from pointrcnn_b200.rpn import heads


def _seeded(module, seed):
    """every float parameter and buffer drawn from one generator; channel 0 of every BN gets bias -0.0 and mean 0 with a
    positive scale, so its shift is -0.0 unless the fold adds a zero bias term"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, t in list(module.named_parameters()) + list(module.named_buffers()):
            if not t.is_floating_point():
                continue
            if name.endswith("running_var"):
                t.copy_(torch.rand(t.shape, generator=g) + 0.5)
            else:
                t.copy_(torch.randn(t.shape, generator=g) * 0.2)
        for m in module.modules():
            if isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d)):
                m.weight[0] = m.weight[0].abs()
                m.bias[0], m.running_mean[0] = -0.0, 0.0
    return module.eval()


def _digest(chain):
    h = hashlib.sha256()
    for t in (chain.packed, chain.scale, chain.shift):
        if t is None:
            h.update(b"none")
        else:
            a = t.detach().cpu().contiguous().numpy()
            h.update(np.int64(a.size).tobytes() + a.tobytes())
    d = chain.desc
    fields = [d.num_layers, d.c_in] + list(d.c_out) + [d.flags, d.scale is not None]
    h.update(np.array(fields, np.int64).tobytes())
    return h.hexdigest()


SKIP = [1, 96, 256, 512]    # skip channels of FP k in Pointnet2MSG(input_channels=1)


def _chains():
    """{name: chain} of the seeded backbone (fold_scale on and off, FP projection split), RPN heads and RCNN row MLPs"""
    out = {}
    net = _seeded(Pointnet2MSG(input_channels=1), 1)
    rpn_cls = nn.Sequential(pt_utils.Conv1d(128, 128, bn=True), nn.Dropout(0.5), pt_utils.Conv1d(128, 1, activation=None))
    rpn_reg = nn.Sequential(pt_utils.Conv1d(128, 128, bn=True), nn.Dropout(0.5), pt_utils.Conv1d(128, 76, activation=None))
    _seeded(rpn_cls, 2), _seeded(rpn_reg, 3)
    rcnn = {bn: _seeded(RCNNStage(cfg=dict(USE_BN=bn)), 4 + bn) for bn in (False, True)}
    for fold in (True, False):
        with config.override(fold_scale=fold):
            for k, sa in enumerate(net.SA_modules):
                for i, mlp in enumerate(sa.mlps):
                    out["sa%d.%d fold=%d" % (k, i, fold)] = pm._FusedMLP().get(mlp, M.SA, mlp[0].conv.in_channels - 3, "cpu")
            for k, fp in enumerate(net.FP_modules):
                c_known = fp.mlp[0].conv.in_channels - SKIP[k]
                out["fp%d fold=%d" % (k, fold)] = pm._FusedMLP().get(fp.mlp, M.FP, c_known, "cpu")
    with config.override(fold_scale=True):
        for k, fp in enumerate(net.FP_modules):
            c_known = fp.mlp[0].conv.in_channels - SKIP[k]
            if fp.mlp[0].conv.out_channels < c_known:
                f = pm._FusedMLP()
                out["fp%d projected" % k] = f.get(fp.mlp, M.FP, c_known, "cpu", project_known=True)
                out["fp%d projection" % k] = f.proj
        out["rpn heads"] = heads.FusedRPNHeads._build(rpn_cls, rpn_reg, "cpu")[0]
        for bn, r in rcnn.items():
            c_up = r.xyz_up_layer[-1].conv.out_channels
            out["rcnn xyz_up bn=%d" % bn] = pm._FusedMLP().get(r.xyz_up_layer, *M.rows_layout(r.rcnn_input_channel, 0), "cpu")
            out["rcnn merge bn=%d" % bn] = pm._FusedMLP().get(r.merge_down_layer, *M.rows_layout(c_up, c_up), "cpu")
    return out


# captured from the per-module packing code this module replaced
PINNED = {
    "sa0.0 fold=1": "c2f9cbf949bb5953493aeee264798fed9a860f040eb8479f96f573ab12aebf57",
    "sa0.1 fold=1": "f047bdb745cb30bcca35cd47b822559a450dc416542d26e9f93b598a0e6bd276",
    "sa1.0 fold=1": "660b1cde747132adf5cdfd7688fbc9500bf964c58f34a8a09f91ddb8dbf828b8",
    "sa1.1 fold=1": "bb8efa8b38f4f83e9eaff29c05c6e326f6b53bffe9573ddc03cff44a7a43ee64",
    "sa2.0 fold=1": "4241dad6092e87ff7185f559b8383d26ec973745d1c24025ce80062f701b6132",
    "sa2.1 fold=1": "3cad08d5b038c6aae108b2953c0432b95eb4aebe831eabd6b612f0d939ceb101",
    "sa3.0 fold=1": "4c8113d826a02604c0b8b47721df18ca9ff704932be618fb0c4b072e68cb93e6",
    "sa3.1 fold=1": "2ee1157cf0f88bd50f7b3fe16da8caff3d3b7f627faeafea2fb97d0b5c2568b1",
    "fp0 fold=1": "14a5bbaeec5de4a5d6d26a3d5869e64c29fb49d4fe6012a320484fc2163b61f1",
    "fp1 fold=1": "a055d6bc78d543ea2eba2d82711e72bdc29f90a2b63d6adebd71df65590ec44a",
    "fp2 fold=1": "3c2d2068960a0e0c0bfeba2a0b5645a4004c76b65144746f44b742b8794be912",
    "fp3 fold=1": "dc69fd75c2fd1ff68f519189cb1e427a44d2813e115b830f05f4ff9f843583a5",
    "sa0.0 fold=0": "a88d1c20016af6913175620b836fa217d7293ffc9448ddeb9ef17791128a125b",
    "sa0.1 fold=0": "708faf1d3fb1ca193bf4f4671b3edd99b7c0e3e3b05b400a14db5720e1e971af",
    "sa1.0 fold=0": "0db34dd50442f7a5edf26938cfbd41e774bcb40b57b7139003f31f2261e44f9a",
    "sa1.1 fold=0": "c308de802f6b2ceb73025a98e56a82864f46eedf5e450c6e071a7eb26b0fa584",
    "sa2.0 fold=0": "f2404f493b88c7cb5eae299679805f2010bc4c1e2b85242084484d1c47564d8d",
    "sa2.1 fold=0": "844de2bd162ef12066f4f4177ea03230058c565eddd146fa2e6489356e5cd28d",
    "sa3.0 fold=0": "042e132b343b8cba54016d72cf8e57c24a91979062a6d55efb57de3d176d1c47",
    "sa3.1 fold=0": "c39247f126102e111c260bac3192e47dd6a041c2a2eb3c928d160a430a2fbf4f",
    "fp0 fold=0": "d731a694acd6c679767ec6f937cd609ce81b4d327709ab330b39fe33cfaf8dfd",
    "fp1 fold=0": "879c0cbcc2718e5f7a8e634ac8238a22ab24c139c420a2d43e9687eaa1b97e12",
    "fp2 fold=0": "59fde64be84398568e08a309ec577f381f4aa3101e70d51e17974c8f076f0f36",
    "fp3 fold=0": "e7507f43aafa06ed6218db963b346a7299a5f2f83a75a05786322a67f090c26a",
    "fp0 projected": "0265e34df11a701be38cd9e11fc579f1aee325b5df04219101fac3a5197361a5",
    "fp0 projection": "7713b57410022e3e4d3afd3ad1d43e1b3cfe233c4f21960fae0dc8afbe42eb58",
    "fp1 projected": "bd0a384c7d2d42049a626aada197690881d642d11a9e102393494f67a99cfd47",
    "fp1 projection": "7dfa97b31974e2776c7fbfe0760c82d36a22b2a0539fd385d45b92c15a1c1cce",
    "fp3 projected": "8312537472d6eb398a0b770b0270b49f98b86b25c5fe1b474e7b02218eb704fd",
    "fp3 projection": "bccb15db2ccb62e74e90e47873b3936aa5b8a6f01a821258cd1a85246ac5e8c7",
    "rpn heads": "fec47538eee1637773d32b64ba2c275dbf4d67800240b5d76a884e1ccd74a961",
    "rcnn xyz_up bn=0": "541fce5f641bbd0884ecad467409962a0d7eb0f3440b99b495015ac3566e57cd",
    "rcnn merge bn=0": "f24cc25863f3a729c4d2980d17e2cf732b305abb799a155101cf466f225dba8c",
    "rcnn xyz_up bn=1": "7fdc75dda38307bc56e3701db0982c245d3ecdce596fa5d308636a0e030a99b9",
    "rcnn merge bn=1": "5ead9ae51727488a17b28d284d82a07d525a0f78a4f4b7942fa66b099c3511d4",
}


def test_module_chains_match_the_pinned_images():
    got = {name: _digest(chain) for name, chain in _chains().items()}
    assert sorted(got) == sorted(PINNED)
    bad = [name for name in PINNED if got[name] != PINNED[name]]
    assert not bad, "packed image, scale, shift or descriptor changed: %s" % bad


def test_fold_zero_bias_differs_only_in_the_sign_of_a_zero_shift():
    """the heads' fold adds scale * 0 for a missing conv bias: the -0.0 shift of channel 0 becomes +0.0, nothing else moves"""
    conv = pt_utils.Conv1d(16, 8, bn=True)
    _seeded(conv, 9)
    W, s, t = M.fold(conv.conv, conv.bn.bn)
    Wz, sz, tz = M.fold(conv.conv, conv.bn.bn, zero_bias=True)
    assert s is None and sz is None and torch.equal(W, Wz)
    assert t[0].item() == 0.0 and np.signbit(t[0].item()) and not np.signbit(tz[0].item())
    assert torch.equal(t[1:].view(torch.int32), tz[1:].view(torch.int32))


def _cpu(*shape):
    return torch.zeros(shape)


def _sa(chain, c_feat):
    chain.sa(_cpu(2, 64, 3), _cpu(2, 8, 3), _cpu(2, 64, c_feat) if c_feat else None, torch.zeros((2, 8, 16), dtype=torch.int32), 16,
             _cpu(2, chain.c_out[-1], 8), None, 0)


def _fp(chain, c_known, c_skip):
    chain.fp(_cpu(2, 16, c_known), torch.zeros((2, 40, 3), dtype=torch.int32), _cpu(2, 40, 3), _cpu(2, c_skip, 40) if c_skip else None,
             _cpu(2, chain.c_out[-1], 40), None)


def _rows(chain, c_a, c_b):
    chain.rows(_cpu(50, c_a), _cpu(50, c_b) if c_b else None)


def _chain(kind, split, c_in):
    rng = np.random.default_rng(c_in)
    return M.Chain(kind, split, [rng.standard_normal((32, c_in)).astype(np.float32)], [np.zeros(32, np.float32)], device="cpu")


@pytest.mark.parametrize("packed,launch", [
    ((M.SA, 6, 9), lambda ch: _rows(ch, 9, 0)),           # SA image (feats first) read as plain rows
    ((M.SA, 6, 9), lambda ch: _fp(ch, 6, 3)),
    ((M.SA, 1, 4), lambda ch: _sa(ch, 2)),                # another c_feat
    ((M.ROWS, 0, 9), lambda ch: _sa(ch, 6)),              # plain rows read as [xyz | 6 feats]
    ((M.FP, 64, 65), lambda ch: _sa(ch, 62)),
    ((M.FP, 64, 65), lambda ch: _fp(ch, 63, 2)),          # another split between interpolated and skip channels
    ((M.FP, 64, 65), lambda ch: _fp(ch, 64, 2)),          # another width
    ((M.FP, 64, 65), lambda ch: _rows(ch, 65, 0)),        # two segments read as one
    ((M.ROWS, 0, 65), lambda ch: _rows(ch, 64, 1)),       # one segment read as two
    ((M.ROWS, 0, 65), lambda ch: _fp(ch, 64, 1)),
    ((M.ROWS, 0, 65), lambda ch: _rows(ch, 66, 0)),
])
def test_launch_refuses_a_chain_packed_for_another_entry_point(packed, launch):
    """nothing reaches the library: the check raises on CPU tensors, before any workspace or launch"""
    chain = _chain(*packed)
    with pytest.raises(ValueError, match="packed as kind %d, split %d, %d channels" % packed):
        launch(chain)


def test_pack_rejects_layers_that_do_not_chain():
    with pytest.raises(ValueError, match="layer 1 takes 20 inputs"):
        M.pack_image(M.ROWS, 0, [np.zeros((16, 8), np.float32), np.zeros((32, 20), np.float32)])
    with pytest.raises(TypeError):
        M.pack_image(M.ROWS, 0, [np.zeros((16, 8))])

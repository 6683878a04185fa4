"""The fused eval modules on the device against module_reference.py's float64 evaluation of their own torch parameters,
element by element: the SA / FP levels of the RPN backbone at batch 16 (every MSG channel slice, both fold_scale modes,
the FP projection on, off and as dispatched, with and without point-major twins), the RCNN SA stack on duplicate-padded
pooled clouds, the fused RPN heads with a valid, a missing and a stale twin, the RCNN row MLP pair, and the whole
backbone level by level through forward hooks.  Index work (FPS, ball query, 3-NN) is the device's own.  Each check
prints its max err / bound.

The packed-weight caches are checked here too: after a parameter replacement that reuses the old one's id(),
load_state_dict(assign=True), .cpu(), an in-place edit and .cuda(), or a .data edit and invalidate_fused(), a module's
output is bit-identical to a freshly built module's."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import module_reference as MR

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import config  # noqa: E402
from pointrcnn_b200.backbone import Pointnet2MSG  # noqa: E402
from pointrcnn_b200.pointnet2 import pointnet2_modules as pm  # noqa: E402
from pointrcnn_b200.rcnn.stage import RCNNStage  # noqa: E402
from pointrcnn_b200.rpn.heads import rpn_heads  # noqa: E402
from pointrcnn_b200.rpn.stage import RPNStage  # noqa: E402

B = 16          # BASELINE configs[1]: 16 scenes of 16384 points x 4 channels (bench.make_scenes)


def within(got, ref, bound, label):
    ok, ratio, bad = MR.check(got, ref, bound)
    print("%-44s max err/bound %.3f" % (label, ratio))
    assert ok, "%s: %d of %d elements outside the bound, max err/bound %.3g" % (label, bad, got.numel(), ratio)


def twin_is_transpose(out, label):
    twin = getattr(out, "_prb_pm", None)
    assert twin is not None, "%s: no point-major twin" % label
    assert torch.equal(twin[0], out.transpose(1, 2).contiguous()), "%s: the twin is not the transpose" % label


@pytest.fixture(scope="module")
def scenes(cuda):
    import bench
    pc = torch.from_numpy(bench.make_scenes(700, B)).to(cuda)
    return pc[..., :3].contiguous(), pc[..., 3:].transpose(1, 2).contiguous()


@pytest.fixture(scope="module")
def backbone(cuda):
    torch.manual_seed(3)
    return MR.seeded(Pointnet2MSG(input_channels=1), 5).to(cuda)


def check_sa(sa, xyz, feats, new_xyz, out, label):
    """every MSG channel slice of `out` against the reference of its scale, on the device's centres and ball queries"""
    _, centres, idxs, _ = sa.fused_geometry(xyz, new_xyz)
    off = 0
    for s, (mlp, idx) in enumerate(zip(sa.mlps, idxs)):
        ref, bound = MR.sa_scale(mlp, xyz, feats, centres, idx)
        c = ref.size(1)
        within(out[:, off:off + c], ref, bound, "%s scale %d" % (label, s))
        off += c
    assert off == out.size(1)


def check_fp(fp, unknown, known, skip, known_feats, out, label):
    idx, weight = fp.fused_geometry(unknown, known)
    projected = fp._fused.proj is not None
    ref, bound = MR.fp_module(fp.mlp, idx, weight, skip, known_feats, projected)
    within(out, ref, bound, "%s%s" % (label, " (projected)" if projected else ""))
    return projected


def sa_levels(net, xyz, feats):
    l_xyz, l_f = [xyz], [feats]
    for sa in net.SA_modules:
        nx, nf = sa(l_xyz[-1], l_f[-1])
        l_xyz.append(nx)
        l_f.append(nf)
    return l_xyz, l_f


# ------------------------------------------------------------------------------------------------ RPN backbone levels
@pytest.mark.parametrize("fold", [True, False])
def test_rpn_sa_levels_within_bound(backbone, scenes, fold):
    xyz, feats = scenes
    with torch.no_grad(), config.override(fold_scale=fold):
        for k, sa in enumerate(backbone.SA_modules):
            nx, out = sa(xyz, feats)
            label = "SA%d fold_scale=%d" % (k + 1, fold)
            check_sa(sa, xyz, feats, nx, out, label)
            twin_is_transpose(out, label)
            xyz, feats = nx, out


@pytest.fixture(scope="module")
def sa_outputs(backbone, scenes):
    with torch.no_grad():
        return sa_levels(backbone, *scenes)


FP_FORMS = {"dispatched": {}, "projection forced on": dict(fp_project_min_rows=0), "projection off": dict(fp_project=False)}


@pytest.mark.parametrize("emit", [True, False])
@pytest.mark.parametrize("form", sorted(FP_FORMS))
def test_rpn_fp_levels_within_bound(backbone, sa_outputs, form, emit):
    l_xyz, l_f = sa_outputs
    l_f = list(l_f)
    fps = backbone.FP_modules
    saved = [fp.emit_point_major for fp in fps]
    projected = []
    try:
        with torch.no_grad(), config.override(**FP_FORMS[form]):
            for i in range(-1, -(len(fps) + 1), -1):
                fp = fps[i]
                fp.emit_point_major = emit
                out = fp(l_xyz[i - 1], l_xyz[i], l_f[i - 1], l_f[i])
                label = "FP%d %s emit_pm=%d" % (len(fps) + i, form, emit)
                projected.append(check_fp(fp, l_xyz[i - 1], l_xyz[i], l_f[i - 1], l_f[i], out, label))
                if emit:
                    twin_is_transpose(out, label)
                else:
                    assert not hasattr(out, "_prb_pm"), "%s: a twin was written" % label
                l_f[i - 1] = out
    finally:
        for fp, e in zip(fps, saved):
            fp.emit_point_major = e
    projected = projected[::-1]          # FP0 first
    narrows = [fp.mlp[0].conv.out_channels < fp.mlp[0].conv.in_channels - (1, 96, 256, 512)[k] for k, fp in enumerate(fps)]
    want = {"dispatched": [True, False, False, False], "projection forced on": narrows,
            "projection off": [False] * 4}[form]
    assert projected == want, "%s: projected levels %s" % (form, projected)


def test_backbone_b16_level_by_level_within_bound(backbone, scenes):
    """the whole backbone forward, each module's output against its reference on the inputs it was given (hooks)"""
    xyz, feats = scenes
    seen = []
    hooks = [m.register_forward_hook(lambda mod, args, out: seen.append((mod, args, out)))
             for m in list(backbone.SA_modules) + list(backbone.FP_modules)]
    try:
        with torch.no_grad():
            backbone(torch.cat([xyz, feats.transpose(1, 2)], 2))
    finally:
        for h in hooks:
            h.remove()
    assert len(seen) == 8
    with torch.no_grad():
        for mod, args, out in seen:
            if isinstance(mod, pm.PointnetFPModule):
                check_fp(mod, *args, out, "backbone FP%d" % list(backbone.FP_modules).index(mod))
            else:
                check_sa(mod, args[0], args[1], out[0], out[1], "backbone SA%d" % (list(backbone.SA_modules).index(mod) + 1))


# ------------------------------------------------------------------------------------------------ RCNN
def pooled_clouds(rois, points, channels, seed, dev):
    """canonical pooled RoI clouds: roi r has cnt_r distinct points and point k is point k % cnt_r (the pooling's
    duplicate padding); counts 1 and 2 included"""
    rng = np.random.default_rng(seed)
    cnt = rng.integers(1, points + 1, rois)
    cnt[:3] = (1, 2, points)
    base = rng.standard_normal((rois, points, 3 + channels)).astype(np.float32)
    base[..., :3] *= np.float32(0.8)
    k = np.arange(points)[None, :] % cnt[:, None]
    return torch.from_numpy(np.take_along_axis(base, k[..., None], 1)).to(dev)


@pytest.mark.parametrize("bn", [False, True])
def test_rcnn_sa_stack_within_bound(cuda, bn):
    torch.manual_seed(9)
    r = MR.seeded(RCNNStage(cfg=dict(USE_BN=bn)), 17 + bn).to(cuda)
    pts = pooled_clouds(96, 512, 128, 3 + bn, cuda)
    xyz, feats = pts[..., :3].contiguous(), pts[..., 3:].transpose(1, 2).contiguous()
    with torch.no_grad():
        for k, sa in enumerate(r.SA_modules):
            nx, out = sa(xyz, feats)
            if sa.npoint is None:
                assert out.shape == (96, 512, 1)
                nx = None
            check_sa(sa, xyz, feats, nx, out, "RCNN SA%d bn=%d" % (k + 1, bn))
            twin_is_transpose(out, "RCNN SA%d" % (k + 1))
            xyz, feats = nx, out


@pytest.mark.parametrize("bn", [False, True])
def test_rcnn_rows_mlp_pair_within_bound(cuda, bn):
    torch.manual_seed(10)
    r = MR.seeded(RCNNStage(cfg=dict(USE_BN=bn)), 19 + bn).to(cuda)
    ci = r.rcnn_input_channel
    rows = pooled_clouds(128, 512, ci - 3 + 128, 5, cuda).view(128 * 512, -1)
    fused = (pm._FusedMLP(), pm._FusedMLP())
    with torch.no_grad():
        up = pm.rows_mlp(fused[0], r.xyz_up_layer, rows[:, :ci])
        merged = pm.rows_mlp(fused[1], r.merge_down_layer, up, rows[:, ci:])
    within(up, *MR.rows_mlp(r.xyz_up_layer, rows[:, :ci]), "RCNN xyz_up bn=%d" % bn)
    within(merged, *MR.rows_mlp(r.merge_down_layer, up, rows[:, ci:]), "RCNN merge bn=%d" % bn)


# ------------------------------------------------------------------------------------------------ RPN heads
@pytest.fixture(scope="module")
def rpn(cuda):
    torch.manual_seed(5)
    return MR.seeded(RPNStage(), 23).to(cuda)


@pytest.mark.parametrize("twin", ["valid", "none", "stale"])
def test_fused_rpn_heads_within_bound(rpn, cuda, twin):
    n = 16384
    f = torch.randn(B, 128, n, device=cuda, generator=torch.Generator(cuda).manual_seed(1)).relu_()
    if twin != "none":
        f = pm._attach_pm(f, f.transpose(1, 2).contiguous())
    if twin == "stale":
        f.mul_(-0.5).add_(1.0)          # in place: the twin no longer matches, the heads must transpose again
    with torch.no_grad():
        cls, reg = rpn_heads(rpn, f)
    rows = f.transpose(1, 2).reshape(B * n, 128)
    (rc, bc), (rr, br) = MR.heads(rpn.rpn_cls_layer, rpn.rpn_reg_layer, rows)
    within(cls.view(B * n, -1), rc, bc, "RPN heads cls, twin %s" % twin)
    within(reg.view(B * n, -1), rr, br, "RPN heads reg, twin %s" % twin)


# ------------------------------------------------------------------------------------------------ caches on the device
BUILD = {
    "sa": lambda: pm.PointnetSAModuleMSG(npoint=256, radii=[0.2, 0.4], nsamples=[16, 32], mlps=[[8, 16, 32], [8, 32, 64]]),
    "fp": lambda: pm.PointnetFPModule(mlp=[64 + 8, 32, 48]),      # c_out0 < c_known: projected below
    "heads": RPNStage,
}


def _build(kind, dev, seed):
    return MR.seeded(BUILD[kind](), seed).to(dev)


def _cache_inputs(dev):
    g = torch.Generator().manual_seed(4)
    xyz = torch.rand(2, 2048, 3, generator=g)
    return [t.to(dev) for t in (xyz, torch.randn(2, 8, 2048, generator=g), xyz[:, :512].contiguous(),
                                torch.randn(2, 64, 512, generator=g), torch.randn(2, 128, 512, generator=g))]


def _run(kind, mod, inputs):
    xyz, feats, known, known_feats, head_feats = inputs
    with torch.no_grad(), config.override(fp_project_min_rows=0):
        if kind == "sa":
            return mod(xyz, feats)[1]
        if kind == "fp":
            return mod(xyz, known, feats, known_feats)
        return torch.cat(rpn_heads(mod, head_feats), 2)


def _conv(kind, mod):
    return mod.rpn_reg_layer[0].conv if kind == "heads" else next(m for m in mod.modules() if isinstance(m, nn.Conv2d))


def replace_reusing_id(kind, mod, dev):
    """a new nn.Parameter that takes the freed slot, so the id() and version 0 of the one it replaces whenever nothing but
    an id() remembers that one (MR.replace_parameter; from the second change on, the old parameter is itself version 0)"""
    conv = _conv(kind, mod)
    MR.replace_parameter(conv, "weight", torch.randn(conv.weight.shape, device=dev) * 0.3)


def load_assign(kind, mod, dev):
    mod.load_state_dict(_build(kind, dev, 41).state_dict(), assign=True)


def cpu_edit_cuda(kind, mod, dev):
    mod.cpu()
    with torch.no_grad():
        _conv(kind, mod).weight.mul_(-1.5)
    mod.to(dev)


def data_edit_invalidate(kind, mod, dev):
    """a write through .data bumps no version counter: invalidate_fused() is the way to drop the chain"""
    _conv(kind, mod).weight.data.mul_(0.5)
    mod.invalidate_fused()


@pytest.mark.parametrize("change", [replace_reusing_id, load_assign, cpu_edit_cuda, data_edit_invalidate], ids=lambda f: f.__name__)
@pytest.mark.parametrize("kind", sorted(BUILD))
def test_cache_after_a_parameter_change_matches_a_fresh_module(cuda, kind, change):
    inputs = _cache_inputs(cuda)
    mod = _build(kind, cuda, 40)
    for rep in range(3):               # each change three times over, from a chain the call before cached
        _run(kind, mod, inputs)
        change(kind, mod, cuda)
        got = _run(kind, mod, inputs)
        fresh = BUILD[kind]().to(cuda).eval()
        fresh.load_state_dict(mod.state_dict())
        assert torch.equal(got, _run(kind, fresh, inputs)), "%s, %s #%d: the cached chain is stale" % (kind, change.__name__, rep)

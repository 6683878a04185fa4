"""GPU tests of the wgmma MLP chain and of the fused SA / FP module paths.

Tolerances.  The reference's MLP is torch.nn.Conv2d (cuDNN, TF32 allowed by torch's default) and is not
pinned by any reference test (SURVEY.md 8c).  Two checks:
  tight : against an fp32 numpy evaluation whose OPERANDS are rounded to TF32 exactly as the kernel does
          (weights at pack time, activations per layer) -- only the fp32 accumulation order differs, so any
          layout / descriptor / pipeline bug shows up as a gross error.  One layer: |err| <= 2e-4*(1+|ref|)
          everywhere.  Chains: an intermediate activation that sits on a TF32 rounding boundary may round the
          other way (1 tf32 ulp = 1e-3 rel) and moves every output of the next layer a little, so for chains
          97% of the outputs must meet 2e-4 and all of them 5e-3.
  fp32  : against the plain fp32 oracle / fp32 torch evaluation: max|err| <= 2e-3 * max|ref| -- the a6 / a11 contract of
          SURVEY.md 8(c) (TF32 operands, fp32 accumulation, up to three chained layers).
"""
import ctypes

import numpy as np
import pytest
import torch

import synth
from oracle import oracle as O

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200.backbone import Pointnet2MSG  # noqa: E402
from pointrcnn_b200.mlp_chain import Chain  # noqa: E402
from pointrcnn_b200.pointnet2 import pointnet2_modules as pm  # noqa: E402
from pointrcnn_b200.pointnet2 import pointnet2_utils as pu  # noqa: E402



TOL_BACKBONE = 5e-3   # the whole backbone chains 8 levels (20 TF32 layers); per-op contract is TOL
TOL = 2e-3      # SURVEY.md 8(c): a6 / a11 parity vs an fp32 evaluation of the same weights (norm-wise: max|err| / max|ref|)

def tf32(x):
    """cvt.rna.tf32.f32 on a numpy array"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).copy()
    finite = (u & 0x7F800000) != 0x7F800000
    u[finite] += 0x1000
    u &= 0xFFFFE000
    return u.view(np.float32)


def tf32_rn(x):
    """cvt.rn.tf32.f32 (round to nearest even), used for the activations between layers (fused with the ReLU)"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    lsb = (u >> 13) & 1
    u = (u + 0xFFF + lsb) & 0xFFFFE000
    return u.astype(np.uint32).view(np.float32)


def mlp_tf32_ref(x, layers):
    """weights are rounded at pack time (host, ties away), every A operand built in registers with cvt.rn (ties even)"""
    h = x.astype(np.float32)
    for W, sc, sh in layers:
        h = tf32_rn(h) @ tf32(W).T
        h = np.maximum(h * sc[None] + sh[None], 0).astype(np.float32)
    return h


def _rand_layers(rng, dims):
    layers = []
    for ci, co in zip(dims[:-1], dims[1:]):
        W = (rng.standard_normal((co, ci)) * np.sqrt(2.0 / ci)).astype(np.float32)
        sc = rng.uniform(0.5, 1.5, co).astype(np.float32)
        sh = rng.normal(0, 0.2, co).astype(np.float32)
        layers.append((W, sc, sh))
    return layers


def _fold(layers):
    """BN scale folded into the weights: (W, s, t) -> (s * W, 1, t), the form the modules hand to the kernel"""
    return [((W * sc[:, None]).astype(np.float32), np.ones_like(sc), sh) for W, sc, sh in layers]


def _chain(layers, kind, split, dev, folded=False):
    """folded: `layers` come from _fold(); the descriptor then carries scale = NULL"""
    return Chain(kind, split, [l[0] for l in layers], [l[2] for l in layers], None if folded else [l[1] for l in layers],
                 device=dev)


ROW_CASES = [
    (128, [32, 32]),                 # one tile, one chunk, one K-step group: the smallest possible UMMA
    (128, [64, 64]),
    (1000, [40, 48]),                # K and N not multiples of 32, tail tile
    (4096, [99, 64, 64, 128]),       # SA2 scale 0 shape
    (3000, [259, 128, 196, 256]),    # SA3: N padded 196 -> 224
    (2000, [515, 256, 256, 512]),    # SA4 s0: split after two layers (N=512 layers: one launch each)
    (1500, [515, 256, 384, 512]),    # SA4 s1: every layer its own launch
    (20000, [257, 128, 128]),        # FP0, many tiles per CTA (ring wrap-around, phase bits)
    (700, [1536, 512, 512]),         # FP3: two N halves per K chunk
]


@pytest.mark.parametrize("rows,c_a,c_b,off_a,off_b,width,dims", [
    (4096, 5, 0, 0, 0, 133, [128, 128]),          # xyz_up_layer on the first 5 columns of the pooled rows (pitch 133: scalar loads)
    (4096, 128, 128, 0, 5, 133, [128]),           # merge_down_layer: [up rows (own tensor) | columns 5.. of the pooled rows]
    (1000, 40, 24, 4, 48, 80, [64, 32]),          # both segments slices of one 16-byte aligned tensor, tail tile
    (300, 33, 7, 1, 35, 45, [48]),                # misaligned slices, widths that are not multiples of 4
])
def test_mlp_rows2_strided_segments(cuda, rows, c_a, c_b, off_a, off_b, width, dims):
    """prb_mlp_rows2: layer 0 reads [a | b] from strided row views -- cat(xyz_feature, rpn_feature) of rcnn_net.py:171-175 is
    never materialised"""
    rng = np.random.default_rng(rows + c_a)
    layers = _rand_layers(rng, [c_a + c_b] + dims)
    wide = rng.standard_normal((rows, width)).astype(np.float32)
    own = rng.standard_normal((rows, c_a)).astype(np.float32)
    wt, ot = torch.from_numpy(wide).to(cuda), torch.from_numpy(own).to(cuda)
    if c_b and off_a == 0 and c_a == 128:          # the merge case: segment a is its own contiguous tensor
        a_t, a_np = ot, own
    else:
        a_t, a_np = wt[:, off_a:off_a + c_a], wide[:, off_a:off_a + c_a]
    b_t = wt[:, off_b:off_b + c_b] if c_b else None
    x = np.concatenate([a_np] + ([wide[:, off_b:off_b + c_b]] if c_b else []), axis=1)
    ch = _chain(layers, 1 if c_b else 2, c_a if c_b else 0, cuda, False)
    lib = C.lib()
    np_last = (dims[-1] + 31) // 32 * 32
    out = torch.full((rows, np_last), float("nan"), device=cuda)
    wsb = lib.prb_rows2_workspace_bytes(C.c_long(rows), c_a, c_b, len(layers), ch.co)
    ws = torch.empty(wsb, dtype=torch.uint8, device=cuda)
    C.check(lib.prb_mlp_rows2(C.c_long(rows), c_a, C.ptr(a_t), a_t.stride(0), c_b, C.ptr(b_t) if c_b else None,
                              b_t.stride(0) if c_b else 0, ctypes.byref(ch.desc), C.ptr(out), np_last, C.ptr(ws), C.c_size_t(wsb),
                              C.stream()), "mlp_rows2")
    torch.cuda.synchronize()
    got = out.cpu().numpy()[:, :dims[-1]]
    tight = mlp_tf32_ref(x, layers)
    err = np.abs(got - tight)
    assert (err <= 5e-3 * (1 + np.abs(tight))).all() and (err <= 2e-4 * (1 + np.abs(tight))).mean() >= 0.97, err.max()
    loose = O.shared_mlp(x, layers)
    assert np.abs(got - loose).max() <= TOL * np.abs(loose).max()


@pytest.mark.parametrize("folded", [False, True])
@pytest.mark.parametrize("rows,dims", ROW_CASES)
def test_mlp_rows_tcgen05(cuda, rows, dims, folded):
    rng = np.random.default_rng(rows + len(dims))
    layers = _rand_layers(rng, dims)
    if folded:
        layers = _fold(layers)
    x = rng.standard_normal((rows, dims[0])).astype(np.float32)
    ch = _chain(layers, 2, 0, cuda, folded)
    lib = C.lib()
    np_last = (dims[-1] + 31) // 32 * 32
    out = torch.full((rows, np_last), float("nan"), device=cuda)
    wsb = lib.prb_rows_workspace_bytes(C.c_long(rows), dims[0], len(layers), ch.co)
    ws = torch.empty(wsb, dtype=torch.uint8, device=cuda)
    xt = torch.from_numpy(x).to(cuda)
    C.check(lib.prb_mlp_rows(C.c_long(rows), dims[0], C.ptr(xt), ctypes.byref(ch.desc), C.ptr(out), np_last, C.ptr(ws),
                             C.c_size_t(wsb), C.stream()), "mlp_rows")
    torch.cuda.synchronize()
    got = out.cpu().numpy()[:, :dims[-1]]
    assert np.isfinite(got).all()
    tight = mlp_tf32_ref(x, layers)
    err = np.abs(got - tight)
    ok = err <= 2e-4 * (1 + np.abs(tight))
    if len(layers) == 1:
        assert ok.all(), "tight check failed: max err %g" % err.max()
    else:
        assert ok.mean() >= 0.97 and (err <= 5e-3 * (1 + np.abs(tight))).all(), "tight check failed: %g ok, max err %g" % (ok.mean(), err.max())
    loose = O.shared_mlp(x, layers)
    assert np.abs(got - loose).max() <= TOL * np.abs(loose).max()
    if np_last > dims[-1]:
        assert np.count_nonzero(out.cpu().numpy()[:, dims[-1]:]) == 0, "padding channels must be exactly zero"


# ------------------------------------------------------------------------------------------------ modules
def _randomise_bn(module, seed):
    g = torch.Generator().manual_seed(seed)
    for m in module.modules():
        if isinstance(m, (torch.nn.BatchNorm2d, torch.nn.BatchNorm1d)):
            m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
            m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
            m.weight.data.copy_(torch.rand(m.num_features, generator=g) + 0.5)
            m.bias.data.copy_(torch.randn(m.num_features, generator=g) * 0.1)


def _folded(mlp):
    layers = []
    for layer in mlp.children():
        conv = layer.conv
        bn = None
        if hasattr(layer, "bn"):
            b = layer.bn.bn
            bn = dict(weight=b.weight.detach().cpu().numpy(), bias=b.bias.detach().cpu().numpy(),
                      running_mean=b.running_mean.cpu().numpy(), running_var=b.running_var.cpu().numpy(), eps=b.eps)
        layers.append(O.fold_bn(conv.weight.detach().cpu().numpy(), None if conv.bias is None else conv.bias.detach().cpu().numpy(), bn))
    return layers


def _unfused(fn):
    from pointrcnn_b200 import config
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with config.override(disable_fused=True):
            return fn()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


SA_CASES = [
    # npoint, radii, nsamples, mlps, c_feat, N, cloud
    (256, [0.1, 0.2], [16, 32], [[16, 16, 32], [32, 32, 64]], 0, 2048, "cube"),      # SA1-like, no features
    (512, [0.1], [32], [[16, 32]], 1, 4096, "cube"),                                 # BASELINE config 1 shape (C0=1)
    (128, [0.2, 0.4], [16, 32], [[64, 64, 128], [64, 96, 128]], 96, 1024, "cube"),   # SA2
    (64, [0.3, 0.5], [16, 32], [[128, 196, 256], [128, 196, 256]], 256, 256, "cube"),  # SA3
    (16, [0.5, 0.9], [16, 32], [[256, 256, 512], [256, 384, 512]], 512, 64, "cube"),   # SA4 (split launches)
    (32, [0.4], [64], [[128, 128, 256]], 128, 128, "cube"),                          # RCNN SA2 (nsample 64)
]


@pytest.mark.parametrize("npoint,radii,nsamples,mlps,c_feat,N,kind", SA_CASES)
def test_sa_module_fused_vs_unfused_vs_oracle(cuda, npoint, radii, nsamples, mlps, c_feat, N, kind):
    torch.manual_seed(0)
    B = 2
    spec = [[c_feat] + list(m) for m in mlps]
    mod = pm.PointnetSAModuleMSG(npoint=npoint, radii=list(radii), nsamples=list(nsamples), mlps=spec, bn=True).to(cuda).eval()
    _randomise_bn(mod, 1)
    xyz = synth.u_cube(B, N, 5 + N)
    feats = np.random.default_rng(2).standard_normal((B, c_feat, N)).astype(np.float32) if c_feat else None
    x = torch.from_numpy(xyz).to(cuda)
    f = torch.from_numpy(feats).to(cuda) if c_feat else None
    with torch.no_grad():
        new_xyz, out = mod(x, f)
        ref_xyz, ref_out = _unfused(lambda: mod(x, f))
    assert torch.equal(new_xyz, ref_xyz)
    assert out.shape == ref_out.shape == (B, sum(m[-1] for m in mlps), npoint)
    scale = ref_out.abs().max().item()
    assert (out - ref_out).abs().max().item() <= TOL * scale, "fused SA differs from the op-by-op fp32 path"
    # CPU oracle (fp32) of the whole module
    o_xyz, o_out, _ = O.sa_module_msg(xyz, feats, npoint, radii, nsamples, [_folded(m) for m in mod.mlps])
    assert np.array_equal(new_xyz.cpu().numpy(), o_xyz)
    assert np.abs(out.cpu().numpy() - o_out).max() <= TOL * np.abs(o_out).max()
    # the point-major twin written by the same launch is the exact transpose, and it is dropped once
    # the channel-major tensor is modified in place
    twin = out._prb_pm[0]
    assert torch.equal(twin, out.transpose(1, 2).contiguous())
    assert pm._point_major(out) is twin
    out.mul_(2.0)
    fresh = pm._point_major(out)
    assert fresh is not twin and torch.equal(fresh, out.transpose(1, 2).contiguous())


@pytest.mark.parametrize("ns", [8, 16, 32, 64])
def test_sa_module_scale_fold_modes_agree(cuda, ns):
    """fold_scale=True (default: BN scale inside the weights, raw accumulators pooled, shift/ReLU after the max) against
    fold_scale=False (scale as an epilogue multiply); negative BN scales included -- max_s relu(x_s + t) = relu(max_s x_s + t)"""
    from pointrcnn_b200 import config
    torch.manual_seed(7)
    mod = pm.PointnetSAModuleMSG(npoint=200, radii=[0.25], nsamples=[ns], mlps=[[24, 64, 48, 96]], bn=True).to(cuda).eval()
    _randomise_bn(mod, 11)
    with torch.no_grad():
        for m in mod.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.data[::3] *= -1.0
    x = torch.from_numpy(synth.u_cube(2, 3000, 77)).to(cuda)
    f = torch.randn(2, 24, 3000, device=cuda)
    outs = {}
    for mode in ("0", "1"):
        with torch.no_grad(), config.override(fold_scale=(mode == "1")):
            outs[mode] = mod(x, f)[1]
    with torch.no_grad():
        ref = _unfused(lambda: mod(x, f))[1]
    scale = ref.abs().max().item()
    for mode in ("0", "1"):
        assert (outs[mode] - ref).abs().max().item() <= TOL * scale, "fold mode %s differs from the fp32 op-by-op path" % mode
    assert (outs["0"] - outs["1"]).abs().max().item() <= TOL * scale


@pytest.mark.parametrize("ns,widths", [(16, [16, 16, 32]), (32, [32, 32, 64])])
def test_sa_builds_bit_identical(cuda, ns, widths):
    """the launch plans of the chain (CTAs per SM, SMs of the persistent grid, resident or streamed weights;
    prb_options.mlp_occ / mlp_sms / mlp_resident) compute the same bits: K order and per-element arithmetic do not depend on
    the plan.  SA1-shaped chains (xyz + 1 feature channel) through the module."""
    from pointrcnn_b200 import _cabi as C
    torch.manual_seed(3 + ns)
    mod = pm.PointnetSAModuleMSG(npoint=700, radii=[0.3], nsamples=[ns], mlps=[[1] + widths], bn=True).to(cuda).eval()
    _randomise_bn(mod, 9)
    x = torch.from_numpy(synth.u_cube(3, 4000, 13)).to(cuda)
    f = torch.randn(3, 1, 4000, device=cuda)
    outs = []
    for opt in ({}, {"mlp_occ": 3}, {"mlp_occ": 1}, {"mlp_sms": 7}, {"mlp_resident": 0}, {"mlp_resident": 0, "mlp_occ": 1}):
        with torch.no_grad(), C.options(**opt):
            outs.append(mod(x, f)[1].clone())
    for k in range(1, len(outs)):
        assert torch.equal(outs[0], outs[k]), "build %d differs" % k
    with torch.no_grad():
        ref = _unfused(lambda: mod(x, f))[1]
    assert (outs[0] - ref).abs().max().item() <= TOL * ref.abs().max().item()


def test_sa_module_group_all_and_no_bn(cuda):
    torch.manual_seed(1)
    B, N, c_feat = 6, 32, 256
    mod = pm.PointnetSAModule(mlp=[c_feat, 256, 256, 512], npoint=None, radius=None, nsample=None, bn=False).to(cuda).eval()
    for p in mod.parameters():
        if p.dim() == 1:
            p.data.normal_(0, 0.1)   # non-zero conv biases
    xyz = torch.from_numpy(synth.u_cube(B, N, 3)).to(cuda)
    f = torch.randn(B, c_feat, N, device=cuda)
    with torch.no_grad():
        nx, out = mod(xyz, f)
        rx, ref = _unfused(lambda: mod(xyz, f))
    assert nx is None and rx is None
    assert out.shape == ref.shape == (B, 512, 1)
    assert (out - ref).abs().max().item() <= TOL * ref.abs().max().item()


@pytest.mark.parametrize("conv", [dict(stride=(1, 2)), dict(groups=2)])
def test_sa_module_with_a_block_the_kernel_cannot_compute_matches_unfused(cuda, conv):
    """a strided or grouped 1x1 convolution in the SharedMLP: the module computes what the op-by-op path computes (the fused
    kernel would pool every sample / read every input channel, or refuse the grouped weight)"""
    torch.manual_seed(6)
    mod = pm.PointnetSAModuleMSG(npoint=64, radii=[0.3], nsamples=[16], mlps=[[8, 16, 32]], bn=True)
    mod.mlps[0].layer1.conv = torch.nn.Conv2d(16, 32, kernel_size=1, bias=False, **conv)
    mod = mod.to(cuda).eval()
    _randomise_bn(mod, 2)
    x = torch.from_numpy(synth.u_cube(2, 512, 21)).to(cuda)
    f = torch.randn(2, 8, 512, device=cuda)
    with torch.no_grad():
        out = mod(x, f)[1]
        ref = _unfused(lambda: mod(x, f))[1]
    assert out.shape == ref.shape == (2, 32, 64)
    assert (out - ref).abs().max().item() <= TOL * ref.abs().max().item()


FP_CASES = [
    (256, 64, 1024, 512, [512, 512]),     # FP3 (split: N=512 twice)
    (1024, 256, 512, 256, [512, 512]),    # FP2
    (4096, 1024, 512, 96, [256, 256]),    # FP1
    (2048, 512, 256, 1, [128, 128]),      # FP0 with intensity
    (2048, 512, 256, 0, [128, 128]),      # FP0 without skip features
    (200, 50, 64, 3, [64]),               # n not a multiple of 128 -> tiles straddle scenes
]


@pytest.mark.parametrize("n,m,c_known,c_skip,mlp", FP_CASES)
def test_fp_module_fused_vs_unfused_vs_oracle(cuda, n, m, c_known, c_skip, mlp):
    torch.manual_seed(2)
    B = 2
    mod = pm.PointnetFPModule(mlp=[c_known + c_skip] + list(mlp)).to(cuda).eval()
    _randomise_bn(mod, 3)
    unknown = synth.u_cube(B, n, 7 + n)
    known = np.ascontiguousarray(unknown[:, ::n // m][:, :m])
    rng = np.random.default_rng(4)
    kf = rng.standard_normal((B, c_known, m)).astype(np.float32)
    sf = rng.standard_normal((B, c_skip, n)).astype(np.float32) if c_skip else None
    tu, tk, tkf = torch.from_numpy(unknown).to(cuda), torch.from_numpy(known).to(cuda), torch.from_numpy(kf).to(cuda)
    tsf = torch.from_numpy(sf).to(cuda) if c_skip else None
    with torch.no_grad():
        out = mod(tu, tk, tsf, tkf)
        ref = _unfused(lambda: mod(tu, tk, tsf, tkf))
    assert out.shape == ref.shape == (B, mlp[-1], n)
    assert (out - ref).abs().max().item() <= TOL * ref.abs().max().item()
    o = O.fp_module(unknown, known, sf, kf, _folded(mod.mlp))
    assert np.abs(out.cpu().numpy() - o).max() <= TOL * np.abs(o).max()
    assert torch.equal(out._prb_pm[0], out.transpose(1, 2).contiguous())
    mod.emit_point_major = False
    with torch.no_grad():
        out2 = mod(tu, tk, tsf, tkf)
    assert not hasattr(out2, "_prb_pm") and torch.equal(out2, out)


def test_backbone_fused_vs_unfused(cuda):
    torch.manual_seed(3)
    net = Pointnet2MSG(input_channels=1).to(cuda).eval()
    _randomise_bn(net, 5)
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 99, channels=4)).to(cuda)
    with torch.no_grad():
        xyz, feats = net(pc)
        rxyz, rfeats = _unfused(lambda: net(pc))
    assert feats.shape == (2, 128, 16384)
    assert torch.equal(xyz, rxyz)
    rel = (feats - rfeats).abs().max().item() / rfeats.abs().max().item()
    assert rel <= TOL_BACKBONE, "backbone output differs: %g" % rel


def test_backbone_b16_against_the_cpu_oracle(cuda):
    """BASELINE configs[1] at its stated shape (B=16, 16384x4 points): the fused backbone against the CPU oracle
    (O.sa_module_msg / O.fp_module, fp32 MLP, exact index ops) -- sampled centres exact, features within TOL_BACKBONE"""
    import bench
    torch.manual_seed(3)
    net = Pointnet2MSG(input_channels=1).to(cuda).eval()
    _randomise_bn(net, 5)
    pc = bench.make_scenes(700, 16)
    with torch.no_grad():
        xyz, feats = net(torch.from_numpy(pc).to(cuda))
    want = bench.cpu_backbone(pc, *bench.folded_specs(net))
    got = feats.cpu().numpy()
    assert got.shape == want.shape == (16, 128, 16384)
    rel = np.abs(got - want).max() / np.abs(want).max()
    assert rel <= TOL_BACKBONE, "backbone output differs from the oracle: %g" % rel


def test_c1_single_sa_layer_at_baseline_shape(cuda):
    """BASELINE configs[0] / SURVEY 8(d) C1 at its stated shape: one SA layer (npoint 4096, r 0.1, nsample 32, MLP [1+3,16,32])
    on one 16384x4 cloud (U-CUBE: dense balls): FPS and ball-query indices exact, grouped features exact, pooled output
    within the MLP tolerance"""
    torch.manual_seed(11)
    pc = synth.u_cube(1, 16384, 1001)
    inten = (np.random.default_rng(1001).random((1, 1, 16384), dtype=np.float32) - np.float32(0.5))
    mod = pm.PointnetSAModuleMSG(npoint=4096, radii=[0.1], nsamples=[32], mlps=[[1, 16, 32]], bn=True).to(cuda).eval()
    _randomise_bn(mod, 3)
    x, f = torch.from_numpy(pc).to(cuda), torch.from_numpy(inten).to(cuda)
    with torch.no_grad():
        new_xyz, out = mod(x, f)
        idx = pu.ball_query(0.1, 32, x, new_xyz)
        grouped = mod.groupers[0](x, new_xyz, f)
    o_xyz, o_out, _ = O.sa_module_msg(pc, inten, 4096, [0.1], [32], [_folded(mod.mlps[0])])
    assert np.array_equal(new_xyz.cpu().numpy(), o_xyz), "FPS picks differ"
    o_idx = O.ball_query(0.1, 32, pc, o_xyz)
    assert np.array_equal(idx.cpu().numpy(), o_idx), "ball-query indices differ"
    o_grouped = O.query_and_group(0.1, 32, pc, o_xyz, inten)
    np.testing.assert_allclose(grouped.cpu().numpy(), o_grouped, rtol=1e-5, atol=0)
    assert np.abs(out.cpu().numpy() - o_out).max() <= TOL * np.abs(o_out).max()


def test_training_path_autograd(cuda):
    """grad-enabled calls take the op-by-op path and back-propagate through the H100 scatter kernels"""
    torch.manual_seed(4)
    sa = pm.PointnetSAModuleMSG(npoint=64, radii=[0.3], nsamples=[16], mlps=[[8, 16, 32]], bn=True).to(cuda).train()
    fp = pm.PointnetFPModule(mlp=[32 + 8, 16]).to(cuda).train()
    xyz = torch.from_numpy(synth.u_cube(2, 512, 1)).to(cuda)
    f = torch.randn(2, 8, 512, device=cuda, requires_grad=True)
    nx, nf = sa(xyz, f)
    up = fp(xyz, nx, f, nf)
    up.sum().backward()
    assert f.grad is not None and torch.isfinite(f.grad).all() and f.grad.abs().sum() > 0
    assert all(p.grad is not None for p in sa.parameters())


def test_batch_pipeline_matches_sequential(cuda):
    """independent batches on alternating streams give bit-identical results to the one-after-another loop"""
    from pointrcnn_b200.pipeline import BatchPipeline
    torch.manual_seed(4)
    net = Pointnet2MSG(input_channels=1).to(cuda).eval()
    _randomise_bn(net, 9)
    batches = [torch.from_numpy(synth.u_kitti(2, 16384, 200 + i, channels=4)).to(cuda) for i in range(5)]
    with torch.no_grad():
        want = [net(b)[1].clone() for b in batches]
        pipe = BatchPipeline(lambda x: net(x)[1], inflight=3, device=cuda)
        got = pipe.run(batches)
        torch.cuda.synchronize()
        for w, g in zip(want, got):
            assert torch.equal(w, g)
        # host-side inputs and results (pinned), and the fire-and-forget mode
        host = [b.cpu().pin_memory() for b in batches]
        pipe2 = BatchPipeline(lambda x: net(x)[1].mean(dim=(1, 2)), inflight=2, device=cuda)
        res = pipe2.run(host, to_host=True)
        for w, r in zip(want, res):
            assert not r.is_cuda and torch.allclose(r, w.mean(dim=(1, 2)).cpu(), rtol=1e-6, atol=1e-7)
        assert pipe.run(batches, keep=False) == [None] * 5
        # results of an earlier run() stay valid after a later one (ADVICE r1: slot buffers are never handed out)
        res2 = pipe2.run(host[::-1], to_host=True)
        for w, r in zip(want, res):
            assert torch.allclose(r, w.mean(dim=(1, 2)).cpu(), rtol=1e-6, atol=1e-7)
        assert len(res2) == 5
        # streaming consumer: called once per batch, in order of completion per slot, before the slot is reused
        seen = []
        out = pipe2.run(host, to_host=True, consume=lambda i, r: seen.append((i, r.clone())) or i)
        assert out == list(range(5)) and sorted(i for i, _ in seen) == list(range(5))
        for i, r in seen:
            assert torch.allclose(r, want[i].mean(dim=(1, 2)).cpu(), rtol=1e-6, atol=1e-7)
        # CUDA-graph replay per slot: same bits as the eager launches
        pipe3 = BatchPipeline(lambda x: net(x)[1], inflight=2, device=cuda, graphs=True)
        for rep in range(2):
            got3 = pipe3.run(batches)
            torch.cuda.synchronize()
            for w, g in zip(want, got3):
                assert torch.equal(w, g)
        res3 = pipe3.run(host, to_host=True)
        for w, r in zip(want, res3):
            assert torch.equal(r, w.cpu())

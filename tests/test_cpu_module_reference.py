"""The module-level float64 reference (module_reference.py) checked on the host, and the packed-weight cache.

Chains are built by the real module code (_FusedMLP.get on "cpu", FusedRPNHeads._build), read back from their packed
images and run through mlp_reference.emulate's fp32 model of the kernel: every element must sit inside the module bound
for every accumulation order, and each planted mistake in the module-to-image path must fall outside it.  Which of those
mistakes the older norm-wise check (max |err| <= 2e-3 max |ref|) lets through is pinned too."""
import gc

import numpy as np
import pytest
import torch
import torch.nn as nn

import mlp_reference as R
import module_reference as MR
from pointrcnn_b200 import config
from pointrcnn_b200 import mlp_chain as M
from pointrcnn_b200.pointnet2 import pointnet2_modules as pm
from pointrcnn_b200.pointnet2 import pytorch_utils as pt_utils
from pointrcnn_b200.rcnn.stage import RCNNStage
from pointrcnn_b200.rpn import heads as H


class Unpacked:
    """an mlp_chain.Chain read back from its packed image, in the form mlp_reference.emulate takes"""

    def __init__(self, chain):
        self.kind, self.split, self.c_in, self.c_out = chain.kind, chain.split, chain.c_in, list(chain.c_out)
        self.linear = bool(chain.flags & 1)
        self.layers = R.unpack(chain.packed.numpy(), self.kind, self.split, self.c_in, self.c_out)
        offs = np.cumsum([0] + [R.round_up(c, 32) for c in self.c_out])
        per_layer = lambda v: [v.numpy()[o:o + c].copy() for o, c in zip(offs, self.c_out)]   # noqa: E731
        self.shift = per_layer(chain.shift)
        self.scale = None if chain.scale is None else per_layer(chain.scale)


def emulate(kind, chain, inp, order):
    u = Unpacked(chain) if not isinstance(chain, Unpacked) else chain
    return R.emulate(kind, u, u.layers, inp, order)


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


# ------------------------------------------------------------------------------------------------ the modules
B = 2
SA_SPEC = dict(npoint=12, N=96, radii=[0.2, 0.4], nsamples=[16, 32], mlps=[[1, 16, 16, 32], [1, 32, 32, 64]])
FP_SPEC = dict(n=80, m=20, c_known=64, c_skip=16, mlp=[32, 48])


def sa_case():
    mod = MR.seeded(pm.PointnetSAModuleMSG(npoint=SA_SPEC["npoint"], radii=SA_SPEC["radii"], nsamples=SA_SPEC["nsamples"],
                                        mlps=[list(m) for m in SA_SPEC["mlps"]]), 11)
    rng = np.random.default_rng(5)
    N, npoint = SA_SPEC["N"], SA_SPEC["npoint"]
    xyz = rng.uniform(-1, 1, (B, N, 3)).astype(np.float32)
    feats = rng.standard_normal((B, 1, N)).astype(np.float32)
    centres = xyz[:, :npoint].copy()
    idxs = []
    for ns in SA_SPEC["nsamples"]:
        idx = rng.integers(0, N, (B, npoint, ns)).astype(np.int32)
        idx[:, :, ns // 2:] = idx[:, :, :1]          # the ball query pads with the first neighbour
        idxs.append(idx)
    return mod, xyz, feats, centres, idxs


def run_sa(mod, xyz, feats, centres, idxs, order="sequential", msg_offset_mutant=False):
    """the module output (B, sum C, npoint) as the fused path assembles it, from emulated chains"""
    fused = [pm._FusedMLP() for _ in mod.mlps]
    chains = [f.get(mlp, M.SA, feats.shape[1], "cpu") for f, mlp in zip(fused, mod.mlps)]
    out = np.zeros((B, sum(c.c_out[-1] for c in chains), centres.shape[1]), np.float32)
    off = 0
    for k, (chain, idx) in enumerate(zip(chains, idxs)):
        inp = dict(xyz=xyz, new_xyz=centres, idx=idx, feats_pm=np.ascontiguousarray(feats.transpose(0, 2, 1)))
        at = 0 if (msg_offset_mutant and k == 1) else off
        out[:, at:at + chain.c_out[-1]] = emulate("sa", chain, inp, order)
        off += chain.c_out[-1]
    return out


def ref_sa(mod, xyz, feats, centres, idxs):
    parts = [MR.sa_scale(mlp, t(xyz), t(feats), t(centres), t(idx)) for mlp, idx in zip(mod.mlps, idxs)]
    return torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1)


def fp_case():
    s = FP_SPEC
    mod = MR.seeded(pm.PointnetFPModule(mlp=[s["c_known"] + s["c_skip"]] + s["mlp"]), 12)
    rng = np.random.default_rng(6)
    w = rng.uniform(0.05, 1.0, (B, s["n"], 3)).astype(np.float32)
    return (mod, rng.integers(0, s["m"], (B, s["n"], 3)).astype(np.int32), (w / w.sum(-1, keepdims=True)).astype(np.float32),
            rng.standard_normal((B, s["c_skip"], s["n"])).astype(np.float32),
            rng.standard_normal((B, s["c_known"], s["m"])).astype(np.float32))


def run_fp(mod, idx, weight, skip, known, projected, order="sequential", proj_shift_mutant=False):
    f = pm._FusedMLP()
    c_known = known.shape[1]
    chain = f.get(mod.mlp, M.FP, c_known, "cpu", project_known=projected)
    known_pm = np.ascontiguousarray(known.transpose(0, 2, 1))
    main = Unpacked(chain)
    if projected:
        proj = Unpacked(f.proj)
        if proj_shift_mutant:
            proj.shift[0] = main.shift[0]
        c1 = proj.c_out[0]
        rows = R.emulate("rows", proj, proj.layers, dict(a=known_pm.reshape(-1, c_known), a_off=0, c_a=c_known), order)
        known_pm = np.ascontiguousarray(rows[:, :c1].reshape(B, -1, c1))
    return R.emulate("fp", main, main.layers, dict(known_pm=known_pm, idx=idx, weight=weight, skip=skip), order)


def heads_case():
    cls = nn.Sequential(pt_utils.Conv1d(128, 128, bn=True), nn.Dropout(0.5), pt_utils.Conv1d(128, 1, activation=None))
    reg = nn.Sequential(pt_utils.Conv1d(128, 128, bn=True), nn.Dropout(0.5), pt_utils.Conv1d(128, 76, activation=None))
    MR.seeded(cls, 13), MR.seeded(reg, 14)
    return cls, reg, np.random.default_rng(7).standard_normal((48, 128)).astype(np.float32)


def heads_build_block_offset_mutant(cls_seq, reg_seq, device):
    """FusedRPNHeads._build with the reg block of the second layer one hidden channel to the left"""
    (c0, cb0, _), (c1, _, _) = H._layers(cls_seq)
    (r0, rb0, _), (r1, _, _) = H._layers(reg_seq)
    Wc0, _, sc0 = M.fold(c0, cb0, zero_bias=True)
    Wr0, _, sr0 = M.fold(r0, rb0, zero_bias=True)
    Wc1, _, sc1 = M.fold(c1, None)
    Wr1, _, sr1 = M.fold(r1, None)
    hc, hr = Wc0.shape[0], Wr0.shape[0]
    W1 = torch.zeros(Wc1.shape[0] + Wr1.shape[0], hc + hr)
    W1[:Wc1.shape[0], :hc] = Wc1
    W1[Wc1.shape[0]:, hc - 1:hc + hr - 1] = Wr1
    chain = M.Chain(M.ROWS, 0, [torch.cat([Wc0, Wr0], 0), W1], [torch.cat([sc0, sr0]), torch.cat([sc1, sr1])],
                    linear_last=True, device=device)
    return chain, Wc1.shape[0]


def run_heads(cls, reg, rows, order="sequential", build=H.FusedRPNHeads._build):
    chain, n_cls = build(cls, reg, "cpu")
    out = emulate("rows", chain, dict(a=rows, a_off=0, c_a=rows.shape[1]), order)
    return out[:, :n_cls], out[:, n_cls:chain.c_out[-1]]


def rcnn_case(bn):
    r = MR.seeded(RCNNStage(cfg=dict(USE_BN=bn)), 15 + bn)
    rows = np.random.default_rng(8).standard_normal((40, r.rcnn_input_channel + 128)).astype(np.float32)
    return r, rows


def run_rcnn(r, rows, order="sequential"):
    ci = r.rcnn_input_channel
    up_chain = pm._FusedMLP().get(r.xyz_up_layer, *M.rows_layout(ci, 0), "cpu")
    up = emulate("rows", up_chain, dict(a=rows, a_off=0, c_a=ci), order)[:, :up_chain.c_out[-1]]
    c_up = up.shape[1]
    merge_chain = pm._FusedMLP().get(r.merge_down_layer, *M.rows_layout(c_up, rows.shape[1] - ci), "cpu")
    merged = emulate("rows", merge_chain, dict(a=up, a_off=0, c_a=c_up, b=rows, b_off=ci, c_b=rows.shape[1] - ci), order)
    return up, merged[:, :merge_chain.c_out[-1]]


# ------------------------------------------------------------------------------------------------ the bound holds
def _within(got, ref, bound, label):
    ok, ratio, bad = MR.check(t(got), ref, bound)
    assert ok, "%s: %d elements outside the bound, max err/bound %.3g" % (label, bad, ratio)
    return ratio


@pytest.mark.parametrize("fold", [True, False])
def test_sa_msg_module_within_bound(fold):
    mod, xyz, feats, centres, idxs = sa_case()
    with config.override(fold_scale=fold):
        ref, bound = ref_sa(mod, xyz, feats, centres, idxs)
        worst = max(_within(run_sa(mod, xyz, feats, centres, idxs, order), ref, bound, order) for order in R.ORDERS)
    assert worst > 0
    print("SA MSG fold_scale=%d: max err/bound %.3g" % (fold, worst))


@pytest.mark.parametrize("fold,projected", [(True, False), (False, False), (True, True)])
def test_fp_module_within_bound(fold, projected):
    mod, idx, weight, skip, known = fp_case()
    ref, bound = MR.fp_module(mod.mlp, t(idx), t(weight), t(skip), t(known), projected)
    with config.override(fold_scale=fold):
        worst = max(_within(run_fp(mod, idx, weight, skip, known, projected, order), ref, bound, order) for order in R.ORDERS)
    assert worst > 0
    print("FP fold_scale=%d projected=%d: max err/bound %.3g" % (fold, projected, worst))


def test_heads_within_bound():
    cls, reg, rows = heads_case()
    (rc, bc), (rr, br) = MR.heads(cls, reg, t(rows))
    for order in R.ORDERS:
        gc_, gr = run_heads(cls, reg, rows, order)
        _within(gc_, rc, bc, "cls " + order)
        _within(gr, rr, br, "reg " + order)


@pytest.mark.parametrize("bn", [False, True])
def test_rcnn_rows_mlp_within_bound(bn):
    r, rows = rcnn_case(bn)
    ci = r.rcnn_input_channel
    for order in R.ORDERS:
        up, merged = run_rcnn(r, rows, order)
        _within(up, *MR.rows_mlp(r.xyz_up_layer, t(rows[:, :ci])), "xyz_up " + order)
        # the merge's own reference, on the up rows the chain produced (as the device test captures them)
        _within(merged, *MR.rows_mlp(r.merge_down_layer, t(up), t(rows[:, ci:])), "merge " + order)


# ------------------------------------------------------------------------------------------------ mutants
_FOLD = M.fold


class _Shadow:
    """a BatchNorm's parameters with some replaced"""

    def __init__(self, bn, **over):
        for k in ("weight", "bias", "running_mean", "running_var", "eps"):
            setattr(self, k, over.get(k, getattr(bn, k)))


def _fold_without_eps(conv, bn, fold_scale=True, zero_bias=False):
    if bn is not None:
        bn = _Shadow(bn, eps=0.0)
    return _FOLD(conv, bn, fold_scale, zero_bias)


def _fold_without_mean(conv, bn, fold_scale=True, zero_bias=False):
    if bn is not None:
        bn = _Shadow(bn, running_mean=torch.zeros_like(bn.running_mean))
    return _FOLD(conv, bn, fold_scale, zero_bias)


def _fold_small_channels_without_mean(conv, bn, fold_scale=True, zero_bias=False):
    """the mean term dropped from the shift of the small channels only (|gamma / std| < 0.05)"""
    if bn is not None:
        inv = bn.weight.detach() / torch.sqrt(bn.running_var + bn.eps)
        bn = _Shadow(bn, running_mean=torch.where(inv.abs() < 0.05, torch.zeros_like(bn.running_mean), bn.running_mean))
    return _FOLD(conv, bn, fold_scale, zero_bias)


def _fold_zero_bias(conv, bn, fold_scale=True, zero_bias=False):
    return _FOLD(conv, bn, fold_scale, True)


def _sa_mutant(monkeypatch, fold_fn=None, msg_offset=False):
    mod, xyz, feats, centres, idxs = sa_case()
    ref, bound = ref_sa(mod, xyz, feats, centres, idxs)
    if fold_fn is not None:
        monkeypatch.setattr(M, "fold", fold_fn)
    got = run_sa(mod, xyz, feats, centres, idxs, msg_offset_mutant=msg_offset)
    return got, ref, bound


def _proj_shift_mutant(monkeypatch):
    mod, idx, weight, skip, known = fp_case()
    ref, bound = MR.fp_module(mod.mlp, t(idx), t(weight), t(skip), t(known), True)
    return run_fp(mod, idx, weight, skip, known, True, proj_shift_mutant=True), ref, bound


def _heads_mutant(monkeypatch):
    cls, reg, rows = heads_case()
    _, (rr, br) = MR.heads(cls, reg, t(rows))
    _, gr = run_heads(cls, reg, rows, build=heads_build_block_offset_mutant)
    return gr, rr, br


def _rcnn_zero_bias(monkeypatch):
    r, rows = rcnn_case(True)
    ci = r.rcnn_input_channel
    monkeypatch.setattr(M, "fold", _fold_zero_bias)
    up, _ = run_rcnn(r, rows)
    return up, *MR.rows_mlp(r.xyz_up_layer, t(rows[:, :ci]))


# name: (run, whether the norm-wise 2e-3 check passes it, whether the bound can see it)
MUTANTS = {
    "fold_ignores_eps": (lambda mp: _sa_mutant(mp, _fold_without_eps), False, True),
    "shift_without_mean": (lambda mp: _sa_mutant(mp, _fold_without_mean), False, True),
    "small_channel_shift_without_mean": (lambda mp: _sa_mutant(mp, _fold_small_channels_without_mean), True, True),
    "projection_carries_shift": (_proj_shift_mutant, False, True),
    "heads_w1_block_offset": (_heads_mutant, False, True),
    "msg_scale1_at_scale0_offset": (lambda mp: _sa_mutant(mp, msg_offset=True), False, True),
    "zero_bias_on_shared_mlp": (_rcnn_zero_bias, True, False),
}


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_bound_catches_a_wrong_module_to_image_step(name, monkeypatch):
    """each planted mistake between the module and the packed image falls outside the bound (the norm-wise check that
    preceded it is recorded beside it).  zero_bias on a SharedMLP is the exception: it adds inv * 0 to the shift, which
    changes the sign of a -0.0 shift and nothing else, so no output value moves; the pinned image digests of
    test_cpu_mlp_chain.py are what see it."""
    run, tol_passes, visible = MUTANTS[name]
    got, ref, bound = run(monkeypatch)
    ok, ratio, bad = MR.check(t(got), ref, bound)
    old = MR.old_tol_passes(t(got), ref)
    print("mutant %-33s outside the bound: %5d elements, max err/bound %.3g; norm-wise 2e-3 check %s"
          % (name, bad, ratio, "passes it" if old else "fails it"))
    assert ok != visible, "mutant %s: bound check %s" % (name, "passed" if ok else "failed")
    assert old == tol_passes, "mutant %s: the norm-wise check %s" % (name, "passes" if old else "fails")


# ------------------------------------------------------------------------------------------------ the cache
def _same(a, b):
    return (torch.equal(a.packed, b.packed) and torch.equal(a.shift, b.shift)
            and (a.scale is None) == (b.scale is None) and (a.scale is None or torch.equal(a.scale, b.scale)))


def _sa_mlp():
    return MR.seeded(pt_utils.SharedMLP([7, 32, 64], bn=True), 21)


def _get(f, mlp):
    return f.get(mlp, M.SA, 4, "cpu")


def _fresh(mlp):
    return pm._FusedMLP().get(mlp, M.SA, 4, "cpu")


def test_a_replaced_parameter_takes_the_id_of_the_one_it_replaces():
    """the construction the cache tests use: with nothing but an id() remembering the old parameter (what a cache keyed
    on (id, version) keeps), the new nn.Parameter has the old one's id() and version 0 every time"""
    conv = _sa_mlp()[0].conv
    conv.weight = nn.Parameter(torch.randn(32, 7, 1, 1))
    for k in range(50):
        old = (id(conv.weight), conv.weight._version)
        assert MR.replace_parameter(conv, "weight", torch.randn(32, 7, 1, 1)), "replacement %d got a new id()" % k
        assert (id(conv.weight), conv.weight._version) == old


def test_cache_sees_a_parameter_replaced_by_one_that_reuses_its_id():
    """a cache that remembers a parameter by (id, version) returns the chain of the replaced weight here: the new
    Parameter has the old one's id() and version 0 (see the test above)"""
    mlp = _sa_mlp()
    conv = mlp[0].conv
    conv.weight = nn.Parameter(torch.randn(32, 7, 1, 1))
    f = pm._FusedMLP()
    stale = 0
    for _ in range(50):
        _get(f, mlp)
        MR.replace_parameter(conv, "weight", torch.randn(32, 7, 1, 1))
        stale += not _same(_get(f, mlp), _fresh(mlp))
    assert stale == 0, "%d of 50 calls returned the chain of a replaced weight" % stale


@pytest.mark.parametrize("assign", [False, True])
def test_cache_sees_load_state_dict(assign):
    mlp = _sa_mlp()
    f = pm._FusedMLP()
    _get(f, mlp)
    for seed in (31, 32):
        mlp.load_state_dict(MR.seeded(pt_utils.SharedMLP([7, 32, 64], bn=True), seed).state_dict(), assign=assign)
        gc.collect()
        assert _same(_get(f, mlp), _fresh(mlp)), "load_state_dict(assign=%s) #%d" % (assign, seed - 30)


def test_cache_sees_an_in_place_edit():
    mlp = _sa_mlp()
    f = pm._FusedMLP()
    before = _get(f, mlp)
    with torch.no_grad():
        mlp[1].bn.bn.running_var.mul_(2.0)
        mlp[0].conv.weight[3].neg_()
    after = _get(f, mlp)
    assert after is not before and _same(after, _fresh(mlp))


def test_cache_sees_fold_scale_toggled():
    mlp = _sa_mlp()
    f = pm._FusedMLP()
    for fold in (True, False, True):
        with config.override(fold_scale=fold):
            got = _get(f, mlp)
            assert (got.scale is None) == fold and _same(got, _fresh(mlp))


def test_cache_reuses_an_unchanged_chain():
    mlp = _sa_mlp()
    f = pm._FusedMLP()
    assert _get(f, mlp) is _get(f, mlp)

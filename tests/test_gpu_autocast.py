"""Training under torch.autocast(bfloat16) on the device: the bfloat16 grouping / gather / interpolation natives bit for bit
against the numpy restatement of test_cpu_autocast_ops.py (forward; ordered backward) and within the stated fp32-sum
bound (atomic backward), float32 calls still on the float32 entries, and the RPN / RCNN trainers at B = 2 under
autocast: a finite loss, the first step within a bound of the fp32 step (derived from the same step with the three index
ops written as torch indexing under autocast), no host synchronisation on the device paths, and two seeded runs under
torch.use_deterministic_algorithms(True) that end with the same bits."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_cpu_autocast_ops import (_group_vals, _interp_vals, atomic_interval, bf16_bits, gather_bf16_ref, group_bf16_ref,
                                   group_grad_bf16_ref, interp_bf16_ref, interp_grad_bf16_ref, within_bf16_interval)
from pointrcnn_b200 import _cabi as C
from pointrcnn_b200.pointnet2 import pointnet2_utils as pu

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


def _dev(bits, cuda):
    """uint16 bit patterns -> a bfloat16 CUDA tensor"""
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).to(cuda).view(torch.bfloat16)


def _host(t):
    return t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def _bits_equal(got, want):
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = got != want
    assert not bad.any(), "%d of %d values differ, first at %s: %#06x vs %#06x" % (bad.sum(), bad.size, np.argwhere(bad)[0].tolist(),
                                                                               got[bad][0], want[bad][0])


def _rand_bits(gen, shape):
    return bf16_bits(torch.randn(shape, generator=gen).numpy())


def _padded_idx(gen, b, npoint, ns, n):
    idx = torch.randint(0, n, (b, npoint, ns), generator=gen)
    hits = torch.randint(1, ns + 1, (b, npoint, 1), generator=gen)
    return torch.where(torch.arange(ns) >= hits, idx[:, :, :1], idx).int()


def _taps(gen, B, n, m):
    idx = torch.randint(0, m, (B, n, 3), generator=gen)
    w = torch.rand(B, n, 3, generator=gen) + 0.01
    return idx.int().contiguous(), (w / w.sum(2, keepdim=True)).contiguous()


# ------------------------------------------------------------------------------------------ the ops
GROUP_SHAPES = {
    # name: (B, C, N, npoint, nsample): RPN B = 16 levels fed by a bfloat16 level, RCNN B = 4 (64 RoIs per scene)
    "rpn_sa2_ns16": (16, 96, 4096, 1024, 16),
    "rpn_sa2_ns32": (16, 96, 4096, 1024, 32),
    "rpn_sa3_ns32": (16, 256, 1024, 256, 32),
    "rpn_sa4_ns16": (16, 512, 256, 64, 16),
    "rcnn_sa1_b4": (256, 128, 512, 128, 64),
    "rcnn_sa2_b4": (256, 128, 128, 32, 64),
    "odd_channels_13": (2, 13, 333, 100, 16),
    "odd_length_185": (3, 11, 90, 37, 5),       # npoints * nsample not a multiple of 8: the element-wise kernel
}
INTERP_SHAPES = {
    # (B, C, n unknown, m known): the RPN FP levels at B = 16, and odd sizes
    "rpn_fp3": (16, 1024, 256, 64),
    "rpn_fp2": (16, 512, 1024, 256),
    "rpn_fp1": (16, 512, 4096, 1024),
    "rpn_fp0": (16, 256, 16384, 4096),
    "odd_13_257": (2, 13, 257, 333),
}


def _chunks(c, step):
    return [(c0, min(c0 + step, c)) for c0 in range(0, c, step)]


@pytest.mark.parametrize("name", list(GROUP_SHAPES))
def test_group_forward_is_exact(cuda, name):
    B, Cc, N, P, S = GROUP_SHAPES[name]
    gen = torch.Generator().manual_seed(len(name))
    pts = _rand_bits(gen, (B, Cc, N))
    idx = _padded_idx(gen, B, P, S, N)
    out = pu.grouping_operation(_dev(pts, cuda), idx.to(cuda))
    assert out.dtype == torch.bfloat16 and out.shape == (B, Cc, P, S)
    _bits_equal(_host(out), group_bf16_ref(pts, idx.numpy()))


@pytest.mark.parametrize("B,Cc,N,P", [(16, 96, 4096, 1024), (256, 128, 512, 128), (3, 13, 50, 37)])
def test_gather_forward_is_exact(cuda, B, Cc, N, P):
    gen = torch.Generator().manual_seed(N)
    pts = _rand_bits(gen, (B, Cc, N))
    idx = torch.randint(0, N, (B, P), generator=gen).int()
    out = pu.gather_operation(_dev(pts, cuda), idx.to(cuda))
    _bits_equal(_host(out), gather_bf16_ref(pts, idx.numpy()))


@pytest.mark.parametrize("name", list(INTERP_SHAPES))
def test_three_interpolate_forward_is_exact(cuda, name):
    B, Cc, n, m = INTERP_SHAPES[name]
    gen = torch.Generator().manual_seed(len(name))
    pts = _rand_bits(gen, (B, Cc, m))
    idx, w = _taps(gen, B, n, m)
    got = _host(pu.three_interpolate(_dev(pts, cuda), idx.to(cuda), w.to(cuda)))
    for c0, c1 in _chunks(Cc, 32):
        _bits_equal(got[:, c0:c1], interp_bf16_ref(pts[:, c0:c1], idx.numpy(), w.numpy()))


ORDERED_GROUP = ["rpn_sa2_ns32", "rpn_sa4_ns16", "rcnn_sa1_b4", "odd_channels_13", "odd_length_185"]


def _group_backward(cuda, pts, idx, g):
    feats = _dev(pts, cuda).requires_grad_(True)
    pu.grouping_operation(feats, idx.to(cuda)).backward(_dev(g, cuda))
    assert feats.grad.dtype == torch.bfloat16
    return _host(feats.grad)


@pytest.mark.parametrize("name", ORDERED_GROUP)
def test_group_backward_ordered_is_exact(cuda, deterministic, name):
    B, Cc, N, P, S = GROUP_SHAPES[name]
    gen = torch.Generator().manual_seed(len(name) + 1)
    pts, idx, g = _rand_bits(gen, (B, Cc, N)), _padded_idx(gen, B, P, S, N), _rand_bits(gen, (B, Cc, P, S))
    got = _group_backward(cuda, pts, idx, g)
    _bits_equal(got, _group_backward(cuda, pts, idx, g))
    for c0, c1 in _chunks(Cc, 32):
        _bits_equal(got[:, c0:c1], group_grad_bf16_ref(g[:, c0:c1], idx.numpy(), N))


@pytest.mark.parametrize("name", ORDERED_GROUP)
def test_group_backward_atomic_within_the_fp32_sum_bound(cuda, name):
    B, Cc, N, P, S = GROUP_SHAPES[name]
    gen = torch.Generator().manual_seed(len(name) + 1)
    pts, idx, g = _rand_bits(gen, (B, Cc, N)), _padded_idx(gen, B, P, S, N), _rand_bits(gen, (B, Cc, P, S))
    got = _group_backward(cuda, pts, idx, g)
    for c0, c1 in _chunks(Cc, 32):
        lo, hi = atomic_interval(*_group_vals(g[:, c0:c1], idx.numpy()), N)
        assert within_bf16_interval(got[:, c0:c1], lo, hi).all()


def test_lone_points_ordered_and_atomic(cuda, deterministic):
    """one point names every centre of scene 1 (19200 references): the longest sums"""
    B, Cc, N, P, S = 2, 11, 40, 300, 64
    gen = torch.Generator().manual_seed(2)
    idx = _padded_idx(gen, B, P, S, N)
    idx[1] = 7
    pts, g = _rand_bits(gen, (B, Cc, N)), _rand_bits(gen, (B, Cc, P, S))
    _bits_equal(_group_backward(cuda, pts, idx, g), group_grad_bf16_ref(g, idx.numpy(), N))
    torch.use_deterministic_algorithms(False)
    lo, hi = atomic_interval(*_group_vals(g, idx.numpy()), N)
    assert within_bf16_interval(_group_backward(cuda, pts, idx, g), lo, hi).all()


@pytest.mark.parametrize("ordered", [True, False])
def test_gather_backward(cuda, ordered):
    B, Cc, N, P = 3, 13, 50, 200                # points named several times
    gen = torch.Generator().manual_seed(5)
    pts, idx, g = _rand_bits(gen, (B, Cc, N)), torch.randint(0, N, (B, P), generator=gen).int(), _rand_bits(gen, (B, Cc, P))
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(ordered)
    try:
        feats = _dev(pts, cuda).requires_grad_(True)
        pu.gather_operation(feats, idx.to(cuda)).backward(_dev(g, cuda))
    finally:
        torch.use_deterministic_algorithms(was)
    got = _host(feats.grad)
    if ordered:
        _bits_equal(got, group_grad_bf16_ref(g, idx.numpy(), N))
    else:
        assert within_bf16_interval(got, *atomic_interval(*_group_vals(g, idx.numpy()), N)).all()


def _interp_backward(cuda, pts, idx, w, g):
    feats = _dev(pts, cuda).requires_grad_(True)
    pu.three_interpolate(feats, idx.to(cuda), w.to(cuda)).backward(_dev(g, cuda))
    return _host(feats.grad)


@pytest.mark.parametrize("name", ["rpn_fp1", "rpn_fp3", "odd_13_257"])
def test_three_interpolate_backward(cuda, name):
    B, Cc, n, m = INTERP_SHAPES[name]
    gen = torch.Generator().manual_seed(len(name) + 2)
    pts, (idx, w), g = _rand_bits(gen, (B, Cc, m)), _taps(gen, B, n, m), _rand_bits(gen, (B, Cc, n))
    atomic = _interp_backward(cuda, pts, idx, w, g)
    torch.use_deterministic_algorithms(True)
    try:
        ordered = _interp_backward(cuda, pts, idx, w, g)
        _bits_equal(_interp_backward(cuda, pts, idx, w, g), ordered)
    finally:
        torch.use_deterministic_algorithms(False)
    for c0, c1 in _chunks(Cc, 32):
        _bits_equal(ordered[:, c0:c1], interp_grad_bf16_ref(g[:, c0:c1], idx.numpy(), w.numpy(), m))
        lo, hi = atomic_interval(*_interp_vals(g[:, c0:c1], idx.numpy(), w.numpy()), m)
        assert within_bf16_interval(atomic[:, c0:c1], lo, hi).all()


class _Recorder:
    """the real library, recording the names of the entries called through it"""

    def __init__(self, lib):
        self.lib, self.names = lib, []

    def __getattr__(self, name):
        if name.startswith("prb_") and not name.endswith("_workspace_bytes"):
            self.names.append(name)
        return getattr(self.lib, name)


def test_float32_calls_reach_the_float32_entries(cuda, monkeypatch):
    """float32 features: the float32 entries and the float32 results, bit for bit what the entries give when called directly"""
    rec = _Recorder(C.lib())
    gen = torch.Generator().manual_seed(6)
    B, Cc, N, P, S = 2, 16, 500, 64, 16
    feats = torch.randn(B, Cc, N, generator=gen).to(cuda).requires_grad_(True)
    idx = _padded_idx(gen, B, P, S, N).to(cuda)
    gidx = torch.randint(0, N, (B, P), generator=gen).int().to(cuda)
    ti, tw = (t.to(cuda) for t in _taps(gen, B, 100, N))
    monkeypatch.setattr(C, "lib", lambda: rec)
    y = [pu.grouping_operation(feats, idx), pu.gather_operation(feats, gidx), pu.three_interpolate(feats, ti, tw)]
    sum(t.sum() for t in y).backward()
    monkeypatch.undo()
    assert rec.names[:3] == ["prb_group_points", "prb_gather_points", "prb_three_interpolate"]
    assert sorted(rec.names[3:]) == ["prb_gather_points_grad", "prb_group_points_grad", "prb_three_interpolate_grad"]
    assert all(t.dtype == torch.float32 for t in y) and feats.grad.dtype == torch.float32
    direct = torch.empty_like(y[0])
    C.check(C.lib().prb_group_points(B, Cc, N, P, S, C.ptr(feats), C.ptr(idx), C.ptr(direct), C.stream()), "group_points")
    assert torch.equal(direct.view(torch.int32), y[0].detach().view(torch.int32))


# ------------------------------------------------------------------------------------------ the trainers
def _torch_gather(features, idx):
    return torch.gather(features, 2, idx.long().unsqueeze(1).expand(-1, features.size(1), -1))


def _torch_group(features, idx):
    B, Cc, _ = features.shape
    _, M, S = idx.shape
    return torch.gather(features, 2, idx.long().view(B, 1, M * S).expand(-1, Cc, -1)).view(B, Cc, M, S)


def _torch_interp(features, idx, weight):
    B, Cc, _ = features.shape
    N = idx.shape[1]
    g = torch.gather(features, 2, idx.long().view(B, 1, N * 3).expand(-1, Cc, -1)).view(B, Cc, N, 3)
    return (g * weight.unsqueeze(1)).sum(dim=3)


def _torch_index_ops(monkeypatch):
    monkeypatch.setattr(pu, "gather_operation", _torch_gather)
    monkeypatch.setattr(pu, "grouping_operation", _torch_group)
    monkeypatch.setattr(pu, "three_interpolate", _torch_interp)


RPN_CONFIGS = {"torch": dict(), "device": dict(loss_impl="device", sa_train="device", fp_train="device")}
RCNN_CONFIGS = {"torch": dict(target_draw="torch", loss_impl="torch"), "device": dict(target_draw="device", loss_impl="device")}


def _rpn_batch(cuda):
    import synth
    from pointrcnn_b200.train.step import synthetic_labels
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 123, channels=4)).to(cuda)
    return (pc,) + tuple(synthetic_labels(pc, seed=1))


def _jit_batch(cuda):
    from oracle import rcnn_offline as RO
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    scenes = [RO.synth_scene(s, k, n_feat=128) for s, k in ((51, "mixed"), (52, "hard"))]
    return RCNNOfflineSampler(device=cuda).prepare_jit_batch(scenes)


def _rpn_first_step(cuda, config, batch, autocast):
    """(loss, [grads]) of a fresh trainer's first step; the heads' Dropout off, so every variant drops the same nothing"""
    from pointrcnn_b200.train.step import RPNTrainer
    tr = RPNTrainer(device=cuda, seed=3, **RPN_CONFIGS[config])
    for m in tr.model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    torch.manual_seed(0)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        loss, _ = tr.step(*batch)
    return loss.double(), [p.grad.detach().double().clone() for p in tr.params]


def _rcnn_first_step(cuda, config, batch, autocast):
    from pointrcnn_b200.train.step import RCNNTrainer
    tr = RCNNTrainer(device=cuda, seed=5, **RCNN_CONFIGS[config])
    torch.manual_seed(0)
    np.random.seed(0)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        loss, _ = tr.step_jit(batch)
    return loss.double(), [p.grad.detach().double().clone() for p in tr.params]


def _distance(a, b):
    """(relative loss difference, norm-wise relative gradient difference) of two (loss, grads)"""
    ga, gb = torch.cat([g.reshape(-1) for g in a[1]]), torch.cat([g.reshape(-1) for g in b[1]])
    return float((a[0] - b[0]).abs() / b[0].abs()), float((ga - gb).norm() / gb.norm())


def _compare(first_step, cuda, config, batch, monkeypatch, record_property):
    ref32 = first_step(cuda, config, batch, False)
    ours = first_step(cuda, config, batch, True)
    assert torch.isfinite(ours[0]) and all(torch.isfinite(g).all() for g in ours[1])
    with monkeypatch.context() as mp:
        _torch_index_ops(mp)
        native = first_step(cuda, config, batch, True)
    d_ours, d_native = _distance(ours, ref32), _distance(native, ref32)
    record_property("bf16_natives_vs_fp32", d_ours)
    record_property("torch_indexing_vs_fp32", d_native)
    print("%s: bf16 natives vs fp32 (loss, grads) = (%.3g, %.3g); torch indexing under autocast vs fp32 = (%.3g, %.3g)"
          % (config, d_ours[0], d_ours[1], d_native[0], d_native[1]))
    # the bound: twice what bfloat16 autocast with torch's own indexing costs, and never below a few bfloat16 ulps
    for ours_d, native_d, floor in zip(d_ours, d_native, (2.0 ** -7, 2.0 ** -6)):
        assert ours_d <= max(2.0 * native_d, floor), (d_ours, d_native)


@pytest.mark.parametrize("config", list(RPN_CONFIGS))
def test_rpn_step_under_autocast_within_the_bound_of_fp32(cuda, config, monkeypatch, record_property):
    _compare(_rpn_first_step, cuda, config, _rpn_batch(cuda), monkeypatch, record_property)


@pytest.mark.parametrize("config", list(RCNN_CONFIGS))
def test_rcnn_step_jit_under_autocast_within_the_bound_of_fp32(cuda, config, monkeypatch, record_property):
    _compare(_rcnn_first_step, cuda, config, _jit_batch(cuda), monkeypatch, record_property)


def test_rcnn_step_offline_runs_under_autocast(cuda):
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    from pointrcnn_b200.train.step import RCNNTrainer
    from oracle import rcnn_offline as RO
    scenes = [RO.synth_scene(s, k, n_feat=128) for s, k in ((51, "mixed"), (52, "hard"))]
    batch = RCNNOfflineSampler(device=cuda).prepare_batch(scenes)
    for impl in ("torch", "device"):
        tr = RCNNTrainer(device=cuda, seed=5, loss_impl=impl)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss, _ = tr.step_offline(batch)
        assert torch.isfinite(loss) and all(p.dtype == torch.float32 for p in tr.params)
        assert all(torch.isfinite(p.grad).all() and p.grad.dtype == torch.float32 for p in tr.params)


def test_device_paths_add_no_host_synchronisation(cuda):
    from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer
    rpn, batch = RPNTrainer(device=cuda, seed=3, **RPN_CONFIGS["device"]), _rpn_batch(cuda)
    rcnn, jit = RCNNTrainer(device=cuda, seed=5, **RCNN_CONFIGS["device"]), _jit_batch(cuda)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        rpn.step(*batch)                         # first-call set-up outside the checked steps
        rcnn.step_jit(jit)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            loss_rpn, _ = rpn.step(*batch, grad_norm_clip=1.0)
            loss_rcnn, _ = rcnn.step_jit(jit, grad_norm_clip=1.0)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(loss_rpn) and torch.isfinite(loss_rcnn)


# ------------------------------------------------------------------------------------------ two seeded runs
def _state_digest(tr):
    h = hashlib.sha256()
    for p in tr.params:
        h.update(p.detach().cpu().numpy().tobytes())
    for b in tr.model.buffers():
        h.update(b.detach().cpu().numpy().tobytes())
    for p in tr.params:
        for k, v in sorted(tr.opt.state.get(p, {}).items()):
            if torch.is_tensor(v):
                h.update(v.detach().cpu().numpy().tobytes())
    return h.hexdigest()


def _worker():
    """two runs of three autocast steps per trainer configuration from the same seed and batches, flag on -> JSON digests"""
    from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer
    torch.use_deterministic_algorithms(True)
    dev = torch.device("cuda:0")
    batch, jit = _rpn_batch(dev), _jit_batch(dev)
    res = {}
    for _ in range(2):
        for config in RPN_CONFIGS:
            tr = RPNTrainer(device=dev, seed=3, **RPN_CONFIGS[config])
            torch.manual_seed(0)
            for _ in range(3):
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    tr.step(*batch, grad_norm_clip=1.0)
            res.setdefault("rpn_" + config, []).append(_state_digest(tr))
        tr = RCNNTrainer(device=dev, seed=5, **RCNN_CONFIGS["device"])
        for _ in range(3):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                tr.step_jit(jit, grad_norm_clip=1.0)
        res.setdefault("rcnn_device", []).append(_state_digest(tr))
    print("DIGESTS " + json.dumps(res))


def test_two_seeded_autocast_runs_end_with_the_same_bits(cuda):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker"], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("DIGESTS ")][-1]
    res = json.loads(line[len("DIGESTS "):])
    assert len(res) == 3
    for key, (a, b) in res.items():
        assert a == b, "%s: two seeded autocast runs differ" % key


if __name__ == "__main__" and "--worker" in sys.argv:
    _worker()

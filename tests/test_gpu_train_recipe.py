"""The reference's default training recipe (train/recipe.py) on the device training path: the true-weight-decay Adam step
against a single-tensor replay, no host synchronisation in a scheduled step, two deterministic runs with the same bits,
the scheduled BN momentum inside the device SA / FP training kernels, the phase-1 checkpoint handed to the RCNN phase and
to PointRCNNInference, and the epoch loop's one host copy per epoch."""
import hashlib
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

import synth
from pointrcnn_b200.train import recipe
from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer, synthetic_labels

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEVICE_PATHS = dict(loss_impl="device", sa_train="device", fp_train="device")


def _batch(dev, seed=123):
    pc = torch.from_numpy(synth.u_kitti(2, 16384, seed, channels=4)).to(dev)
    cls, reg = synthetic_labels(pc, seed=1)
    return pc, cls, reg


def test_onecycle_step_matches_a_single_tensor_replay(cuda):
    """three scheduled steps of the fused inner Adam against torch's single-tensor Adam plus the decay, on the gradients the
    trainer's steps left behind (after clipping)"""
    tr = RPNTrainer(device=cuda, optimizer="adam_onecycle", total_steps=10, **DEVICE_PATHS)
    groups = [[p.detach().clone().requires_grad_(True) for p in pg["params"]] for pg in tr.opt.param_groups]
    replay = torch.optim.Adam([{"params": g} for g in groups], foreach=False, fused=False)
    batch = _batch(cuda)
    for it in range(3):
        tr.schedule_iteration(it, 0, 10)
        tr.step(*batch, grad_norm_clip=recipe.GRAD_NORM_CLIP)
        lr, betas = tr.opt.param_groups[0]["lr"], tr.opt.param_groups[0]["betas"]
        with torch.no_grad():
            for pg, mine in zip(tr.opt.param_groups, groups):
                for p, q in zip(pg["params"], mine):
                    q.grad = None if p.grad is None else p.grad.detach().clone()
                    q.mul_(1 - recipe.WEIGHT_DECAY * lr)
        for g in replay.param_groups:
            g["lr"], g["betas"] = lr, betas
        replay.step()
    worst = 0.0
    for pg, mine in zip(tr.opt.param_groups, groups):
        for p, q in zip(pg["params"], mine):
            err = float((p.detach() - q.detach()).abs().max() / q.detach().abs().max().clamp(min=1e-30))
            worst = max(worst, err)
    print("worst relative difference to the single-tensor replay: %.3g" % worst)
    assert worst <= 1e-6


def test_scheduled_step_does_not_synchronise(cuda):
    tr = RPNTrainer(device=cuda, optimizer="adam_onecycle", total_steps=10, **DEVICE_PATHS)
    batch = _batch(cuda)
    tr.schedule_iteration(0, 0, 10)
    tr.step(*batch, grad_norm_clip=recipe.GRAD_NORM_CLIP)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        tr.schedule_epoch(0, 1)
        tr.schedule_iteration(1, 0, 10)
        tr.step(*batch, grad_norm_clip=recipe.GRAD_NORM_CLIP)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def _state_digest(tr):
    h = hashlib.sha256()
    for p in tr.params:
        h.update(p.detach().cpu().numpy().tobytes())
    for b in tr.model.buffers():
        h.update(b.detach().cpu().numpy().tobytes())
    for p in tr.params:
        for k, v in sorted(tr.opt.opt.state.get(p, {}).items()):
            h.update(v.detach().cpu().numpy().tobytes())
    return h.hexdigest()


def _worker():
    """two seeded runs of three scheduled onecycle steps under torch.use_deterministic_algorithms(True) -> JSON digests"""
    torch.use_deterministic_algorithms(True)
    dev = torch.device("cuda:0")
    batch = _batch(dev)
    res = []
    for _ in range(2):
        tr = RPNTrainer(device=dev, seed=3, optimizer="adam_onecycle", total_steps=10, **DEVICE_PATHS)
        for it in range(3):
            tr.schedule_iteration(it, 0, 10)
            tr.step(*batch, grad_norm_clip=recipe.GRAD_NORM_CLIP)
        res.append(_state_digest(tr))
    print("DIGESTS " + json.dumps(res))


def test_two_deterministic_onecycle_runs_end_with_the_same_bits(cuda):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker"], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    res = json.loads([l for l in r.stdout.splitlines() if l.startswith("DIGESTS ")][-1][len("DIGESTS "):])
    assert res[0] == res[1], "two seeded runs differ"


def _bn_layers(tr):
    """the BatchNorm layers of RPN SA module 0 and FP module 0"""
    bb = tr.model.backbone_net
    return [m for mod in (bb.SA_modules[0], bb.FP_modules[0]) for m in mod.modules() if isinstance(m, torch.nn.BatchNorm2d)]


def test_scheduled_bn_momentum_reaches_the_device_training_paths(cuda):
    """at it = 1000 the momentum halves; the running statistics the device SA / FP paths then update move like the torch
    path's (a device path still on momentum 0.1 would move them twice as far)"""
    batch = _batch(cuda)
    moved = {}
    for path in ("torch", "device"):
        tr = RPNTrainer(device=cuda, seed=3, loss_impl="device", sa_train=path, fp_train=path)
        tr.schedule_epoch(3, 1000)
        layers = _bn_layers(tr)
        assert layers and all(bn.momentum == 0.05 for bn in layers)
        before = [(bn.running_mean.clone(), bn.running_var.clone()) for bn in layers]
        tr.forward_loss(*batch)
        moved[path] = [(bn.running_mean - m0, bn.running_var - v0) for bn, (m0, v0) in zip(layers, before)]
    for k, ((tm, tv), (dm, dv)) in enumerate(zip(moved["torch"], moved["device"])):
        for name, t, d in (("mean", tm, dm), ("var", tv, dv)):
            rel = float(torch.linalg.norm(d - t) / torch.linalg.norm(t))
            assert rel <= 1e-2, (k, name, rel)


def test_rcnn_phase_from_a_phase1_checkpoint(cuda, tmp_path):
    """phase 1 -> checkpoint -> load_part into RCNNTrainer -> one scheduled RCNN step; the frozen RPN keeps the loaded
    weights (no decay, no gradient), and the RCNN-phase checkpoint loads into PointRCNNInference with strict keys"""
    from pointrcnn_b200.point_rcnn import PointRCNNInference
    rpn = RPNTrainer(device=cuda, seed=3, optimizer="adam_onecycle", total_steps=10, **DEVICE_PATHS)
    rpn.schedule_iteration(0, 0, 10)
    rpn.step(*_batch(cuda), grad_norm_clip=recipe.GRAD_NORM_CLIP)
    with torch.no_grad():
        rpn.model.rpn_reg_layer[-1].conv.weight.mul_(0.2)           # usable box sizes on near-random weights
    phase1 = str(tmp_path / "checkpoint_epoch_1.pth")
    recipe.save_checkpoint(rpn, phase1, 1, 1)
    saved = torch.load(phase1, map_location="cpu", weights_only=True)["model_state"]

    tr = RCNNTrainer(device=cuda, seed=5, optimizer="adam_onecycle", total_steps=10, loss_impl="device")
    assert recipe.load_part(tr.net, phase1) == len(saved)
    for k, v in tr.rpn.state_dict().items():
        assert torch.equal(v.cpu(), saved["rpn." + k]), k
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 321, channels=4)).to(cuda)
    rois = tr.rpn_outputs(pc, None)["roi_boxes3d"]
    gt = torch.zeros((2, 12, 7), device=cuda)
    gt[:, :8] = rois[:, ::40][:, :8]
    assert (gt[:, :8, 3:6] > 0).all(), "degenerate proposals"
    w0 = tr.model.cls_layer[0].conv.weight.detach().clone()
    tr.schedule_epoch(0, 0)
    tr.schedule_iteration(0, 0, 10)
    loss, _ = tr.step(pc, gt, grad_norm_clip=recipe.GRAD_NORM_CLIP)
    assert torch.isfinite(loss)
    assert not torch.equal(tr.model.cls_layer[0].conv.weight, w0)
    for k, v in tr.rpn.state_dict().items():
        assert torch.equal(v.cpu(), saved["rpn." + k]), "the fixed RPN changed: " + k

    phase2 = str(tmp_path / "rcnn.pth")
    recipe.save_checkpoint(tr, phase2, 1, 1)
    ckpt = torch.load(phase2, map_location="cpu", weights_only=True)
    inf = PointRCNNInference()
    inf.load_state_dict(ckpt["model_state"])
    assert len(ckpt["optimizer_state"]["param_groups"]) == 2


def test_fit_copies_once_per_epoch_and_writes_checkpoints(cuda, tmp_path):
    tr = RPNTrainer(device=cuda, seed=3, optimizer="adam_onecycle", total_steps=4, **DEVICE_PATHS)
    batches = [_batch(cuda, seed=s) for s in (11, 12)]
    tr.step(*batches[0])                         # first-call set-up (packing, workspaces) outside the counted loop
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            hist = recipe.fit(tr, batches, 2)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in caught if "synchroniz" in str(w.message)]
    assert len(syncs) == 2, [str(w.message) for w in syncs]
    assert len(hist) == 2 and all(h["loss"].shape == (2,) and np.isfinite(h["loss"]).all() for h in hist)
    assert {"rpn_loss_cls", "rpn_loss_reg"} <= set(hist[0])

    tr = RPNTrainer(device=cuda, seed=3, optimizer="adam_onecycle", total_steps=4, **DEVICE_PATHS)
    recipe.fit(tr, batches, 2, ckpt_dir=str(tmp_path), ckpt_every=1)
    assert sorted(os.listdir(tmp_path)) == ["checkpoint_epoch_1.pth", "checkpoint_epoch_2.pth"]
    ckpt = torch.load(str(tmp_path / "checkpoint_epoch_2.pth"), map_location="cpu", weights_only=True)
    assert (ckpt["epoch"], ckpt["it"]) == (2, 4)
    resumed = RPNTrainer(device=cuda, seed=9, optimizer="adam_onecycle", total_steps=4, **DEVICE_PATHS)
    assert recipe.load_checkpoint(resumed, str(tmp_path / "checkpoint_epoch_2.pth")) == (4, 2)
    assert all(torch.equal(a, b) for a, b in zip(tr.params, resumed.params))
    assert all(g["fused"] for g in resumed.opt.param_groups)


if __name__ == "__main__" and "--worker" in sys.argv:
    _worker()

"""Training steps replayed as CUDA graphs (RPNTrainer / RCNNTrainer with cuda_graph=True) on the device: eager and graphed
runs end with the same bits under torch.use_deterministic_algorithms(True), replays draw fresh RCNN samples and dropout
masks, replays do not synchronise with the host, the device-seed sampler entries equal the host-seed ones, the fused
eval caches follow the replayed weights, recipe.fit keeps one loss per iteration, and a 2-rank graphed step equals the
2-rank eager step when two GPUs are visible."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import synth
from pointrcnn_b200.train import recipe

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = 4


def _rpn_batch(dev, seed=123):
    from pointrcnn_b200.train.step import synthetic_labels
    pc = torch.from_numpy(synth.u_kitti(2, 16384, seed, channels=4)).to(dev)
    cls, reg = synthetic_labels(pc, seed=1)
    return pc, cls, reg


def _rcnn_batch(dev, seed=123):
    pc = torch.from_numpy(synth.u_kitti(2, 16384, seed, channels=4)).to(dev)
    gts = torch.from_numpy(np.stack([synth.boxes3d(4, s)[0] for s in (7, 8)]).astype(np.float32)).to(dev)
    return pc, gts


def _rpn(dev, graph, dropout=0.0, **kw):
    from pointrcnn_b200.train.step import RPNTrainer
    kw.setdefault("optimizer", "adam_onecycle")
    kw.setdefault("total_steps", 10)
    tr = RPNTrainer(device=dev, seed=3, loss_impl="device", cuda_graph=graph, **kw)
    for m in tr.model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = dropout
    return tr


def _rcnn(dev, graph, **kw):
    from pointrcnn_b200.train.step import RCNNTrainer
    kw.setdefault("optimizer", "adam_onecycle")
    kw.setdefault("total_steps", 10)
    kw.setdefault("gt_rows", 8)
    return RCNNTrainer(device=dev, seed=5, loss_impl="device", target_draw="device", cuda_graph=graph, **kw)


def _run(tr, batch, steps=STEPS, after_two=None):
    """`steps` steps with OneCycle's per-iteration schedule; the BN momentum drops at the last one (a recapture).
    after_two: called after the second step.  -> per step [loss, terms by name] as hex"""
    losses = []
    for it in range(steps):
        if it == 2 and after_two is not None:
            after_two()
        tr.schedule_iteration(it, 0, steps)
        if it == steps - 1:
            recipe.set_bn_momentum(tr.net, 0.05)
        loss, terms = tr.step(*batch, grad_norm_clip=1.0)
        losses.append([loss] + [terms[k] for k in sorted(terms)])
    return [[v.detach().float().cpu().numpy().tobytes().hex() for v in row] for row in losses]


def _state(tr):
    """hex of every parameter, gradient, buffer of the trained stage and Adam state tensor, by name"""
    out = {}
    for name, p in tr.model.named_parameters():
        out["p." + name] = p.detach().cpu().numpy().tobytes().hex()
        if p.grad is not None:
            out["g." + name] = p.grad.detach().cpu().numpy().tobytes().hex()
    for name, b in tr.model.named_buffers():
        out["b." + name] = b.detach().cpu().numpy().tobytes().hex()
    opt = getattr(tr.opt, "opt", tr.opt)
    for i, p in enumerate(tr.params):
        for k, v in sorted(opt.state.get(p, {}).items()):
            out["s.%d.%s" % (i, k)] = v.detach().float().cpu().numpy().tobytes().hex()
    return out


@torch.no_grad()
def _eval_rpn(tr, pc):
    tr.model.eval()
    try:
        rois, scores = tr.model(pc)
        return rois.cpu().numpy().tobytes().hex() + scores.cpu().numpy().tobytes().hex()
    finally:
        tr.model.train()


def _worker():
    """eager vs graphed runs under the deterministic flag -> one JSON line of per-case comparisons"""
    torch.use_deterministic_algorithms(True)
    dev = torch.device("cuda:0")
    res = {}
    rpn_batch, rcnn_batch = _rpn_batch(dev), _rcnn_batch(dev)
    for sw in ("torch", "device"):
        runs = []
        for graph in (False, True):
            tr = _rpn(dev, graph, sa_train=sw, fp_train=sw)
            mid = []        # an eval forward after step 2 builds the fused caches, which the later steps must invalidate
            losses = _run(tr, rpn_batch, after_two=lambda: mid.append(_eval_rpn(tr, rpn_batch[0])))
            ev_mid = mid[0]
            runs.append(dict(losses=losses, state=_state(tr), eval_mid=ev_mid, eval=_eval_rpn(tr, rpn_batch[0]),
                             graphs=len(tr._graphs)))
        res["rpn_" + sw] = runs
    runs = []
    for graph in (False, True):      # the trainers' default optimizer: fused Adam, the warm-up lr per iteration
        tr = _rpn(dev, graph, sa_train="device", fp_train="device", optimizer="adam", total_steps=None)
        runs.append(dict(losses=_run(tr, rpn_batch), state=_state(tr), graphs=len(tr._graphs)))
    res["rpn_adam"] = runs
    runs = []
    for graph in (False, True):
        tr = _rcnn(dev, graph)
        runs.append(dict(losses=_run(tr, rcnn_batch), state=_state(tr), graphs=len(tr._graphs)))
    res["rcnn"] = runs
    # zero GT rows up to gt_rows change nothing: an unpadded eager run against a padded one
    runs = []
    for rows in (None, 8):
        tr = _rcnn(dev, False, gt_rows=rows)
        runs.append(dict(losses=_run(tr, rcnn_batch), state=_state(tr), graphs=0))
    res["rcnn_padding"] = runs
    # a checkpoint loaded into a live trainer mid-run: RPN load_checkpoint, then RCNN load_part of that RPN
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "ckpt.pth")
        runs = []
        for graph in (False, True):
            tr = _rpn(dev, graph, sa_train="device", fp_train="device")
            losses = _run(tr, rpn_batch, 3)
            if not graph:
                recipe.save_checkpoint(tr, path, 0, 3)
            losses += _run(tr, rpn_batch, 1)
            recipe.load_checkpoint(tr, path)
            for it in (3, 4, 5):
                tr.schedule_iteration(it, 0, STEPS)
                loss, terms = tr.step(*rpn_batch, grad_norm_clip=1.0)
                losses.append([v.detach().float().cpu().numpy().tobytes().hex() for v in [loss] + [terms[k] for k in sorted(terms)]])
            runs.append(dict(losses=losses, state=_state(tr), graphs=len(tr._graphs)))
        res["rpn_load"] = runs
        runs = []
        for graph in (False, True):
            tr = _rcnn(dev, graph)
            losses = _run(tr, rcnn_batch, 2)
            recipe.load_part(tr.net, path)
            losses += _run(tr, rcnn_batch, 3)
            runs.append(dict(losses=losses, state=_state(tr), graphs=len(tr._graphs)))
        res["rcnn_load_part"] = runs
    print("RESULT " + json.dumps(res))


@pytest.fixture(scope="module")
def worker_result(cuda):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker"], capture_output=True, text=True, env=env, timeout=1500)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


def _same_run(eager, graphed, graphs):
    assert graphed["graphs"] == graphs, "graphs captured: %d, not %d" % (graphed["graphs"], graphs)
    assert graphed["losses"] == eager["losses"], "per-step losses differ"
    bad = [k for k in eager["state"] if eager["state"][k] != graphed["state"].get(k)]
    assert not bad and eager["state"].keys() == graphed["state"].keys(), "differing state: %s" % bad[:10]


@pytest.mark.parametrize("switch", ["torch", "device"])
def test_rpn_graphed_steps_equal_eager_bits(worker_result, switch):
    eager, graphed = worker_result["rpn_" + switch]
    _same_run(eager, graphed, 2)            # the BN-momentum change captures a second graph


def test_rcnn_graphed_steps_equal_eager_bits(worker_result):
    eager, graphed = worker_result["rcnn"]
    _same_run(eager, graphed, 1)            # the RCNN network has no BatchNorm (USE_BN False): no momentum is baked


def test_rpn_graphed_steps_with_the_default_optimizer_equal_eager_bits(worker_result):
    eager, graphed = worker_result["rpn_adam"]
    _same_run(eager, graphed, 2)


def test_gt_padding_leaves_the_rcnn_step_unchanged(worker_result):
    unpadded, padded = worker_result["rcnn_padding"]
    _same_run(unpadded, padded, 0)


@pytest.mark.parametrize("case", ["rpn_load", "rcnn_load_part"])
def test_a_checkpoint_loaded_mid_run_equals_eager(worker_result, case):
    eager, graphed = worker_result[case]
    # after the load: one eager step, then a capture; the RPN's momentum is one value throughout the last steps
    _same_run(eager, graphed, 1)


@pytest.mark.parametrize("switch", ["torch", "device"])
def test_fused_eval_follows_replayed_weights(worker_result, switch):
    eager, graphed = worker_result["rpn_" + switch]
    assert graphed["eval_mid"] == eager["eval_mid"]
    assert graphed["eval"] == eager["eval"], "an eval forward after graphed steps used stale packed weights"
    assert graphed["eval"] != graphed["eval_mid"]


# ------------------------------------------------------------------------------------------ fresh draws on replay
def _replay_losses(tr, batch, n):
    out = []
    for _ in range(n):
        loss, _ = tr.step(*batch)
        out.append(float(loss))
    return out


def test_replays_draw_fresh_rcnn_samples(cuda):
    batch = _rcnn_batch(cuda)
    tr = _rcnn(cuda, True, optimizer="adam", total_steps=None, lr=0.0, weight_decay=0.0)
    layer = tr.model.proposal_target_layer
    losses = _replay_losses(tr, batch, 4)            # lr 0: the loss changes only with the samples
    assert int(layer.seed_counter.item()) == 4, "the captured step must advance the device seed on every replay"
    assert len(set(losses[1:])) == 3, losses
    again = _replay_losses(_rcnn(cuda, True, optimizer="adam", total_steps=None, lr=0.0, weight_decay=0.0), batch, 4)
    assert again == losses, "two graphed runs from the same seed differ"


def test_replays_draw_fresh_dropout_masks(cuda):
    batch = _rpn_batch(cuda)
    losses = _replay_losses(_rpn(cuda, True, dropout=0.5, optimizer="adam", total_steps=None, lr=0.0, weight_decay=0.0), batch, 4)
    assert len(set(losses[1:])) == 3, losses
    again = _replay_losses(_rpn(cuda, True, dropout=0.5, optimizer="adam", total_steps=None, lr=0.0, weight_decay=0.0), batch, 4)
    assert again == losses, "two graphed runs from the same seed differ"
    still = _replay_losses(_rpn(cuda, True, dropout=0.0, optimizer="adam", total_steps=None, lr=0.0, weight_decay=0.0), batch, 4)
    assert len(set(still[1:])) == 1, still


# ------------------------------------------------------------------------------------------ no host synchronisation
@pytest.mark.parametrize("which", ["rpn", "rcnn"])
def test_replays_do_not_synchronise(cuda, which):
    tr, batch = (_rpn(cuda, True), _rpn_batch(cuda)) if which == "rpn" else (_rcnn(cuda, True), _rcnn_batch(cuda))
    for it in range(2):
        tr.schedule_iteration(it, 0, 6)
        tr.step(*batch, grad_norm_clip=1.0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for it in range(2, 6):
            tr.schedule_iteration(it, 0, 6)
            tr.step(*batch, grad_norm_clip=1.0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ device-seed entries
def test_device_seed_entries_equal_host_seed_entries(cuda):
    from pointrcnn_b200.rcnn import targets
    rng = np.random.default_rng(0)
    B, N, M, G = 3, 2048, 128, 4
    xyz = torch.from_numpy(rng.normal(0, 8, (B, N, 3)).astype(np.float32)).to(cuda)
    feat = torch.from_numpy(rng.normal(0, 1, (B, N, 5)).astype(np.float32)).to(cuda)
    gts = torch.from_numpy(np.stack([synth.boxes3d(G, s)[0] for s in (1, 2, 3)]).astype(np.float32)).to(cuda)
    rois = gts.repeat_interleave(M // G, dim=1) + torch.from_numpy(rng.normal(0, 0.6, (B, M, 7)).astype(np.float32)).to(cuda)
    rois[..., 3:6] = rois[..., 3:6].abs() + 0.5
    rc = targets.layer_recipe(targets.ns(targets.DEFAULT_CFG))
    for seed in (0, 7, 0xfffffffe):
        host = targets.run(rc, xyz, feat, rois.contiguous(), gts, None, seed)
        dev = targets.run(rc, xyz, feat, rois.contiguous(), gts, None, 12345,
                          seed_dev=torch.tensor([seed], dtype=torch.int64).to(torch.int32).to(cuda))
        for k in host:
            assert torch.equal(host[k].view(torch.int32) if host[k].dtype == torch.float32 else host[k],
                               dev[k].view(torch.int32) if dev[k].dtype == torch.float32 else dev[k]), (seed, k)
    other = targets.run(rc, xyz, feat, rois.contiguous(), gts, None, 8)
    assert not torch.equal(other["rois"], targets.run(rc, xyz, feat, rois.contiguous(), gts, None, 7)["rois"])


# ------------------------------------------------------------------------------------------ recipe.fit
def test_fit_returns_distinct_per_iteration_losses(cuda):
    tr = _rpn(cuda, True, optimizer="adam_onecycle", total_steps=5)
    batch = _rpn_batch(cuda)
    hist = recipe.fit(tr, [batch] * 5, epochs=1)
    loss = hist[0]["loss"]
    assert loss.shape == (5,) and np.isfinite(loss).all()
    assert len(set(loss.tolist())) == 5, loss


# ------------------------------------------------------------------------------------------ two ranks
def _rank(rank, path, out):
    import torch.distributed as dist
    from pointrcnn_b200.train.step import RPNTrainer
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="file://" + path, rank=rank, world_size=2)
    dev = torch.device("cuda", rank)
    batch = _rpn_batch(dev, seed=200 + rank)
    res = []
    for graph in (False, True):
        tr = RPNTrainer(device=dev, world=2, seed=3, loss_impl="device", cuda_graph=graph)
        for m in tr.model.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        for _ in range(3):
            tr.step(*batch, grad_norm_clip=1.0)
        res.append(torch.cat([p.detach().reshape(-1) for p in tr.params]).cpu())
    torch.save(res, out + ".%d" % rank)
    dist.destroy_process_group()


def test_two_rank_graphed_step_equals_eager(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_rank, args=(os.path.join(d, "init"), os.path.join(d, "out")), nprocs=2)
        for r in range(2):
            eager, graphed = torch.load(os.path.join(d, "out.%d" % r))
            # the same step; without the deterministic flag the scatter gradients add with atomics, hence the tolerance
            assert torch.allclose(eager, graphed, rtol=1e-4, atol=1e-6), "rank %d" % r


if __name__ == "__main__" and "--worker" in sys.argv:
    _worker()

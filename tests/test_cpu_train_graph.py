"""The host side of CUDA-graph training steps (cuda_graph=True): the refusals raise before anything is captured, the
graph cache key changes exactly when a value a replay cannot change does, and the schedule hooks of a graphed trainer
write into the optimizer's device tensors in place instead of storing new Python floats."""
import contextlib

import pytest
import torch
from torch import nn

from pointrcnn_b200 import _cabi as C
from pointrcnn_b200 import config
from pointrcnn_b200.train import recipe, step
from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer, _Recipe
from test_cpu_deterministic_grads import _FakeLib


@pytest.fixture
def fake_lib(monkeypatch):
    lib = _FakeLib()
    monkeypatch.setattr(C, "lib", lambda: lib)
    monkeypatch.setattr(C, "stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    return lib


@pytest.fixture
def no_capture(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a graph was captured")
    monkeypatch.setattr(torch.cuda, "CUDAGraph", refuse)
    monkeypatch.setattr(torch.cuda, "graph", refuse)


# ------------------------------------------------------------------------------------------ refusals
def test_a_cpu_device_is_refused_at_construction():
    with pytest.raises(ValueError, match="CUDA device"):
        RPNTrainer(device="cpu", loss_impl="device", cuda_graph=True)
    with pytest.raises(ValueError, match="CUDA device"):
        RCNNTrainer(device="cpu", loss_impl="device", target_draw="device", cuda_graph=True)


@pytest.mark.parametrize("kw, match", [(dict(loss_impl="torch"), "loss_impl"),
                                       (dict(loss_impl="device", target_draw="torch"), "target_draw")])
def test_torch_paths_are_refused(kw, match):
    cuda = torch.device("cuda")
    assert match in step._graph_refusal(cuda, kw["loss_impl"], kw.get("target_draw", "device"))
    assert step._graph_refusal(cuda, "device", "device") is None
    assert step._graph_refusal(cuda, "device", False) is None


def _graphed_on_paper(tr):
    """a CPU trainer that takes the cuda_graph branch, as far as the refusals go"""
    tr.cuda_graph, tr._warm, tr._graphs = True, True, {}
    tr.device = torch.device("cuda")
    return tr


def test_the_torch_loss_path_is_refused_at_the_step_before_capture(no_capture):
    tr = _graphed_on_paper(RPNTrainer(device="cpu"))                   # loss_impl None: the config switch, "torch"
    pts = torch.zeros(1, 64, 4)
    with config.override(loss_impl="torch"), pytest.raises(ValueError, match="loss_impl"):
        tr.step(pts, torch.zeros(1, 64, dtype=torch.long), torch.zeros(1, 64, 7))


def test_the_torch_target_draw_is_refused_at_the_step_before_capture(no_capture):
    tr = _graphed_on_paper(RCNNTrainer(device="cpu", loss_impl="device"))
    with config.override(target_draw="torch"), pytest.raises(ValueError, match="target_draw"):
        tr.step(torch.zeros(1, 64, 4), torch.zeros(1, 2, 7))


def test_cached_autocast_is_refused_at_the_step_before_capture(no_capture, monkeypatch):
    tr = _graphed_on_paper(RPNTrainer(device="cpu", loss_impl="device"))
    monkeypatch.setattr(torch, "is_autocast_enabled", lambda *a: True)
    monkeypatch.setattr(torch, "is_autocast_cache_enabled", lambda: True)
    with pytest.raises(ValueError, match="cache_enabled=False"):
        tr.step(torch.zeros(1, 64, 4), torch.zeros(1, 64, dtype=torch.long), torch.zeros(1, 64, 7))
    monkeypatch.setattr(torch, "is_autocast_cache_enabled", lambda: False)
    assert step._graph_refusal(torch.device("cuda"), "device") is None


def test_a_batch_over_the_gt_capacity_is_refused(no_capture):
    tr = RCNNTrainer(device="cpu", loss_impl="device", target_draw="device", gt_rows=4)
    with pytest.raises(ValueError, match="gt_rows=4"):
        tr.step(torch.zeros(1, 64, 4), torch.zeros(1, 5, 7))


# ------------------------------------------------------------------------------------------ the graph cache key
def test_the_key_changes_exactly_when_a_baked_value_changes(monkeypatch):
    tr = RPNTrainer(device="cpu", loss_impl="device")
    inputs = (torch.zeros(2, 64, 4), torch.zeros(2, 64, dtype=torch.long), torch.zeros(2, 64, 7))
    base = tr.graph_key(inputs, 1.0)
    assert tr.graph_key(tuple(t.clone() + 1 for t in inputs), 1.0) == base, "input values are not part of the key"
    recipe.set_bn_momentum(tr.net, 0.1)
    assert tr.graph_key(inputs, 1.0) == base, "the same momentum again"
    tr.schedule_iteration(5, 0, 10)
    assert tr.graph_key(inputs, 1.0) == base, "the lr schedule reaches replays through tensors"
    changed = [tr.graph_key(inputs, None), tr.graph_key(inputs, 0.5),
               tr.graph_key((torch.zeros(4, 64, 4),) + inputs[1:], 1.0)]
    recipe.set_bn_momentum(tr.net, 0.05)
    changed.append(tr.graph_key(inputs, 1.0))
    recipe.set_bn_momentum(tr.net, 0.1)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        changed.append(tr.graph_key(inputs, 1.0))
    finally:
        torch.use_deterministic_algorithms(was)
    monkeypatch.setattr(torch, "is_autocast_enabled", lambda *a: True)
    for dtype in (torch.bfloat16, torch.float16):
        monkeypatch.setattr(torch, "get_autocast_dtype", lambda *a, d=dtype: d)
        changed.append(tr.graph_key(inputs, 1.0))
    assert all(k != base for k in changed)
    assert len(set(changed)) == len(changed)


# ------------------------------------------------------------------------------------------ schedule hooks
class GraphedSmall(_Recipe):
    """the trainers' optimizer switch in graph mode over a small module"""

    def __init__(self, optimizer):
        self.device = torch.device("cpu")
        self.cuda_graph = True
        self.net = nn.Sequential(nn.Conv1d(4, 8, 1), nn.BatchNorm1d(8), nn.ReLU(), nn.Conv1d(8, 3, 1))
        self.params = list(self.net.parameters())
        self._build_optimizer(recipe.OneCycle(20) if optimizer == "adam_onecycle" else None, recipe.LR, recipe.WEIGHT_DECAY)


@pytest.mark.parametrize("optimizer", ["adam", "adam_onecycle"])
def test_graphed_schedule_hooks_write_into_the_tensors(optimizer):
    t = GraphedSmall(optimizer)
    groups = t.opt.param_groups
    lrs = [g["lr"] for g in groups]
    assert all(torch.is_tensor(v) and v.numel() == 1 for v in lrs)
    ptrs = [v.data_ptr() for v in lrs]
    for it in (0, 7, 15):
        t.schedule_iteration(it, 0, 20)
        assert [g["lr"] for g in groups] == lrs or all(a is b for a, b in zip((g["lr"] for g in groups), lrs))
        assert [g["lr"].data_ptr() for g in groups] == ptrs
        if optimizer == "adam_onecycle":
            lr, mom = t.schedule(it)
            assert t.opt.hyper.tolist()[:2] == [lr, mom]
            assert all(torch.is_tensor(g["betas"][0]) and float(g["betas"][0]) == mom for g in groups)
        else:
            want = recipe.warmup_lr(it, recipe.WARMUP_EPOCH * 20, recipe.LR)
            assert float(groups[0]["lr"]) == torch.tensor(want, dtype=torch.float32).item()
    t.schedule_epoch(5, 1500)
    assert [g["lr"].data_ptr() for g in groups] == ptrs


def test_graphed_true_wd_adam_steps_through_one_device_entry(fake_lib):
    t = GraphedSmall("adam_onecycle")
    for p in t.params:
        p.grad = torch.ones_like(p)
    t.opt.step()
    t.opt.step()
    assert fake_lib.calls == ["prb_adam_true_wd_step"] * 2
    state = t.opt.opt.state
    assert all(float(state[p]["step"]) == 2.0 for p in t.params), "the step counters advance before each launch"
    sd = t.opt.state_dict()
    assert all(isinstance(g["lr"], float) and isinstance(g["betas"][0], float) for g in sd["param_groups"])
    t.opt.load_state_dict(sd)
    assert torch.is_tensor(t.opt.param_groups[0]["lr"]) and t.opt._table is None


def _graphed_cpu(trainer):
    """a CPU trainer with the graph bookkeeping of cuda_graph=True: the load hook, a warm flag and one cached graph"""
    trainer._init_graphs(True)
    trainer._warm = True
    trainer._graphs[("key",)] = object()
    return trainer


def test_load_checkpoint_and_load_part_drop_the_graphs_and_the_warm_step(tmp_path):
    path = str(tmp_path / "ckpt.pth")
    rpn = _graphed_cpu(RPNTrainer(device="cpu", loss_impl="device", optimizer="adam_onecycle", total_steps=10))
    recipe.save_checkpoint(rpn, path, 0, 3)
    assert recipe.load_checkpoint(rpn, path) == (3, 0)
    assert rpn._graphs == {} and not rpn._warm, "the next step must run eager, then capture again"
    rcnn = _graphed_cpu(RCNNTrainer(device="cpu", loss_impl="device", target_draw="device"))
    assert recipe.load_part(rcnn.net, path) > 0
    assert rcnn._graphs == {} and not rcnn._warm


def test_the_key_follows_the_config_switches_the_trainer_leaves_to_the_config():
    inputs = (torch.zeros(2, 64, 4), torch.zeros(2, 64, dtype=torch.long), torch.zeros(2, 64, 7))
    free = RPNTrainer(device="cpu", loss_impl="device")
    fixed = RPNTrainer(device="cpu", loss_impl="device", sa_train="device", fp_train="torch")
    keys = {}
    for sw in (dict(), dict(sa_train="device"), dict(fp_train="device"), dict(disable_fused=True)):
        with config.override(**sw):
            keys[tuple(sw.items())] = (free.graph_key(inputs, 1.0), fixed.graph_key(inputs, 1.0))
    free_keys = [k[0] for k in keys.values()]
    assert len(set(free_keys)) == 4
    assert keys[(("sa_train", "device"),)][1] == keys[()][1], "an explicit sa_train is the trainer's, not the config's"
    assert keys[(("fp_train", "device"),)][1] == keys[()][1]
    assert keys[(("disable_fused", True),)][1] != keys[()][1]

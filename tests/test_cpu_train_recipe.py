"""The training recipe of train/recipe.py against the reference's own code (tests/golden/train_recipe.npz, written by
oracle/make_golden_train_recipe.py): OneCycle, warm-up, step-decay and BN-momentum schedules value for value, the
OptimWrapper parameter groups of both training phases by name, the true-weight-decay Adam trajectory, loading a
reference-written optimizer_state, and checkpoints that resume bit for bit."""
import io
import os

import numpy as np
import pytest
import torch
from torch import nn

from pointrcnn_b200.train import recipe
from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer, _Recipe

with np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_recipe.npz")) as _z:
    GOLD = dict(_z)
TRAJ_TOTAL, TRAJ_STEPS, TRAJ_SAVE = (int(v) for v in GOLD["traj_consts"])
WARMUP_ITERS, BNM_ITERS = (int(v) for v in GOLD["consts"])
NAMES = list(GOLD["traj_names"])


def small_module():
    """oracle/make_golden_train_recipe.py small_module()"""
    return nn.Sequential(nn.Conv1d(4, 8, 1), nn.BatchNorm1d(8), nn.ReLU(), nn.Conv1d(8, 3, 1))


class SmallTrainer(_Recipe):
    """the trainers' optimizer switch and schedule hooks over the golden's small module, stepped on the golden gradients"""

    def __init__(self, optimizer="adam_onecycle", total_steps=TRAJ_TOTAL):
        self.device = torch.device("cpu")
        self.net = small_module()
        with torch.no_grad():
            for n, p in self.net.named_parameters():
                p.copy_(torch.from_numpy(GOLD["traj_init_" + n]))
        self.params = list(self.net.parameters())
        self._build_optimizer(recipe.OneCycle(total_steps) if optimizer == "adam_onecycle" else None, recipe.LR, recipe.WEIGHT_DECAY)

    def run(self, its):
        for it in its:
            self.schedule_iteration(it, 0, TRAJ_TOTAL)
            for n, p in self.net.named_parameters():
                p.grad = torch.from_numpy(GOLD["traj_grad%d_%s" % (it, n)].copy())
            self.opt.step()


def _check_state(trainer, tag):
    for n, p in trainer.net.named_parameters():
        st = trainer.opt.opt.state[p]
        for got, key in ((p.detach(), "param"), (st["exp_avg"], "exp_avg"), (st["exp_avg_sq"], "exp_avg_sq")):
            want = GOLD["traj_%s_%s_%s" % (tag, key, n)]
            np.testing.assert_allclose(got.numpy(), want, rtol=1e-7, atol=0, err_msg="%s %s" % (key, n))


@pytest.mark.parametrize("total", [3, 7, 37, 1000])
def test_onecycle_matches_the_reference_at_every_step(total):
    sched = recipe.OneCycle(total)
    np.testing.assert_allclose(sched.initial, GOLD["onecycle_%d_init" % total], rtol=1e-15, atol=0)
    got = np.array([sched(it) for it in range(total + 5)])          # past total_step the cosine extrapolates
    # np.cos (reference) and math.cos may differ in the last bit; near the end of a phase cos + 1 ~ 0 amplifies that
    np.testing.assert_allclose(got[:, 0], GOLD["onecycle_%d_lr" % total], rtol=1e-12, atol=0)
    np.testing.assert_allclose(got[:, 1], GOLD["onecycle_%d_mom" % total], rtol=1e-12, atol=0)


@pytest.mark.parametrize("total", [0, 1, 2])
def test_onecycle_refuses_an_empty_phase(total):
    with pytest.raises(ValueError):
        recipe.OneCycle(total)


def test_adam_warmup_and_step_decay_match_the_reference():
    t = SmallTrainer("adam")
    got, it = [], 0
    for epoch in range(2):
        t.schedule_epoch(epoch, it)
        for _ in range(WARMUP_ITERS):
            t.schedule_iteration(it, epoch, WARMUP_ITERS)
            got.append(t.opt.param_groups[0]["lr"])
            it += 1
    np.testing.assert_array_equal(got, GOLD["warmup_lr"])
    dec = []
    for epoch in GOLD["decay_epoch"]:
        t.schedule_epoch(int(epoch), 0)
        dec.append(t.opt.param_groups[0]["lr"])
    np.testing.assert_array_equal(dec, GOLD["decay_lr"])


def test_bn_momentum_follows_the_iteration_count_and_the_resume_quirk():
    t = SmallTrainer()
    got = [t.net[1].momentum]
    for it in GOLD["bnm_it"][1:]:
        t.schedule_epoch(0, int(it))
        got.append(t.net[1].momentum)
    np.testing.assert_array_equal(got, GOLD["bnm_mom"])
    res = []
    for start_epoch in GOLD["bnm_resume_epoch"]:
        t.resume_schedule(0, int(start_epoch))
        res.append(t.net[1].momentum)
    np.testing.assert_array_equal(res, GOLD["bnm_resume_mom"])


@pytest.mark.parametrize("phase", ["rpn", "rcnn"])
def test_parameter_groups_match_the_reference_point_rcnn(phase):
    t = (RPNTrainer if phase == "rpn" else RCNNTrainer)(device="cpu", optimizer="adam_onecycle", total_steps=10)
    names = {id(p): n for n, p in t.net.named_parameters()}
    groups = t.opt.opt.param_groups
    assert len(groups) == 2
    for g, pg in enumerate(groups):
        assert [names[id(p)] for p in pg["params"]] == list(GOLD["groups_%s_%d" % (phase, g)])
        assert pg["weight_decay"] == 0 and pg["betas"] == (recipe.MOMS[0], recipe.BETA2) and pg["lr"] == recipe.LR / recipe.DIV_FACTOR
    frozen = [n for n, p in t.net.named_parameters() if not p.requires_grad]
    assert all(n.startswith("rpn.") for n in frozen) and bool(frozen) == (phase == "rcnn")


def test_true_weight_decay_adam_trajectory_matches_the_reference():
    t = SmallTrainer()
    t.run(range(TRAJ_SAVE))
    _check_state(t, "save")
    t.run(range(TRAJ_SAVE, TRAJ_STEPS))
    _check_state(t, "end")
    # the all-zero gradient still steps Adam (its moments stay zero) and the parameter is still decayed
    bias = t.net[3].bias
    assert torch.count_nonzero(t.opt.opt.state[bias]["exp_avg"]) == 0
    assert not np.array_equal(bias.detach().numpy(), GOLD["traj_init_3.bias"])


def _save_as_reference(obj, path):
    """torch.save as the reference's PyTorch 1.0 with numpy 1.x wrote its files: the legacy (non-zip) format, with numpy
    scalars pickled under numpy 1.x's global name numpy.core.multiarray.scalar (numpy 2 writes numpy._core...)"""
    buf = io.BytesIO()
    torch.save(obj, buf, _use_new_zipfile_serialization=False)
    raw = buf.getvalue()
    new, old = b"cnumpy._core.multiarray\nscalar\n", b"cnumpy.core.multiarray\nscalar\n"
    assert new in raw
    with open(path, "wb") as f:
        f.write(raw.replace(new, old))


def _reference_checkpoint(path):
    """a checkpoint as the reference writes it after TRAJ_SAVE steps: torch 1.x Adam state (integer step, no fused / foreach
    / capturable keys) and OneCycle's numpy float64 lr and betas in the groups, in the reference's file format"""
    idx, counts = list(GOLD["ckpt_index"]), list(GOLD["ckpt_group_params"])
    state = {int(i): {"step": int(GOLD["ckpt_step_%d" % i]), "exp_avg": torch.from_numpy(GOLD["ckpt_exp_avg_%d" % i]),
                      "exp_avg_sq": torch.from_numpy(GOLD["ckpt_exp_avg_sq_%d" % i])} for i in idx}
    groups, at = [], 0
    for g, n in enumerate(counts):
        b1, b2 = GOLD["ckpt_group_betas"][g]
        groups.append({"lr": np.float64(GOLD["ckpt_group_lr"][g]), "betas": (np.float64(b1), float(b2)), "eps": float(GOLD["ckpt_group_eps"][g]),
                       "weight_decay": float(GOLD["ckpt_group_weight_decay"][g]), "amsgrad": bool(GOLD["ckpt_group_amsgrad"][g]),
                       "params": [int(i) for i in idx[at:at + n]]})
        at += n
    model = small_module().state_dict()
    for n in NAMES:
        model[n] = torch.from_numpy(GOLD["traj_save_param_" + n])
    _save_as_reference({"epoch": 1, "it": TRAJ_SAVE, "model_state": model, "optimizer_state": {"state": state, "param_groups": groups}}, path)


def test_reference_optimizer_state_loads_and_continues(tmp_path):
    path = str(tmp_path / "ref.pth")
    _reference_checkpoint(path)
    t = SmallTrainer()
    assert recipe.load_checkpoint(t, path) == (TRAJ_SAVE, 1)
    assert t.opt.param_groups[0]["weight_decay"] == 0 and t.opt.wd == recipe.WEIGHT_DECAY
    t.run(range(TRAJ_SAVE, TRAJ_STEPS))
    _check_state(t, "end")


def test_save_load_continue_equals_an_uninterrupted_run(tmp_path):
    whole = SmallTrainer()
    whole.run(range(TRAJ_STEPS))
    part = SmallTrainer()
    part.run(range(TRAJ_SAVE))
    path = str(tmp_path / "checkpoint_epoch_1.pth")
    recipe.save_checkpoint(part, path, 1, TRAJ_SAVE)
    resumed = SmallTrainer()
    assert recipe.load_checkpoint(resumed, path) == (TRAJ_SAVE, 1)
    resumed.run(range(TRAJ_SAVE, TRAJ_STEPS))
    for (n, a), b in zip(whole.net.named_parameters(), resumed.net.parameters()):
        assert torch.equal(a, b), n
        sa, sb = whole.opt.opt.state[a], resumed.opt.opt.state[b]
        assert all(torch.equal(sa[k], sb[k]) for k in ("step", "exp_avg", "exp_avg_sq")), n
    assert whole.opt.param_groups[0]["lr"] == resumed.opt.param_groups[0]["lr"]


@pytest.mark.parametrize("cls", [RPNTrainer, RCNNTrainer])
def test_adam_default_builds_todays_optimizer(cls):
    t = cls(device="cpu")
    assert type(t.opt) is torch.optim.Adam and len(t.opt.param_groups) == 1
    today = torch.optim.Adam(t.params, lr=0.002, weight_decay=0.001)
    assert t.opt.param_groups[0]["params"] == t.params
    assert {k: v for k, v in t.opt.param_groups[0].items() if k != "params"} == {k: v for k, v in today.param_groups[0].items() if k != "params"}


@pytest.mark.parametrize("kw", [dict(optimizer="sgd"), dict(optimizer="adamw", total_steps=10), dict(optimizer="adam_onecycle"),
                                dict(optimizer="adam_onecycle", total_steps=2)])
def test_bad_optimizer_arguments_raise(kw):
    with pytest.raises(ValueError):
        RPNTrainer(device="cpu", **kw)


def test_load_part_takes_the_rpn_of_a_phase1_checkpoint(tmp_path):
    rpn = RPNTrainer(device="cpu", seed=1, optimizer="adam_onecycle", total_steps=10)
    path = str(tmp_path / "rpn.pth")
    recipe.save_checkpoint(rpn, path, 5, 50)
    saved = torch.load(path, weights_only=True)["model_state"]
    assert set(saved) == {"rpn." + k for k in rpn.model.state_dict()}
    rcnn = RCNNTrainer(device="cpu", seed=0, optimizer="adam_onecycle", total_steps=10)
    before = {k: v.clone() for k, v in rcnn.model.state_dict().items()}
    assert recipe.load_part(rcnn.net, path) == len(saved)
    assert all(torch.equal(v, saved["rpn." + k]) for k, v in rcnn.rpn.state_dict().items())
    assert all(torch.equal(v, before[k]) for k, v in rcnn.model.state_dict().items())
    torch.save({"model_state": {"backbone.weight": torch.zeros(1)}}, str(tmp_path / "other.pth"))
    with pytest.raises(RuntimeError):
        recipe.load_part(rcnn.net, str(tmp_path / "other.pth"))


def test_load_part_reads_a_reference_written_phase1_checkpoint(tmp_path):
    """--rpn_ckpt from a file in the reference's format: its optimizer_state groups hold numpy 1.x float64 scalars"""
    rpn = RPNTrainer(device="cpu", seed=1, optimizer="adam_onecycle", total_steps=10)
    opt = rpn.opt.state_dict()
    for g in opt["param_groups"]:
        g["lr"], g["betas"] = np.float64(g["lr"]), (np.float64(g["betas"][0]), g["betas"][1])
    path = str(tmp_path / "checkpoint_epoch_100.pth")
    _save_as_reference({"epoch": 100, "it": 1000, "model_state": rpn.net.state_dict(), "optimizer_state": opt}, path)
    rcnn = RCNNTrainer(device="cpu", seed=0, optimizer="adam_onecycle", total_steps=10)
    assert recipe.load_part(rcnn.net, path) == len(rpn.net.state_dict())
    assert all(torch.equal(v, w) for v, w in zip(rcnn.rpn.state_dict().values(), rpn.model.state_dict().values()))


def test_fit_lines_every_term_up_with_its_iteration(tmp_path):
    class TermTrainer(SmallTrainer):
        """stepped by fit with the loss terms of the torch loss path, whose regression terms are missing in an iteration
        without a foreground point (here iteration 1 of each epoch)"""

        def step(self, k, grad_norm_clip=None):
            for n, p in self.net.named_parameters():
                p.grad = torch.from_numpy(GOLD["traj_grad%d_%s" % (k, n)].copy())
            self.opt.step()
            terms = {"rpn_loss_cls": torch.tensor(10.0 + k)}
            if k != 1:
                terms["loss_size"] = torch.tensor(20.0 + k)
            return torch.tensor(float(k)), terms

    t = TermTrainer()
    hist = recipe.fit(t, [(0,), (1,), (2,)], 2, ckpt_dir=str(tmp_path), ckpt_every=2)
    assert len(hist) == 2
    for h in hist:
        np.testing.assert_array_equal(h["loss"], [0, 1, 2])
        np.testing.assert_array_equal(h["rpn_loss_cls"], [10, 11, 12])
        np.testing.assert_array_equal(h["loss_size"], [20, np.nan, 22])
    assert sorted(os.listdir(tmp_path)) == ["checkpoint_epoch_2.pth"]
    assert recipe.load_checkpoint(TermTrainer(), str(tmp_path / "checkpoint_epoch_2.pth")) == (6, 2)

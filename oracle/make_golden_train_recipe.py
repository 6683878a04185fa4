"""oracle/make_golden_train_recipe.py -- golden schedules, parameter groups and optimizer trajectories of the reference's
training recipe.  TEST INFRASTRUCTURE ONLY.
    python oracle/make_golden_train_recipe.py

Runs the reference's OWN code on the CPU and writes tests/golden/train_recipe.npz:
  - create_optimizer and create_scheduler, their source taken from tools/train_rcnn.py (which parses the command line when
    imported) with `ast`, on cfgs/default.yaml;
  - tools/train_utils/{fastai_optim,learning_schedules_fastai,train_utils}.py imported unchanged; fastai_optim.py does
    `from collections import Iterable`, which Python 3.10 removed, so `collections.Iterable` is supplied before the import;
  - the scheduler calls of Trainer.train (train_utils.py:170-240) replayed in its order, without data.
Recorded:
  - onecycle_<T>_{lr,mom}: OneCycle's lr / momentum after step(it) for it in [0, T + 5) (steps past the end extrapolate);
    onecycle_<T>_init: the values OneCycle writes when it is built;
  - warmup_{lr,epoch,it}: OPTIMIZER=adam, the lr each training iteration runs with over two epochs of WARMUP_ITERS
    iterations (LambdaLR built first, then CosineWarmupLR on the same optimizer); decay_{epoch,lr}: the LambdaLR step at the
    start of epochs 1..220;
  - bnm_{it,mom}: BN momentum at each epoch start (BNMomentumScheduler.step(it)) with BNM_ITERS iterations per epoch;
    bnm_resume_{epoch,mom}: the momentum the scheduler's constructor sets on resume (last_epoch = start_epoch + 1);
  - groups_{rpn,rcnn}_{0,1}: the state-dict names of the parameters in the OptimWrapper's two groups for
    PointRCNN(num_classes=2, mode='TRAIN') with --train_mode rpn / rcnn (built with dropin.activate());
  - traj_*: the small conv + BN + ReLU module of `small_module()` trained by OptimWrapper + OneCycle(TRAJ_TOTAL) for
    TRAJ_STEPS steps on seeded gradients (the last conv's bias gets an all-zero gradient): initial parameters, the
    gradients, the parameters and Adam state after TRAJ_SAVE steps and after TRAJ_STEPS;
  - ckpt_*: the inner Adam's state_dict() after TRAJ_SAVE steps, as the reference writes it into 'optimizer_state': per
    parameter index its step (an integer, as torch 1.x stores it), exp_avg and exp_avg_sq; the group hyperparameters.
"""
import ast
import collections
import collections.abc
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "train_recipe.npz")

ONECYCLE_TOTALS = (3, 7, 37, 1000)
WARMUP_ITERS = 6
BNM_ITERS = 300
BNM_RESUME_EPOCHS = (0, 5, 997, 998, 1000)
TRAJ_TOTAL, TRAJ_STEPS, TRAJ_SAVE = 9, 7, 3


def small_module():
    """the trajectory module (tests/test_cpu_train_recipe.py builds the same one): conv + BN + ReLU + conv"""
    return nn.Sequential(nn.Conv1d(4, 8, 1), nn.BatchNorm1d(8), nn.ReLU(), nn.Conv1d(8, 3, 1))


def reference_namespace(cfg):
    """create_optimizer / create_scheduler from tools/train_rcnn.py, in a namespace with the module's own imports"""
    from functools import partial

    import torch.optim as optim
    import torch.optim.lr_scheduler as lr_sched
    import tools.train_utils.train_utils as train_utils
    from tools.train_utils import learning_schedules_fastai as lsf
    from tools.train_utils.fastai_optim import OptimWrapper
    src = open(os.path.join(REF, "tools", "train_rcnn.py")).read()
    nodes = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in ("create_optimizer", "create_scheduler")]
    ns = dict(torch=torch, optim=optim, lr_sched=lr_sched, nn=nn, partial=partial, cfg=cfg, train_utils=train_utils, lsf=lsf,
              OptimWrapper=OptimWrapper)
    exec(compile(ast.Module(body=nodes, type_ignores=[]), "train_rcnn.py", "exec"), ns)
    return ns


def onecycle(ns, cfg, out):
    cfg.TRAIN.OPTIMIZER = "adam_onecycle"
    cfg.RPN.ENABLED, cfg.RPN.FIXED = True, False
    for total in ONECYCLE_TOTALS:
        model = small_module()
        ns["model"] = model
        opt = ns["create_optimizer"](model)
        sched, _ = ns["create_scheduler"](opt, total_steps=total, last_epoch=-1)
        out["onecycle_%d_init" % total] = np.array([opt.lr, opt.mom], np.float64)
        lr, mom = [], []
        for it in range(total + 5):
            sched.step(it)
            lr.append(opt.lr)
            mom.append(opt.mom)
            assert opt.opt.param_groups[0]["betas"] == (mom[-1], 0.99) and opt.opt.param_groups[1]["lr"] == lr[-1]
        out["onecycle_%d_lr" % total], out["onecycle_%d_mom" % total] = np.array(lr, np.float64), np.array(mom, np.float64)


def warmup(ns, cfg, out):
    """Trainer.train's lr calls for OPTIMIZER=adam with LR_WARMUP, in train_rcnn.py's construction order"""
    import tools.train_utils.train_utils as train_utils
    cfg.TRAIN.OPTIMIZER = "adam"
    model = small_module()
    ns["model"] = model
    opt = ns["create_optimizer"](model)
    lr_scheduler, _ = ns["create_scheduler"](opt, total_steps=2 * WARMUP_ITERS, last_epoch=-1)
    warm = train_utils.CosineWarmupLR(opt, T_max=cfg.TRAIN.WARMUP_EPOCH * WARMUP_ITERS, eta_min=cfg.TRAIN.WARMUP_MIN)
    lrs, epochs, its = [], [], []
    it = 0
    for epoch in range(2):
        if cfg.TRAIN.WARMUP_EPOCH <= epoch:
            lr_scheduler.step(epoch)
        for _ in range(WARMUP_ITERS):
            if epoch < cfg.TRAIN.WARMUP_EPOCH:
                warm.step(it)
            lrs.append(opt.param_groups[0]["lr"])
            epochs.append(epoch)
            its.append(it)
            it += 1
    out["warmup_lr"], out["warmup_epoch"], out["warmup_it"] = np.array(lrs, np.float64), np.array(epochs), np.array(its)
    dec = []
    for epoch in range(1, 221):
        lr_scheduler.step(epoch)
        dec.append(opt.param_groups[0]["lr"])
    out["decay_epoch"], out["decay_lr"] = np.arange(1, 221), np.array(dec, np.float64)


def bn_momentum(ns, cfg, out):
    cfg.TRAIN.OPTIMIZER = "adam_onecycle"
    model = small_module()
    ns["model"] = model
    opt = ns["create_optimizer"](model)
    _, bnm = ns["create_scheduler"](opt, total_steps=10 * BNM_ITERS, last_epoch=-1)
    its, moms = [-1], [model[1].momentum]                      # -1: after the constructor
    for epoch in range(8):
        it = epoch * BNM_ITERS
        bnm.step(it)
        its.append(it)
        moms.append(model[1].momentum)
    out["bnm_it"], out["bnm_mom"] = np.array(its), np.array(moms, np.float64)
    res = []
    for start_epoch in BNM_RESUME_EPOCHS:
        model = small_module()
        ns["model"] = model
        ns["create_scheduler"](ns["create_optimizer"](model), total_steps=10, last_epoch=start_epoch + 1)
        res.append(model[1].momentum)
    out["bnm_resume_epoch"], out["bnm_resume_mom"] = np.array(BNM_RESUME_EPOCHS), np.array(res, np.float64)


def groups(ns, cfg, out):
    from lib.net.point_rcnn import PointRCNN
    cfg.TRAIN.OPTIMIZER = "adam_onecycle"
    for mode in ("rpn", "rcnn"):
        cfg.RPN.ENABLED, cfg.RCNN.ENABLED, cfg.RPN.FIXED = True, mode == "rcnn", mode == "rcnn"
        torch.manual_seed(0)
        model = PointRCNN(num_classes=2, use_xyz=True, mode="TRAIN")
        opt = ns["create_optimizer"](model)
        name = {id(p): n for n, p in model.named_parameters()}
        assert len(opt.opt.param_groups) == 2
        for g, pg in enumerate(opt.opt.param_groups):
            out["groups_%s_%d" % (mode, g)] = np.array([name[id(p)] for p in pg["params"]])
        frozen = sorted(n for n, p in model.named_parameters() if not p.requires_grad)
        assert (mode == "rcnn") == bool(frozen) and all(n.startswith("rpn.") for n in frozen)
    cfg.RPN.ENABLED, cfg.RCNN.ENABLED, cfg.RPN.FIXED = True, False, False


def trajectory(ns, cfg, out):
    cfg.TRAIN.OPTIMIZER = "adam_onecycle"
    torch.manual_seed(3)
    model = small_module()
    ns["model"] = model
    params = list(model.parameters())
    names = [n for n, _ in model.named_parameters()]
    out["traj_names"] = np.array(names)
    for n, p in zip(names, params):
        out["traj_init_" + n] = p.detach().numpy().copy()
    opt = ns["create_optimizer"](model)
    sched, _ = ns["create_scheduler"](opt, total_steps=TRAJ_TOTAL, last_epoch=-1)
    g = torch.Generator().manual_seed(11)
    for it in range(TRAJ_STEPS):
        sched.step(it)
        for n, p in zip(names, params):
            p.grad = torch.randn(p.shape, generator=g) * 0.1
            if n == "3.bias":
                p.grad.zero_()
            out["traj_grad%d_%s" % (it, n)] = p.grad.numpy().copy()
        opt.step()
        if it + 1 in (TRAJ_SAVE, TRAJ_STEPS):
            tag = "save" if it + 1 == TRAJ_SAVE else "end"
            for n, p in zip(names, params):
                st = opt.opt.state[p]
                out["traj_%s_param_%s" % (tag, n)] = p.detach().numpy().copy()
                out["traj_%s_exp_avg_%s" % (tag, n)] = st["exp_avg"].numpy().copy()
                out["traj_%s_exp_avg_sq_%s" % (tag, n)] = st["exp_avg_sq"].numpy().copy()
        if it + 1 == TRAJ_SAVE:
            sd = opt.state_dict()
            idx = [i for pg in sd["param_groups"] for i in pg["params"]]
            out["ckpt_index"] = np.array(idx)
            out["ckpt_group_params"] = np.array([len(pg["params"]) for pg in sd["param_groups"]])
            for i in idx:
                out["ckpt_step_%d" % i] = np.array(int(sd["state"][i]["step"]))
                out["ckpt_exp_avg_%d" % i] = sd["state"][i]["exp_avg"].numpy().copy()
                out["ckpt_exp_avg_sq_%d" % i] = sd["state"][i]["exp_avg_sq"].numpy().copy()
            for key in ("lr", "eps", "weight_decay"):
                out["ckpt_group_" + key] = np.array([pg[key] for pg in sd["param_groups"]], np.float64)
            out["ckpt_group_betas"] = np.array([pg["betas"] for pg in sd["param_groups"]], np.float64)
            out["ckpt_group_amsgrad"] = np.array([pg["amsgrad"] for pg in sd["param_groups"]])
    out["traj_consts"] = np.array([TRAJ_TOTAL, TRAJ_STEPS, TRAJ_SAVE])


def main():
    from pointrcnn_b200 import dropin
    sys.path.insert(0, REF)
    sys.path.insert(0, os.path.join(REF, "lib", "net"))         # tools/_init_path.py: rpn.py imports its backbone by name
    dropin.activate(compat=True)
    collections.Iterable = collections.abc.Iterable           # fastai_optim.py: `from collections import Iterable`
    if "tqdm" not in sys.modules:
        try:
            import tqdm  # noqa: F401
        except ImportError:
            sys.modules["tqdm"] = types.ModuleType("tqdm")
    from lib.config import cfg, cfg_from_file
    cfg_from_file(os.path.join(REF, "tools/cfgs/default.yaml"))
    cfg.RPN.ENABLED, cfg.RCNN.ENABLED = True, False            # --train_mode rpn
    ns = reference_namespace(cfg)
    out = {"consts": np.array([WARMUP_ITERS, BNM_ITERS])}
    onecycle(ns, cfg, out)
    warmup(ns, cfg, out)
    bn_momentum(ns, cfg, out)
    groups(ns, cfg, out)
    trajectory(ns, cfg, out)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    main()

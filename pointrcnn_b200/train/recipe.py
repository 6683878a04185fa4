"""The reference's training recipe around the training step (tools/train_rcnn.py:88-143, tools/train_utils/*,
cfgs/default.yaml TRAIN): its learning-rate, Adam-momentum and BatchNorm-momentum schedules restated on Python floats, the
OptimWrapper + true-weight-decay Adam of OPTIMIZER=adam_onecycle, checkpoints in the reference's file layout, and the epoch
loop of train_utils.Trainer.train.

Quirks of the reference kept on purpose (tests/golden/train_recipe.npz pins each one):
  - OneCycle's phase boundary is int(PCT_START * total_step), truncated; steps at or past total_step keep extrapolating the
    last cosine.  A phase of zero steps (total_step < 3) divides by zero there; here it raises ValueError up front.
  - the parameter groups are the model's leaf modules in flatten order, split into non-BatchNorm and BatchNorm leaves, and
    hold every parameter the model had when the optimizer was built: in the RCNN phase the frozen RPN's parameters are in
    them (the reference freezes the RPN after building the optimizer), so the optimizer_state indices count them.
  - true weight decay multiplies every parameter that requires grad by (1 - WEIGHT_DECAY * lr) before Adam runs, BatchNorm
    affine parameters and parameters with an all-zero gradient included; Adam itself runs with weight_decay=0.
  - Trainer.train steps the BN-momentum schedule at each epoch start with the ITERATION count, so the momentum halves at the
    first epoch that starts at it >= 1000; a resumed run's scheduler constructor applies bn_momentum(start_epoch + 2).
  - OPTIMIZER=adam: the cosine warm-up runs per iteration during the first WARMUP_EPOCH epochs (from WARMUP_MIN to LR over
    WARMUP_EPOCH * iters_per_epoch iterations); from then on the step decay is applied once at each epoch start.
"""
import math
import os

import torch
from torch import nn

LR, LR_CLIP, LR_DECAY, DECAY_STEP_LIST = 0.002, 0.00001, 0.5, (100, 150, 180, 200)
WARMUP_MIN, WARMUP_EPOCH = 0.0002, 1
BN_MOMENTUM, BN_DECAY, BNM_CLIP, BN_DECAY_STEP_LIST = 0.1, 0.5, 0.01, (1000,)
WEIGHT_DECAY = 0.001
MOMS, DIV_FACTOR, PCT_START = (0.95, 0.85), 10.0, 0.4
BETA2 = 0.99
GRAD_NORM_CLIP = 1.0
BN_TYPES = (nn.BatchNorm1d, nn.BatchNorm2d, nn.BatchNorm3d)
OPTIMIZERS = ("adam", "adam_onecycle")


def annealing_cos(start, end, pct):
    """cosine from `start` (pct = 0) to `end` (pct = 1); pct > 1 continues the cosine"""
    return end + (start - end) / 2 * (math.cos(math.pi * pct) + 1)


class OneCycle:
    """learning_schedules_fastai.OneCycle: lr from lr_max/div_factor up to lr_max and down to lr_max/div_factor/1e4, Adam's
    beta1 from moms[0] down to moms[1] and back, both as two cosine phases split at int(pct_start * total_step)"""

    def __init__(self, total_step, lr_max=LR, moms=MOMS, div_factor=DIV_FACTOR, pct_start=PCT_START):
        mid = int(pct_start * total_step)
        if not 0 < mid < total_step:
            raise ValueError("OneCycle needs at least one step in each phase: total_step=%r splits at %d" % (total_step, mid))
        low = lr_max / div_factor
        self.total_step = total_step
        self.initial = (low, moms[0])
        self.lr_phases = ((0, mid, low, lr_max), (mid, total_step, lr_max, low / 1e4))
        self.mom_phases = ((0, mid, moms[0], moms[1]), (mid, total_step, moms[1], moms[0]))

    def __call__(self, it):
        """(lr, beta1) of iteration `it` >= 0: the last phase that has started decides"""
        lr = next(annealing_cos(a, b, (it - s) / (e - s)) for s, e, a, b in reversed(self.lr_phases) if it >= s)
        mom = next(annealing_cos(a, b, (it - s) / (e - s)) for s, e, a, b in reversed(self.mom_phases) if it >= s)
        return lr, mom


def step_decay(epoch):
    """train_rcnn.py lr_lbmd: the LambdaLR factor of `epoch` for OPTIMIZER=adam"""
    decay = 1
    for step in DECAY_STEP_LIST:
        if epoch >= step:
            decay = decay * LR_DECAY
    return max(decay, LR_CLIP / LR)


def warmup_lr(it, t_max, lr=LR):
    """train_utils.CosineWarmupLR at iteration `it`: from WARMUP_MIN (it = 0) to `lr` (it = t_max)"""
    return WARMUP_MIN + (lr - WARMUP_MIN) * (1 - math.cos(math.pi * it / t_max)) / 2


def bn_momentum(x):
    """train_rcnn.py bnm_lmbd"""
    decay = 1
    for step in BN_DECAY_STEP_LIST:
        if x >= step:
            decay = decay * BN_DECAY
    return max(BN_MOMENTUM * decay, BNM_CLIP)


def set_bn_momentum(model, momentum):
    """train_utils.set_bn_momentum_default over every BatchNorm1d/2d/3d of `model`"""
    for m in model.modules():
        if isinstance(m, BN_TYPES):
            m.momentum = momentum


def flatten_model(m):
    """the leaf modules of `m` in children() order (train_rcnn.py flatten_model)"""
    children = list(m.children())
    return sum(map(flatten_model, children), []) if children else [m]


def param_groups(model):
    """fastai_optim.split_bn_bias over get_layer_groups(model): [non-BatchNorm leaf parameters, BatchNorm leaf parameters],
    every parameter whatever its requires_grad (see the module docstring)"""
    leaves = flatten_model(model)
    return [list(nn.Sequential(*[m for m in leaves if not isinstance(m, BN_TYPES)]).parameters()),
            list(nn.Sequential(*[m for m in leaves if isinstance(m, BN_TYPES)]).parameters())]


def _fused_on_device(opt):
    """torch's Optimizer.load_state_dict takes the groups' flags from the file, and Adam falls back to fused=None when the
    file has none (a torch 1.x checkpoint); put fused back and its step counters on the parameters' device"""
    for group in opt.param_groups:
        group["fused"], group["foreach"] = True, None
        for p in group["params"]:
            st = opt.state.get(p)
            if st:
                st["step"] = st["step"].to(device=p.device, dtype=torch.float32)


class TrueWDAdam:
    """OptimWrapper.create(partial(Adam, betas=(0.9, 0.99)), lr, layer_groups, wd=wd, true_wd=True, bn_wd=True): a
    torch.optim.Adam with weight_decay=0 over `groups`, preceded in step() by the decoupled decay p *= 1 - wd * lr.  The
    schedule writes lr and beta1 into every group (set()); state_dict() is the inner Adam's, as the reference's checkpoints
    hold it.  Not AdamW: its decay lives in the groups, and a reference optimizer_state (weight_decay=0) would switch it off."""

    def __init__(self, groups, lr, mom, wd=WEIGHT_DECAY, fused=False):
        self.opt = torch.optim.Adam([{"params": g, "lr": 0} for g in groups], betas=(0.9, BETA2), **({"fused": True} if fused else {}))
        self.wd = wd
        self.set(lr, mom)

    @property
    def param_groups(self):
        return self.opt.param_groups

    def set(self, lr, mom):
        for group in self.opt.param_groups:
            group["lr"], group["betas"] = lr, (mom, group["betas"][1])

    @torch.no_grad()
    def step(self):
        for group in self.opt.param_groups:
            ps = [p for p in group["params"] if p.requires_grad]
            if ps:
                torch._foreach_mul_(ps, 1 - self.wd * group["lr"])
        self.opt.step()

    def zero_grad(self, set_to_none=True):
        self.opt.zero_grad(set_to_none)

    def state_dict(self):
        return self.opt.state_dict()

    def load_state_dict(self, state_dict):
        self.opt.load_state_dict(state_dict)


def _load(path):
    """a checkpoint file.  The reference's hold numpy float64 learning rates and betas (OneCycle computes them with np.cos);
    numpy 1.x, which wrote them, names the scalar constructor numpy.core.multiarray.scalar, numpy 2 numpy._core...  Both
    names are allowed, and the dtype classes either version pickles."""
    import numpy as np
    scalar = np._core.multiarray.scalar
    scalars = [scalar, (scalar, "numpy.core.multiarray.scalar"), np.dtype, type(np.dtype(np.float64))]
    with torch.serialization.safe_globals(scalars):
        return torch.load(path, map_location="cpu", weights_only=True)


def save_checkpoint(trainer, path, epoch, it):
    """train_utils.checkpoint_state + save_checkpoint: {'epoch', 'it', 'model_state', 'optimizer_state'}, the model state in
    the PointRCNN layout (rpn.*, rcnn_net.*)"""
    torch.save({"epoch": epoch, "it": it, "model_state": trainer.net.state_dict(), "optimizer_state": trainer.opt.state_dict()}, path)


def load_checkpoint(trainer, path):
    """train_utils.load_checkpoint for a file this module wrote, or one the reference wrote with the same optimizer layout
    (adam_onecycle; the trainers' "adam" keeps one group over the trained stage only) -> (it, epoch).  Restores the model
    and the optimizer, sets the schedule to iteration `it` and the BN momentum as the reference's resumed scheduler does"""
    ckpt = _load(path)
    epoch = ckpt.get("epoch", -1)
    it = ckpt.get("it", 0)
    trainer.net.load_state_dict(ckpt["model_state"])
    trainer.opt.load_state_dict(ckpt["optimizer_state"])
    if trainer.device.type == "cuda":
        _fused_on_device(getattr(trainer.opt, "opt", trainer.opt))
    trainer.resume_schedule(it, epoch)
    return it, epoch


def load_part(model, path):
    """train_utils.load_part_ckpt (--rpn_ckpt): load the checkpoint's model_state keys that `model` has, keep the rest of
    `model` as it is; raises when no key matches.  -> the number of keys loaded"""
    state = _load(path)["model_state"]
    own = model.state_dict()
    found = {k: v for k, v in state.items() if k in own}
    if not found:
        raise RuntimeError("no key of %s's model_state is in the model" % path)
    own.update(found)
    model.load_state_dict(own)
    return len(found)


def fit(trainer, batches_per_epoch, epochs, start_it=0, start_epoch=0, ckpt_dir=None, ckpt_every=5):
    """train_utils.Trainer.train without logging or validation: epochs start_epoch .. epochs-1, BN momentum and (adam) the
    step decay at each epoch start, the per-iteration schedule, trainer.step(*batch, grad_norm_clip=GRAD_NORM_CLIP), and
    checkpoint_epoch_<n>.pth in ckpt_dir after every ckpt_every-th epoch.  batches_per_epoch: a re-iterable of argument
    tuples of trainer.step with a len() (a DataLoader).  The reference reads loss.item() every iteration; here each epoch's
    loss and loss terms stay on the device and reach the host in one copy at the epoch's end.
    -> one dict per epoch: {'loss': (iters,) array, term name: (iters,) array}.  Row k of every array is iteration k of
    the epoch; a term an iteration did not return (the torch loss path has no regression terms without a foreground
    point) is NaN there."""
    it = start_it
    history = []
    for epoch in range(start_epoch, epochs):
        trainer.schedule_epoch(epoch, it)
        steps = []
        for batch in batches_per_epoch:
            trainer.schedule_iteration(it, epoch, len(batches_per_epoch))
            steps.append(trainer.step(*batch, grad_norm_clip=GRAD_NORM_CLIP))
            it += 1
        keys = list(dict.fromkeys(k for _, terms in steps for k in terms))
        nan = torch.full((), float("nan"), device=trainer.device)
        rows = [[loss] + [terms.get(k, nan) for k in keys] for loss, terms in steps]
        flat = torch.stack([torch.as_tensor(v, device=trainer.device).detach().float().reshape(()) for row in rows for v in row])
        table = flat.cpu().numpy().reshape(len(steps), 1 + len(keys))
        history.append({k: table[:, j] for j, k in enumerate(["loss"] + keys)})
        trained = epoch + 1
        if ckpt_dir is not None and trained % ckpt_every == 0:
            save_checkpoint(trainer, os.path.join(ckpt_dir, "checkpoint_epoch_%d.pth" % trained), trained, it)
    return history

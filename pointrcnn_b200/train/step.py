"""One RPN training step on the H100 path (BASELINE configs[2]; reference: tools/train_rcnn.py:199-233 +
lib/net/train_functions.py:12-52): forward in training mode (batch-statistics BatchNorm, Dropout), bin-based loss,
backward, gradient all-reduce over the data-parallel ranks, optimizer step.

Forward / backward use the reference-shaped op-by-op path of the mirror modules: this repo's sampling / neighbour / grouping
/ interpolation natives with their scatter backward kernels (gather_points_grad, group_points_grad,
three_interpolate_grad), the shared MLPs through cuDNN / cuBLAS with torch autograd.  (The fused tensor-core chain is an
eval-mode kernel: batch-statistics BatchNorm couples all tiles of a launch.  sa_train="device" runs the SA modules it
supports through csrc/sa_train.cu instead, see pointnet2/sa_train.py.)  What this module adds over the reference's
loop: no `.item()` inside the loss, per-rank processes instead of nn.DataParallel's per-step replicate / scatter / gather,
and the bucketed all-reduce of `parallel_utils.GradBucketReducer` overlapped with backward.

CUDA graphs (cuda_graph=True, both trainers' step()): the first call runs eager (it creates the optimizer state and warms
cuDNN and the allocator), the next captures the whole step -- forward, loss, backward, the bucketed all-reduce, gradient
clipping and the optimizer step -- into a torch.cuda.CUDAGraph and replays it once, and later calls copy their inputs
into the graph's static buffers and replay it.  One graph per key of what a replay cannot change (input shapes and
dtypes, grad_norm_clip, the autocast state and dtype, torch's deterministic flag, the BatchNorm momenta, the config
switches), so a new key captures again.  The returned loss and terms are fresh tensors, not the graph's outputs.  The
schedule reaches replays through device tensors (lr, and beta1 of "adam_onecycle"), the RCNN target layer through a
device seed counter; after a replay the trained modules' fused eval caches are dropped.  Loading a checkpoint
(recipe.load_checkpoint, load_part) drops the graphs: the next step runs eager again and the one after captures.  A step
that cannot be captured (torch loss path, torch target draw, autocast with its weight-cast cache, a CPU device) raises
ValueError before anything is captured (INTEGRATION.md, "Training steps as CUDA graphs").

Mixed precision: call a trainer's step inside `with torch.autocast("cuda", dtype=torch.bfloat16):`.  The forward's
convolutions then run with bfloat16 operands, the grouping / gather / interpolation natives move bfloat16 features, the
device SA / FP / loss paths and both losses compute in fp32; backward, the all-reduce and the optimizer step run with
autocast disabled, and parameters, gradients and optimizer state stay fp32 (INTEGRATION.md, "Training under autocast").
"""
import contextlib

import numpy as np
import torch
from torch import nn

from .. import config
from ..parallel_utils import GradBucketReducer
from ..rpn.stage import CLS_MEAN_SIZE, RPNStage
from . import recipe
from .losses import rcnn_loss, rpn_loss


def _sa_switch(sa_train, fp_train=None):
    """the config.sa_train / config.fp_train override of a trainer's forward (None: leave that switch as it is)"""
    kw = {}
    for name, value in (("sa_train", sa_train), ("fp_train", fp_train)):
        if value is None:
            continue
        if value not in ("torch", "device"):
            raise ValueError("%s must be 'torch', 'device' or None, not %r" % (name, value))
        kw[name] = value
    return config.override(**kw) if kw else contextlib.nullcontext()


def _without_autocast():
    """the backward / all-reduce / optimizer part of a step: with CUDA autocast disabled when the caller enabled it"""
    return torch.autocast("cuda", enabled=False) if torch.is_autocast_enabled("cuda") else contextlib.nullcontext()


def _resolved(value, switch):
    return value or config.get(switch)


def _graph_refusal(device, loss_impl, target_draw=False):
    """why a cuda_graph=True trainer cannot capture its step (None: it can); target_draw False: no target layer.  The
    trainers check the values they were given at construction, and the resolved ones (a switch left to None follows the
    config) at every step, before anything is captured"""
    if device.type != "cuda":
        return "cuda_graph=True needs a CUDA device, not %s" % device
    if _resolved(loss_impl, "loss_impl") != "device":
        return "cuda_graph=True needs loss_impl='device': the torch loss path reads boolean masks on the host"
    if target_draw is not False and _resolved(target_draw, "target_draw") != "device":
        return "cuda_graph=True needs target_draw='device': the torch target layer reads its samples on the host"
    if torch.is_autocast_enabled("cuda") and torch.is_autocast_cache_enabled():
        return ("cuda_graph=True under autocast needs torch.autocast(..., cache_enabled=False): a cached weight cast "
                "cannot be captured")
    return None


def _schedule(optimizer, total_steps, lr):
    """the per-iteration schedule of a trainer's `optimizer` switch (None for "adam", whose schedule is per epoch); raises
    ValueError for an unknown name or "adam_onecycle" without total_steps"""
    if optimizer not in recipe.OPTIMIZERS:
        raise ValueError("optimizer must be one of %s, not %r" % (", ".join(map(repr, recipe.OPTIMIZERS)), optimizer))
    if optimizer == "adam":
        return None
    if total_steps is None:
        raise ValueError("optimizer='adam_onecycle' needs total_steps (iterations per epoch * epochs)")
    return recipe.OneCycle(total_steps, lr_max=lr)


class _PointRCNNLayout(nn.Module):
    """the reference's PointRCNN module tree over a trainer's stages: state-dict keys rpn.* (and rcnn_net.*), leaf modules in
    the order the reference's parameter groups take them"""

    def __init__(self, rpn, rcnn_net=None):
        super().__init__()
        self.rpn = rpn
        if rcnn_net is not None:
            self.rcnn_net = rcnn_net


class _Recipe:
    """the optimizer switch and the schedule hooks of both trainers (see train.recipe).  optimizer="adam": torch Adam with
    L2 weight decay over the trainable parameters (cfgs OPTIMIZER: adam); its warm-up and step decay apply only through
    the hooks.  "adam_onecycle": recipe.TrueWDAdam over the PointRCNN-layout groups with the OneCycle schedule of
    total_steps iterations (the reference's default recipe)"""

    def _build_optimizer(self, schedule, lr, weight_decay):
        self.schedule, self.lr = schedule, lr
        fused = self.device.type == "cuda"
        if schedule is None:
            self.opt = torch.optim.Adam(self.params, lr=lr, weight_decay=weight_decay, **({"fused": True} if fused else {}))
            if self._graph_mode():
                self._lr_tensor = torch.full((1,), lr, dtype=torch.float32, device=self.device)
                self._graph_groups()
                self.opt.register_load_state_dict_post_hook(lambda opt: self._graph_groups(reload=True))
        else:
            self.opt = recipe.TrueWDAdam(recipe.param_groups(self.net), *schedule.initial, wd=weight_decay, fused=fused,
                                         graph=self._graph_mode())

    def _graph_mode(self):
        return getattr(self, "cuda_graph", False)

    def _graph_groups(self, reload=False):
        """cuda_graph with optimizer="adam": torch's fused Adam reading lr from a float32 CUDA tensor (capturable, as torch
        requires for capture).  reload: after load_state_dict, which puts the file's float lr and flags in the groups"""
        for group in self.opt.param_groups:
            if reload:
                self._lr_tensor.fill_(float(group["lr"]))
            group["lr"], group["capturable"] = self._lr_tensor, True

    def _set_lr(self, lr):
        if self._graph_mode():
            self._lr_tensor.fill_(lr)
            return
        for group in self.opt.param_groups:
            group["lr"] = lr

    def _init_graphs(self, cuda_graph):
        self.cuda_graph = bool(cuda_graph)
        self._graphs = {}
        self._warm = False
        self._stream = None
        if self.cuda_graph:
            self.net.register_load_state_dict_post_hook(lambda module, keys: self.drop_graphs())

    def drop_graphs(self):
        """forget every captured step: the next step() runs eager again (it rebuilds what the load replaced: optimizer
        state, packed eval weights) and the one after captures.  Loading a state dict into self.net does this"""
        self._graphs.clear()
        self._warm = False

    def graph_key(self, inputs, grad_norm_clip):
        """everything a replay of the captured step cannot change: input shapes and dtypes, the clip, the CUDA autocast
        state and dtype, torch's deterministic flag (and warn_only), the BatchNorm momenta that cuDNN and the device
        SA / FP kernels take as host values, and the config switches the step reads while it is traced (a switch the
        trainer was given counts with its own value)"""
        autocast = (torch.is_autocast_enabled("cuda"), torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else None)
        momenta = tuple(m.momentum for m in self.model.modules() if isinstance(m, recipe.BN_TYPES))
        own = {k: getattr(self, k, None) for k in ("sa_train", "fp_train", "loss_impl", "target_draw")}
        switches = tuple((k, own.get(k) or config.get(k)) for k in config.names())
        return (tuple((tuple(t.shape), t.dtype) for t in inputs), grad_norm_clip, autocast,
                torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(), momenta,
                switches)

    def _run_step(self, forward_loss, args, grad_norm_clip):
        self.reducer.reset()
        loss, terms = forward_loss(*args)
        with _without_autocast():
            loss.backward()
            self.reducer.finish()
            if grad_norm_clip:
                torch.nn.utils.clip_grad_norm_(self.params, grad_norm_clip)     # train_utils.py: clip_grad_norm_(.., GRAD_NORM_CLIP)
            self.opt.step()
        return loss.detach(), terms

    def _graphed_step(self, forward_loss, inputs, grad_norm_clip):
        """one step of a cuda_graph trainer: eager on the first call, then capture (once per graph_key) and replay"""
        refusal = _graph_refusal(self.device, self.loss_impl, getattr(self, "target_draw", False))
        if refusal:
            raise ValueError(refusal)
        if not self._warm:
            # on the capture stream: autograd keeps each parameter's gradient accumulator, with the stream it was created
            # on, for as long as anything holds this step's graph, and a capture may not join work on another stream
            self._warm = True
            if self._stream is None:
                self._stream = torch.cuda.Stream(self.device)
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self._stream):
                loss, terms = self._run_step(forward_loss, inputs, grad_norm_clip)
            torch.cuda.current_stream(self.device).wait_stream(self._stream)
            return loss, {k: v.detach() for k, v in terms.items()}
        key = self.graph_key(inputs, grad_norm_clip)
        entry = self._graphs.get(key)
        if entry is None:
            static = tuple(t.detach().clone() for t in inputs)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=self._stream):
                loss, terms = self._run_step(forward_loss, static, grad_norm_clip)
            entry = self._graphs[key] = (graph, static, (loss, {k: v.detach() for k, v in terms.items()}))
        graph, static, (loss, terms) = entry
        for dst, src in zip(static, inputs):
            dst.copy_(src, non_blocking=True)
        graph.replay()
        self.model.invalidate_fused()             # replays change parameters and BN buffers without bumping their versions
        return loss.clone(), {k: v.clone() for k, v in terms.items()}

    def schedule_epoch(self, epoch, it):
        """the start of `epoch`, `it` iterations into the run (Trainer.train): the BN momentum of `it` (the reference passes
        the iteration count, not the epoch) and, for "adam" once the warm-up is over, the step decay of `epoch`"""
        recipe.set_bn_momentum(self.net, recipe.bn_momentum(it))
        if self.schedule is None and epoch >= recipe.WARMUP_EPOCH:
            self._set_lr(self.lr * recipe.step_decay(epoch))

    def schedule_iteration(self, it, epoch, iters_per_epoch):
        """before the step of iteration `it`: OneCycle's lr and beta1, or for "adam" in the first WARMUP_EPOCH epochs the
        cosine warm-up over WARMUP_EPOCH * iters_per_epoch iterations"""
        if self.schedule is not None:
            self.opt.set(*self.schedule(it))
        elif epoch < recipe.WARMUP_EPOCH:
            self._set_lr(recipe.warmup_lr(it, recipe.WARMUP_EPOCH * iters_per_epoch, self.lr))

    def resume_schedule(self, it, epoch):
        """after loading a checkpoint of iteration `it`, epoch `epoch`: the BN momentum the reference's resumed scheduler
        constructor sets (last_epoch = epoch + 1, applied as epoch + 2) and OneCycle's values at `it`"""
        recipe.set_bn_momentum(self.net, recipe.bn_momentum(epoch + 2))
        if self.schedule is not None:
            self.opt.set(*self.schedule(it))


class RPNTrainer(_Recipe):
    """loss_impl: which stage-loss path forward_loss takes ("torch" / "device", see train.losses; None: the config switch).
    sa_train: which path the SA modules take in training ("torch" / "device", see pointnet2/sa_train.py; None: the config
    switch).  fp_train: the same for the FP modules (see pointnet2/fp_train.py).  optimizer / total_steps: see _Recipe;
    self.net is the model in the PointRCNN layout (rpn.*) that checkpoints hold.  cuda_graph: replay step() as a CUDA
    graph (see the module docstring; needs loss_impl="device")"""

    def __init__(self, input_channels=1, device="cuda", world=1, lr=0.002, weight_decay=0.001, bucket_mb=4.0, seed=0, loss_impl=None,
                 sa_train=None, fp_train=None, optimizer="adam", total_steps=None, cuda_graph=False):
        schedule = _schedule(optimizer, total_steps, lr)
        if cuda_graph:
            refusal = _graph_refusal(torch.device(device), loss_impl or "device", False)
            if refusal:
                raise ValueError(refusal)
        self.cuda_graph = bool(cuda_graph)
        torch.manual_seed(seed)                       # identical initial weights on every rank
        self.device = torch.device(device)
        self.model = RPNStage(input_channels=input_channels, mode="TRAIN").to(self.device).train()
        self.net = _PointRCNNLayout(self.model)
        self.params = [p for p in self.model.parameters() if p.requires_grad]
        self.reducer = GradBucketReducer(self.params, world=world, bucket_mb=bucket_mb)
        self._build_optimizer(schedule, lr, weight_decay)
        self.mean_size = torch.from_numpy(CLS_MEAN_SIZE[0]).to(self.device)
        self.loss_impl = loss_impl
        self.sa_train = sa_train
        self.fp_train = fp_train
        _sa_switch(sa_train, fp_train)
        self._init_graphs(cuda_graph)

    def forward_loss(self, pts_input, rpn_cls_label, rpn_reg_label):
        m = self.model
        with _sa_switch(self.sa_train, self.fp_train):
            xyz, feats = m.backbone_net(pts_input)
        rpn_cls = m.rpn_cls_layer(feats).transpose(1, 2).contiguous()       # lib/net/rpn.py:76-77
        rpn_reg = m.rpn_reg_layer(feats).transpose(1, 2).contiguous()
        return rpn_loss(rpn_cls, rpn_reg, rpn_cls_label, rpn_reg_label, self.mean_size, impl=self.loss_impl)

    def step(self, pts_input, rpn_cls_label, rpn_reg_label, grad_norm_clip=None):
        """one training step -> (loss, loss terms); with cuda_graph a captured replay after the first call"""
        inputs = (pts_input, rpn_cls_label, rpn_reg_label)
        if self.cuda_graph:
            return self._graphed_step(self.forward_loss, inputs, grad_norm_clip)
        return self._run_step(self.forward_loss, inputs, grad_norm_clip)


def synthetic_labels(pts_input, seed=0):
    """RPN labels of the right shapes / statistics for synthetic scenes (kitti_rcnn_dataset.py:generate_rpn_training_labels
    shapes): ~3 % foreground points, regression targets = offsets to a nearby box centre + size + heading"""
    B, N = pts_input.shape[0], pts_input.shape[1]
    g = torch.Generator().manual_seed(seed)
    cls = (torch.rand(B, N, generator=g) < 0.03).long()
    cls[torch.rand(B, N, generator=g) < 0.01] = -1
    reg = torch.zeros(B, N, 7)
    reg[..., 0:3] = torch.randn(B, N, 3, generator=g) * torch.tensor([1.0, 0.3, 1.0])
    reg[..., 3:6] = torch.from_numpy(CLS_MEAN_SIZE[0]) * (1 + 0.1 * torch.randn(B, N, 3, generator=g))
    reg[..., 6] = (torch.rand(B, N, generator=g) * 2 - 1) * float(np.pi)
    return cls.to(pts_input.device), reg.to(pts_input.device)


class RCNNTrainer(_Recipe):
    """One RCNN training step with the RPN fixed (the reference's second training phase: tools/train_rcnn.py --train_mode rcnn,
    cfg.RPN.FIXED): the RPN stage runs in eval mode without grad on the fused path and hands (rois, point features, mask,
    depth) to the RCNN stage, whose target layer samples 64 RoIs per scene; forward / backward of the RCNN network on the
    op-by-op path, get_rcnn_loss, bucketed gradient all-reduce, optimizer step.  target_draw: how the target layer samples
    ("torch": the reference's random calls, "device": one device pass without host reads; None: the config switch).  loss_impl:
    which stage-loss path every forward_loss* method takes ("torch" / "device", see train.losses; None: the config switch).
    sa_train: which path the RCNN network's SA modules take ("torch" / "device", see pointnet2/sa_train.py; None: the config
    switch).  optimizer / total_steps: see _Recipe; self.net is the PointRCNN layout (rpn.*, rcnn_net.*) that checkpoints
    hold, and recipe.load_part(self.net, path) loads a phase-1 checkpoint's RPN (--rpn_ckpt).  gt_rows: a GT capacity;
    step() pads gt_boxes3d to that many rows with zero rows (the target layer trims them as padding, so nothing changes)
    and raises ValueError for a batch with more.  cuda_graph: replay step() as a CUDA graph (see the module docstring;
    needs loss_impl="device" and target_draw="device"); step_jit and step_offline, whose point and RoI counts vary per
    batch, still run eager."""

    def __init__(self, input_channels=1, device="cuda", world=1, lr=0.002, weight_decay=0.001, bucket_mb=4.0, seed=0, rpn_score_thresh=0.3,
                 target_draw=None, loss_impl=None, sa_train=None, optimizer="adam", total_steps=None, gt_rows=None, cuda_graph=False):
        from ..rcnn.stage import RCNNStage
        from ..rpn.proposal_target_layer import ProposalTargetLayer
        schedule = _schedule(optimizer, total_steps, lr)
        if cuda_graph:
            refusal = _graph_refusal(torch.device(device), loss_impl or "device", target_draw or "device")
            if refusal:
                raise ValueError(refusal)
        self.cuda_graph = bool(cuda_graph)
        torch.manual_seed(seed)
        self.device = torch.device(device)
        self.rpn = RPNStage(input_channels=input_channels, mode="TRAIN").to(self.device).eval()     # TRAIN quotas: 512 RoIs per scene
        for p in self.rpn.parameters():
            p.requires_grad_(False)
        self.model = RCNNStage(num_classes=2, input_channels=128).to(self.device).train()
        self.net = _PointRCNNLayout(self.rpn, self.model)
        self.params = [p for p in self.model.parameters() if p.requires_grad]
        self.reducer = GradBucketReducer(self.params, world=world, bucket_mb=bucket_mb)
        self._build_optimizer(schedule, lr, weight_decay)
        self.mean_size = torch.from_numpy(CLS_MEAN_SIZE[0]).to(self.device)
        self.rpn_score_thresh = rpn_score_thresh
        self.target_draw = target_draw
        self.loss_impl = loss_impl
        self.sa_train = sa_train
        self.gt_rows = gt_rows
        _sa_switch(sa_train)
        self._init_graphs(cuda_graph)
        if self.cuda_graph:
            self.model.proposal_target_layer = ProposalTargetLayer()
            self.model.proposal_target_layer.use_device_seed(self.device)

    @torch.no_grad()
    def rpn_outputs(self, pts_input, gt_boxes3d):
        rois, _, rpn_cls, _, xyz, feats = self.rpn(pts_input, with_features=True)       # point_rcnn.py:36-55
        seg_mask = (torch.sigmoid(rpn_cls[:, :, 0]) > self.rpn_score_thresh).float()
        return {"rpn_xyz": xyz, "rpn_features": feats.permute(0, 2, 1).contiguous(), "seg_mask": seg_mask, "roi_boxes3d": rois,
                "pts_depth": torch.norm(xyz, p=2, dim=2), "gt_boxes3d": gt_boxes3d}

    def forward_loss(self, pts_input, gt_boxes3d):
        return self.forward_loss_jit(self.rpn_outputs(pts_input, gt_boxes3d))

    def forward_loss_jit(self, batch):
        """rcnn_net.forward with ROI_SAMPLE_JIT (:120-126) + get_rcnn_loss on an input dict: the RPN outputs of forward_loss, or
        a batch of saved features and proposals from datasets.rcnn_offline.RCNNOfflineSampler.prepare_jit_batch"""
        with _sa_switch(self.sa_train):
            ret = self.model.forward_train(batch, target_draw=self.target_draw)
        c = self.model.cfg
        return rcnn_loss(ret["rcnn_cls"], ret["rcnn_reg"], ret["cls_label"], ret["reg_valid_mask"], ret["roi_boxes3d"], ret["gt_of_rois"],
                         self.mean_size, loc_scope=c["LOC_SCOPE"], loc_bin_size=c["LOC_BIN_SIZE"], num_head_bin=c["NUM_HEAD_BIN"],
                         loc_y_by_bin=c["LOC_Y_BY_BIN"], loc_y_scope=c["LOC_Y_SCOPE"], loc_y_bin_size=c["LOC_Y_BIN_SIZE"],
                         impl=self.loss_impl)

    def forward_loss_offline(self, batch):
        """the ROI_SAMPLE_JIT=False branch of rcnn_net.forward (:155-163) + get_rcnn_loss on a batch of
        datasets.rcnn_offline.RCNNOfflineSampler.prepare_batch: the network reads the pooled rows as they are (no
        torch.cat of pts_input and pts_features), the targets are the batch's labels and canonical GT boxes"""
        with _sa_switch(self.sa_train):
            rcnn_cls, rcnn_reg = self.model.forward_pts(batch["rows"])
        c = self.model.cfg
        return rcnn_loss(rcnn_cls, rcnn_reg, batch["cls_label"], batch["reg_valid_mask"], batch["roi_boxes3d"], batch["gt_boxes3d_ct"],
                         self.mean_size, loc_scope=c["LOC_SCOPE"], loc_bin_size=c["LOC_BIN_SIZE"], num_head_bin=c["NUM_HEAD_BIN"],
                         loc_y_by_bin=c["LOC_Y_BY_BIN"], loc_y_scope=c["LOC_Y_SCOPE"], loc_y_bin_size=c["LOC_Y_BIN_SIZE"],
                         impl=self.loss_impl)

    def step_offline(self, batch, grad_norm_clip=None):
        """one offline-recipe training step (tools/train_rcnn.py --train_mode rcnn_offline) on a prepared batch; eager also
        with cuda_graph (the RoI count varies per batch)"""
        return self._run_step(self.forward_loss_offline, (batch,), grad_norm_clip)

    def step_jit(self, batch, grad_norm_clip=None):
        """one training step of tools/train_rcnn.py --train_mode rcnn_offline with ROI_SAMPLE_JIT (the target layer inside
        the network) on a prepare_jit_batch batch; eager also with cuda_graph (the point and RoI counts vary per batch)"""
        return self._run_step(self.forward_loss_jit, (batch,), grad_norm_clip)

    def step(self, pts_input, gt_boxes3d, grad_norm_clip=None):
        """one online training step with the RPN fixed -> (loss, loss terms); with cuda_graph a captured replay after the
        first call"""
        if self.gt_rows is not None:
            B, G = gt_boxes3d.shape[0], gt_boxes3d.shape[1]
            if G > self.gt_rows:
                raise ValueError("a batch with %d GT rows exceeds gt_rows=%d" % (G, self.gt_rows))
            if G < self.gt_rows:
                gt_boxes3d = torch.cat([gt_boxes3d, gt_boxes3d.new_zeros((B, self.gt_rows - G) + tuple(gt_boxes3d.shape[2:]))], dim=1)
        inputs = (pts_input, gt_boxes3d)
        if self.cuda_graph:
            return self._graphed_step(self.forward_loss, inputs, grad_norm_clip)
        return self._run_step(self.forward_loss, inputs, grad_norm_clip)

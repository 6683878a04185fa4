"""Scene-level data parallelism helpers (SURVEY.md 8e): scenes are independent, so the forward path shards
the batch across ranks with NO data-path collective; training adds one all-reduce over gradients."""
import torch
import torch.distributed as dist


def shard_scenes(num_scenes, rank, world):
    """contiguous [lo, hi) slice of the scene list owned by `rank` (first ranks take the remainder)"""
    base, rem = divmod(num_scenes, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def max_over_ranks(value, device="cuda"):
    """MAX all-reduce of a python float (timings are reported as the max over ranks)"""
    if not (dist.is_available() and dist.is_initialized()):
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def allreduce_grads(params, world):
    """one flat all-reduce(sum)/world over the gradients (~12 MB fp32 for the RPN): latency-bound on NVSwitch"""
    grads = [p.grad for p in params if p.grad is not None]
    if not grads or world == 1 or not dist.is_initialized():
        return
    flat = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    flat.div_(world)
    off = 0
    for g in grads:
        g.copy_(flat[off:off + g.numel()].view_as(g))
        off += g.numel()


class GradBucketReducer:
    """Bucketed gradient all-reduce overlapped with backward (replaces `nn.DataParallel`'s gather/scatter + serial reduce of
    tools/train_rcnn.py:199 for one-process-per-GPU data parallelism; SURVEY.md 8(e)).

    Parameters are packed -- in REVERSE registration order, the order backward produces their gradients -- into flat fp32
    buckets of ~`bucket_mb` MB; every `p.grad` is a VIEW into its bucket, so autograd accumulates straight into the
    communication buffer (no pack / unpack copies).  A post-accumulate hook per parameter counts arrivals; when a bucket
    is complete its all-reduce is enqueued on a side stream behind an event of the compute stream, so the reduction of
    the heads' gradients runs over NVLink while backward is still working through the backbone.  `finish()` makes the
    compute stream wait for the side stream (the averaged gradients are then in place for the optimizer step).
    Over NVSwitch a 12 MB reduction is latency-bound (tens of microseconds): bucket count trades launch latency against
    overlap, 4 MB buckets give 3-4 collectives per RPN step.  Works on CPU / gloo as well (no streams: collectives run
    inline) for the world-size-2 tests.

    Under CUDA-graph capture (the trainers' cuda_graph=True) the side stream is the fork / join capture needs: reset()'s
    zeroing of the buckets, the event waits and the collectives the hooks enqueue are captured with the step, and a replay
    re-runs exactly those; the hooks and their Python bookkeeping run only while capturing."""

    def __init__(self, params, world=None, bucket_mb=4.0, process_group=None):
        self.params = [p for p in params if p.requires_grad]
        self.group = process_group
        self.world = world if world is not None else (dist.get_world_size(process_group) if dist.is_initialized() else 1)
        self.device = self.params[0].device if self.params else torch.device("cpu")
        self.cuda = self.device.type == "cuda"
        self.comm_stream = torch.cuda.Stream(self.device) if self.cuda else None
        cap = max(1, int(bucket_mb * 1024 * 1024 // 4))
        self.buckets = []                 # each: dict(flat=tensor, params=[...], pending=int, work=handle)
        cur, size = [], 0
        for p in reversed(self.params):
            if cur and size + p.numel() > cap:
                self._close(cur)
                cur, size = [], 0
            cur.append(p)
            size += p.numel()
        if cur:
            self._close(cur)
        self._owner = {}
        for bi, b in enumerate(self.buckets):
            for p in b["params"]:
                self._owner[p] = bi
        self._handles = [p.register_post_accumulate_grad_hook(self._hook) for p in self.params]
        self.bytes_per_step = sum(b["flat"].numel() for b in self.buckets) * 4
        self.reset()

    def _close(self, plist):
        flat = torch.zeros(sum(p.numel() for p in plist), dtype=torch.float32, device=self.device)
        off = 0
        for p in plist:
            p.grad = flat[off:off + p.numel()].view_as(p)       # the gradient lives inside the bucket
            off += p.numel()
        self.buckets.append(dict(flat=flat, params=plist, pending=len(plist), work=None, ready=None))

    def reset(self):
        """call before each backward (instead of optimizer.zero_grad(): grads must stay views of the buckets)"""
        for b in self.buckets:
            b["flat"].zero_()
            b["pending"] = len(b["params"])
            b["work"] = None

    def _hook(self, p):
        b = self.buckets[self._owner[p]]
        b["pending"] -= 1
        if b["pending"] == 0:
            self._launch(b)

    def _launch(self, b):
        if self.world == 1 or not dist.is_initialized():
            return
        if self.cuda:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self.comm_stream):
                self.comm_stream.wait_event(ev)
                dist.all_reduce(b["flat"], op=dist.ReduceOp.SUM, group=self.group)
                b["flat"].div_(self.world)
            b["work"] = True
        else:
            dist.all_reduce(b["flat"], op=dist.ReduceOp.SUM, group=self.group)
            b["flat"].div_(self.world)
            b["work"] = True

    def finish(self):
        """after backward: reduce any bucket whose parameters got no gradient this step, then join the side stream"""
        for b in self.buckets:
            if b["work"] is None:
                self._launch(b)
        if self.cuda and self.world > 1:
            torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)

    def remove(self):
        for h in self._handles:
            h.remove()

"""Batch pipelining: consecutive, independent batches on alternating CUDA streams, optionally as CUDA graphs.

Furthest-point sampling is a dependency chain (4095 serial rounds for the first RPN level) that runs as one CTA per
scene (16 of 132 SMs), and nothing else of the SAME batch can run before it ends.  Consecutive batches are
independent (the reference's eval loop processes them one after another), so batch i+1's sampling chain can
overlap batch i's neighbour searches and tensor-core MLPs.  Results are identical to the sequential loop, bit for bit -- only the stream assignment
differs (tests/test_gpu_mlp.py::test_batch_pipeline_matches_sequential; at bench.py's batch, slot counts and RPN
stage in tests/test_gpu_bench_paths.py).

`graphs=True` captures `fn` once per slot (stream) into a CUDA graph and replays it: the ~45 native launches and the
torch glue of one forward become one graph launch, which matters when batches are small (strong scaling: 2 scenes per
GPU) and the host cannot issue launches as fast as the GPU retires them.  Requirements: `fn` must be capturable (no
host synchronisation, no data-dependent shapes: true for the eval-mode backbone / RPN stage), the batch shape must stay
fixed per pipeline, and the weights must not change between replays (the packed weight pointers are baked into the
graph; build a new pipeline after an optimizer step / load_state_dict).
"""
import torch


class _Slot:
    __slots__ = ("stream", "graph", "static_in", "static_out", "host", "done", "pending")

    def __init__(self, stream):
        self.stream = stream
        self.graph = self.static_in = self.static_out = self.host = None
        self.done = None          # event: the slot's last batch (incl. its D2H copies) has finished
        self.pending = None       # (batch index, host result) not yet handed to the consumer


class BatchPipeline:
    def __init__(self, fn, inflight=6, device=None, graphs=False):
        """fn: callable(batch_on_device) -> tensor or tuple of tensors; inflight: batches in flight (one stream and one
        set of result buffers per slot); graphs: replay fn as a CUDA graph per slot."""
        self.fn = fn
        self.device = torch.device(device if device is not None else "cuda", torch.cuda.current_device()) \
            if not isinstance(device, torch.device) else device
        self.slots = [_Slot(torch.cuda.Stream(self.device)) for _ in range(max(1, int(inflight)))]
        self.graphs = bool(graphs)

    @property
    def streams(self):
        return [s.stream for s in self.slots]

    # ------------------------------------------------------------------ one batch on one slot
    def _forward(self, slot, x):
        """run fn on x (already on the slot's stream); returns the output tuple."""
        if not self.graphs:
            out = self.fn(x)
            return out if isinstance(out, (tuple, list)) else (out,)
        if slot.graph is None or slot.static_in.shape != x.shape or slot.static_in.dtype != x.dtype:
            slot.static_in = torch.empty_like(x)
            slot.static_in.copy_(x, non_blocking=True)
            out = self.fn(slot.static_in)                 # warm-up outside capture: weight images, lazy inits
            del out
            slot.stream.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=slot.stream):
                out = self.fn(slot.static_in)
            slot.graph = g
            slot.static_out = tuple(out) if isinstance(out, (tuple, list)) else (out,)
        slot.static_in.copy_(x, non_blocking=True)
        slot.graph.replay()
        return slot.static_out

    def run(self, batches, to_host=False, keep=True, consume=None):
        """batches: iterable of tensors (device, or pinned host -> copied inside the pipeline, on the slot's stream).
        to_host=False: returns the device results (keep=False: drops every result once its work is queued, so the
            caching allocator recycles the output blocks; with graphs the results live in the slot's static buffers and
            are cloned when kept).
        to_host=True: every result is copied to a pinned buffer OWNED BY THE SLOT.  With `consume(i, result)` the
            callback runs on the host as soon as batch i has finished and before the slot's buffers are reused (the
            streaming form: bounded pinned memory, inflight x result size); the list of its return values is returned.
            Without a callback the results are returned as ordinary (pageable) host copies, valid indefinitely."""
        caller = torch.cuda.current_stream(self.device)
        ready = torch.cuda.Event()
        ready.record(caller)
        for s in self.slots:
            s.stream.wait_event(ready)
        results = []

        def retire(slot):
            if slot.pending is None:
                return
            i, host = slot.pending
            slot.done.synchronize()
            val = host[0] if len(host) == 1 else tuple(host)
            if consume is not None:
                val = consume(i, val)
            else:
                val = val.clone() if torch.is_tensor(val) else tuple(v.clone() for v in val)
            while len(results) <= i:
                results.append(None)
            results[i] = val
            slot.pending = None

        F = len(self.slots)
        for i, b in enumerate(batches):
            slot = self.slots[i % F]
            if to_host:
                retire(slot)               # the slot's pinned buffers are free again
            with torch.cuda.stream(slot.stream):
                x = b if b.is_cuda else b.to(self.device, non_blocking=True)
                outs = self._forward(slot, x)
                if to_host:
                    if slot.host is None or len(slot.host) != len(outs) or \
                            any(h.shape != o.shape or h.dtype != o.dtype for h, o in zip(slot.host, outs)):
                        slot.host = [torch.empty(o.shape, dtype=o.dtype, pin_memory=True) for o in outs]
                    for h, o in zip(slot.host, outs):
                        h.copy_(o, non_blocking=True)
                    if slot.done is None:
                        slot.done = torch.cuda.Event()
                    slot.done.record(slot.stream)
                    slot.pending = (i, slot.host)
                elif keep:
                    if self.graphs:
                        outs = tuple(o.clone() for o in outs)
                    results.append(outs[0] if len(outs) == 1 else tuple(outs))
                else:
                    results.append(None)
                del outs
        if to_host:
            # hand over what is still in flight, oldest first
            for slot in sorted((s for s in self.slots if s.pending is not None), key=lambda s: s.pending[0]):
                retire(slot)
        for s in self.slots:
            caller.wait_stream(s.stream)
        return results

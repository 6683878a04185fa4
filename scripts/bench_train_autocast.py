"""fp32 against bfloat16 autocast training: whole steps and the bfloat16 index natives, alternating.

    python scripts/bench_train_autocast.py [--steps 10] [--warmup 3] [--repeats 3] [--rpn-batch 16] [--rcnn-batch 4]

Steps: RPNTrainer.step at --rpn-batch scenes of 16384 points with the torch switches and with the device SA / FP / loss
switches, and RCNNTrainer.step_jit (device targets and loss) on --rcnn-batch synthetic scenes; each once as it is (fp32) and
once inside torch.autocast("cuda", dtype=torch.bfloat16), alternating, --repeats times --steps steps (ms per step) and the
peak memory the steps allocated.  Kernels: grouping forward / backward at the RPN SA2-SA4 shapes and interpolation forward /
backward at the RPN FP shapes (B = 16), fp32 against bfloat16 features, with the bytes each call must move (its index /
weight reads, its feature reads and writes; the gathered sources counted once) and the rate that gives.  One JSON line per
measurement, with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from pointrcnn_b200.pointnet2 import pointnet2_utils as pu  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def compare_steps(make_step, steps, warmup, repeats):
    """{"fp32": [ms...], "bf16": [ms...], "peak_mb": {...}}, the two alternating; make_step(autocast) -> a step callable"""
    res = {"fp32": [], "bf16": [], "peak_mb": {}}
    fns = {"fp32": make_step(False), "bf16": make_step(True)}
    for _ in range(repeats):
        for mode in ("fp32", "bf16"):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            res[mode].append(round(timed(fns[mode], steps, warmup), 3))
            res["peak_mb"][mode] = round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)
    return res


def rpn_step(batch, switches):
    from pointrcnn_b200.train.step import RPNTrainer

    def make(autocast):
        tr = RPNTrainer(device="cuda", seed=3, **switches)

        def step():
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                tr.step(*batch, grad_norm_clip=1.0)
        return step
    return make


def rcnn_step(batch):
    from pointrcnn_b200.train.step import RCNNTrainer

    def make(autocast):
        tr = RCNNTrainer(device="cuda", seed=5, target_draw="device", loss_impl="device")

        def step():
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                tr.step_jit(batch, grad_norm_clip=1.0)
        return step
    return make


# (B, C, N, npoint, nsample) of the RPN SA levels whose features are bfloat16 under autocast, and (B, C, n, m) of the FP levels
GROUP = {"rpn_sa2_ns32": (16, 96, 4096, 1024, 32), "rpn_sa3_ns32": (16, 256, 1024, 256, 32), "rpn_sa4_ns32": (16, 512, 256, 64, 32)}
INTERP = {"rpn_fp3": (16, 1024, 256, 64), "rpn_fp2": (16, 512, 1024, 256), "rpn_fp1": (16, 512, 4096, 1024), "rpn_fp0": (16, 256, 16384, 4096)}


def kernel_rows(steps, warmup, repeats):
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, (B, C, N, P, S) in GROUP.items():
        idx = torch.randint(0, N, (B, P, S), device="cuda", generator=g).int()
        for dtype in (torch.float32, torch.bfloat16):
            f = torch.randn(B, C, N, device="cuda", generator=g).to(dtype).requires_grad_(True)
            out = pu.grouping_operation(f, idx)
            gout = torch.randn_like(out)
            e = f.element_size()
            fwd_bytes = 4 * B * P * S + e * B * C * P * S + e * B * C * N
            bwd_bytes = 4 * B * P * S + e * B * C * P * S + e * B * C * N + (8 * B * C * N if dtype == torch.bfloat16 else 4 * B * C * N)
            fwd = [timed(lambda: pu.grouping_operation(f, idx), steps, warmup) for _ in range(repeats)]
            bwd = [timed(lambda: torch.autograd.grad(out, f, gout, retain_graph=True), steps, warmup) for _ in range(repeats)]
            yield dict(kernel="group", shape=name, dtype=str(dtype)[6:], fwd_ms=[round(t, 4) for t in fwd], bwd_ms=[round(t, 4) for t in bwd],
                       fwd_bytes=fwd_bytes, bwd_bytes=bwd_bytes, fwd_gbps=round(fwd_bytes / min(fwd) / 1e6, 1),
                       bwd_gbps=round(bwd_bytes / min(bwd) / 1e6, 1))
    for name, (B, C, n, m) in INTERP.items():
        idx = torch.randint(0, m, (B, n, 3), device="cuda", generator=g).int()
        w = torch.rand(B, n, 3, device="cuda", generator=g)
        w = (w / w.sum(2, keepdim=True)).contiguous()
        for dtype in (torch.float32, torch.bfloat16):
            f = torch.randn(B, C, m, device="cuda", generator=g).to(dtype).requires_grad_(True)
            out = pu.three_interpolate(f, idx, w)
            gout = torch.randn_like(out)
            e = f.element_size()
            fwd_bytes = 24 * B * n + e * B * C * n + e * B * C * m
            bwd_bytes = 24 * B * n + e * B * C * n + e * B * C * m + (8 * B * C * m if dtype == torch.bfloat16 else 4 * B * C * m)
            fwd = [timed(lambda: pu.three_interpolate(f, idx, w), steps, warmup) for _ in range(repeats)]
            bwd = [timed(lambda: torch.autograd.grad(out, f, gout, retain_graph=True), steps, warmup) for _ in range(repeats)]
            yield dict(kernel="three_interpolate", shape=name, dtype=str(dtype)[6:], fwd_ms=[round(t, 4) for t in fwd],
                       bwd_ms=[round(t, 4) for t in bwd], fwd_bytes=fwd_bytes, bwd_bytes=bwd_bytes,
                       fwd_gbps=round(fwd_bytes / min(fwd) / 1e6, 1), bwd_gbps=round(bwd_bytes / min(bwd) / 1e6, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--rpn-batch", type=int, default=16)
    ap.add_argument("--rcnn-batch", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_train_autocast: needs a CUDA device")
    import synth
    from oracle import rcnn_offline as RO
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    from pointrcnn_b200.train.step import synthetic_labels
    gpu = card()
    pc = torch.from_numpy(synth.u_kitti(a.rpn_batch, 16384, 123, channels=4)).cuda()
    rpn_batch = (pc,) + tuple(synthetic_labels(pc, seed=1))
    for label, switches in (("torch", {}), ("device", dict(loss_impl="device", sa_train="device", fp_train="device"))):
        res = compare_steps(rpn_step(rpn_batch, switches), a.steps, a.warmup, a.repeats)
        print(json.dumps(dict(bench="RPNTrainer.step", batch=a.rpn_batch, switches=label, gpu=gpu, ms_per_step=res)), flush=True)
    kinds = ("mixed", "hard", "easy", "mixed")
    scenes = [RO.synth_scene(51 + i, kinds[i % len(kinds)], n_feat=128) for i in range(a.rcnn_batch)]
    jit = RCNNOfflineSampler(device="cuda").prepare_jit_batch(scenes)
    res = compare_steps(rcnn_step(jit), a.steps, a.warmup, a.repeats)
    print(json.dumps(dict(bench="RCNNTrainer.step_jit", batch=a.rcnn_batch, switches="device", gpu=gpu, ms_per_step=res)), flush=True)
    for row in kernel_rows(max(a.steps, 20), a.warmup, a.repeats):
        print(json.dumps(dict(bench="index_op", gpu=gpu, **row)), flush=True)


if __name__ == "__main__":
    main()

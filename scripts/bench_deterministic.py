"""The ordered gradient entries against the atomic ones: torch.use_deterministic_algorithms off and on, alternating.

    python scripts/bench_deterministic.py [--steps 20] [--warmup 3] [--repeats 3] [--train-steps 5]

Per op: the reference-named shim (group_points_grad, gather_points_grad, three_interpolate_grad) at the RPN training
shapes (B = 16 scenes of 16384 points: SA1-SA4 grouping of the features and the xyz, FP interpolation) and the RCNN ones
(B = 4 scenes x 64 RoIs = 256 groups of 512 points: SA1, SA2 grouping); idx is ball-query-like (a random number of hits
per centre, the rest padded with the first hit).  With the flag on a call also builds the reverse index of idx and
fills its scratch (torch fills uninitialised memory in deterministic mode).  Then whole steps: RPNTrainer.step (device
SA / FP / loss) at --rpn-batch and RCNNTrainer.step_jit (device targets / loss) on --rcnn-batch synthetic scenes.
Every time is measured --repeats times, off and on alternating, and reported as the list of repeats (ms per call).
One JSON line per measurement, with the card name and power limit read in the same run.  CUBLAS_WORKSPACE_CONFIG is set
to :4096:8 for both variants (deterministic cuBLAS needs it).
"""
import argparse
import json
import os
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import torch  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from pointrcnn_b200.ext import pointnet2_cuda as P  # noqa: E402


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


def compare(fn, steps, warmup, repeats):
    """{"off": [ms...], "on": [ms...]}, the two alternating"""
    res = {"off": [], "on": []}
    for _ in range(repeats):
        for mode in ("off", "on"):
            torch.use_deterministic_algorithms(mode == "on")
            try:
                res[mode].append(round(timed(fn, steps, warmup), 4))
            finally:
                torch.use_deterministic_algorithms(False)
    return res


def padded_idx(gen, b, npoint, ns, n):
    idx = torch.randint(0, n, (b, npoint, ns), generator=gen)
    hits = torch.randint(1, ns + 1, (b, npoint, 1), generator=gen)
    return torch.where(torch.arange(ns) >= hits, idx[:, :, :1], idx).int()


GROUP = {
    # name: (B, C, N, npoint, nsample)
    "rpn_sa1_xyz_ns16": (16, 3, 16384, 4096, 16), "rpn_sa1_xyz_ns32": (16, 3, 16384, 4096, 32),
    "rpn_sa1_feats_ns16": (16, 1, 16384, 4096, 16), "rpn_sa1_feats_ns32": (16, 1, 16384, 4096, 32),
    "rpn_sa2_ns16": (16, 96, 4096, 1024, 16), "rpn_sa2_ns32": (16, 96, 4096, 1024, 32),
    "rpn_sa3_ns16": (16, 256, 1024, 256, 16), "rpn_sa3_ns32": (16, 256, 1024, 256, 32),
    "rpn_sa4_ns16": (16, 512, 256, 64, 16), "rpn_sa4_ns32": (16, 512, 256, 64, 32),
    "rcnn_sa1": (256, 128, 512, 128, 64), "rcnn_sa2": (256, 128, 128, 32, 64),
}
GATHER = {"rpn_sa1_new_xyz": (16, 3, 16384, 4096), "rpn_sa2_new_xyz": (16, 3, 4096, 1024)}
INTERP = {
    # name: (B, C, n unknown, m known)
    "rpn_fp3": (16, 1024, 256, 64), "rpn_fp2": (16, 512, 1024, 256), "rpn_fp1": (16, 512, 4096, 1024), "rpn_fp0": (16, 256, 16384, 4096),
}


def bench_ops(a, name, dev):
    gen = torch.Generator().manual_seed(0)
    for k, (B, Cc, N, npoint, ns) in GROUP.items():
        idx = padded_idx(gen, B, npoint, ns, N).to(dev)
        g = torch.randn(B, Cc, npoint, ns, generator=gen).to(dev)
        gp = torch.zeros(B, Cc, N, device=dev)
        res = compare(lambda: P.group_points_grad_wrapper(B, Cc, N, npoint, ns, g, idx, gp), a.steps, a.warmup, a.repeats)
        print(json.dumps(dict(bench="group_points_grad", shape=k, B=B, C=Cc, N=N, npoint=npoint, nsample=ns, card=name, **res)), flush=True)
    for k, (B, Cc, N, npoint) in GATHER.items():
        idx = torch.randint(0, N, (B, npoint), generator=gen).int().to(dev)
        g = torch.randn(B, Cc, npoint, generator=gen).to(dev)
        gp = torch.zeros(B, Cc, N, device=dev)
        res = compare(lambda: P.gather_points_grad_wrapper(B, Cc, N, npoint, g, idx, gp), a.steps, a.warmup, a.repeats)
        print(json.dumps(dict(bench="gather_points_grad", shape=k, B=B, C=Cc, N=N, npoint=npoint, card=name, **res)), flush=True)
    for k, (B, Cc, n, m) in INTERP.items():
        idx = torch.stack([torch.randperm(m, generator=gen)[:3] for _ in range(64)])[torch.randint(0, 64, (B, n), generator=gen)]
        idx = ((idx + torch.randint(0, m, (B, n, 1), generator=gen)) % m).int().to(dev)
        w = torch.rand(B, n, 3, generator=gen) + 0.01
        w = (w / w.sum(2, keepdim=True)).to(dev)
        g = torch.randn(B, Cc, n, generator=gen).to(dev)
        gp = torch.zeros(B, Cc, m, device=dev)
        res = compare(lambda: P.three_interpolate_grad_wrapper(B, Cc, n, m, g, idx, w, gp), a.steps, a.warmup, a.repeats)
        print(json.dumps(dict(bench="three_interpolate_grad", shape=k, B=B, C=Cc, n=n, m=m, card=name, **res)), flush=True)


def bench_steps(a, name, dev):
    import synth
    from oracle import rcnn_offline as RO
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer, synthetic_labels
    pc = torch.from_numpy(synth.u_kitti(a.rpn_batch, 16384, 123, channels=4)).to(dev)
    cls, reg = synthetic_labels(pc, seed=1)
    tr = RPNTrainer(input_channels=1, device=dev, world=1, seed=3, loss_impl="device", sa_train="device", fp_train="device")
    res = compare(lambda: tr.step(pc, cls, reg, grad_norm_clip=1.0), a.train_steps, a.warmup, a.repeats)
    print(json.dumps(dict(bench="RPNTrainer.step", B=a.rpn_batch, card=name, **res)), flush=True)
    del tr
    kinds = ("mixed", "hard", "easy")
    scenes = [RO.synth_scene(51 + i, kinds[i % 3], n_feat=128) for i in range(a.rcnn_batch)]
    batch = RCNNOfflineSampler(device=dev).prepare_jit_batch(scenes)
    tr = RCNNTrainer(device=dev, seed=5, target_draw="device", loss_impl="device")
    res = compare(lambda: tr.step_jit(batch, grad_norm_clip=1.0), a.train_steps, a.warmup, a.repeats)
    print(json.dumps(dict(bench="RCNNTrainer.step_jit", B=a.rcnn_batch, card=name, **res)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--train-steps", type=int, default=5)
    ap.add_argument("--rpn-batch", type=int, default=16)
    ap.add_argument("--rcnn-batch", type=int, default=4)
    ap.add_argument("--skip-steps", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic: needs a CUDA device")
    dev = torch.device("cuda:0")
    name = card()
    bench_ops(a, name, dev)
    if not a.skip_steps:
        bench_steps(a, name, dev)


if __name__ == "__main__":
    main()

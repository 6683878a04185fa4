"""RPNTrainer.step with optimizer="adam" (torch Adam, L2 decay) against "adam_onecycle" (the reference's default recipe:
true weight decay + fused Adam, OneCycle lr / beta1 set before every step), alternating.

    python scripts/bench_train_recipe.py [--batch 16] [--steps 10] [--warmup 3] [--repeats 3]

Both trainers use the device SA / FP / loss paths and clip the gradient norm to 1.0, on the same synthetic scenes of 16384
points.  Every time is measured --repeats times, the two variants alternating, and reported as the list of repeats (ms per
step).  One JSON line, with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

import synth  # noqa: E402
from pointrcnn_b200.train import recipe  # noqa: E402
from pointrcnn_b200.train.step import RPNTrainer, synthetic_labels  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_recipe needs a CUDA device")
    dev = torch.device("cuda:0")
    pc = torch.from_numpy(synth.u_kitti(a.batch, 16384, 123, channels=4)).to(dev)
    cls, reg = synthetic_labels(pc, seed=1)
    total = (a.warmup + a.steps) * a.repeats
    trainers = {name: RPNTrainer(device=dev, seed=3, optimizer=name, total_steps=total if name == "adam_onecycle" else None,
                                 loss_impl="device", sa_train="device", fp_train="device") for name in recipe.OPTIMIZERS}
    its = dict.fromkeys(trainers, 0)

    def one(name):
        tr = trainers[name]
        tr.schedule_iteration(its[name], 0, total)
        tr.step(pc, cls, reg, grad_norm_clip=recipe.GRAD_NORM_CLIP)
        its[name] += 1

    res = {name: [] for name in trainers}
    for _ in range(a.repeats):
        for name in trainers:
            for _ in range(a.warmup):
                one(name)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                one(name)
            e1.record()
            torch.cuda.synchronize()
            res[name].append(round(e0.elapsed_time(e1) / a.steps, 3))
    print(json.dumps({"bench": "train_recipe_rpn_step", "batch": a.batch, "steps": a.steps, "card": card(), "ms_per_step": res}))


if __name__ == "__main__":
    main()

"""oracle/bench_ref_cuda.py -- time the reference's own CUDA-extension pipeline on the bench workload (B-ref of
BASELINE.md): the UNMODIFIED reference kernels (oracle/_ref, rebuilt for sm_90a) called in exactly the order
pointnet2_modules.py calls them (ref:pointnet2_modules.py:19-55,127-156, pointnet2_utils.py:241-264), with the
MLP through stock torch.nn Conv2d/BatchNorm2d/ReLU/max_pool2d (cuDNN/cuBLAS, torch defaults incl. TF32 convs).

TEST / BASELINE INFRASTRUCTURE ONLY.  Usage on the GPU box:  python oracle/bench_ref_cuda.py [--steps 10]
Prints one JSON line (also the per-family event timings).
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402  (workload definition: model, scenes, constants)
from oracle import refgpu as R  # noqa: E402
from pointrcnn_b200 import prof  # noqa: E402  (event timer only)


from oracle.ref_backbone import backbone  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    net = bench.build_model(dev)
    pc = torch.from_numpy(bench.make_scenes(0, bench.BATCH)).to(dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    with torch.no_grad():
        for _ in range(a.warmup):
            backbone(net, pc)
        torch.cuda.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.steps)]
        prof.enable()
        for s, e in ev:
            flush.fill_(1.0)
            s.record()
            _, feats = backbone(net, pc)
            e.record()
        torch.cuda.synchronize()
        prof.disable()
    ms = sum(s.elapsed_time(e) for s, e in ev) / a.steps
    fam = {k: v[0] / a.steps for k, v in prof.collect().items()}
    print(json.dumps({"impl": "reference CUDA-extension build (oracle/_ref kernels, sm_90a, + torch cuDNN MLP)",
                      "metric": "scenes/sec RPN backbone fwd (16384 pts)", "value": bench.BATCH / (ms * 1e-3), "unit": "scenes/s",
                      "ms_per_step": ms, "steps": a.steps, "batch": bench.BATCH, "family_ms_per_step": fam,
                      "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32, "checksum": float(feats.double().mean())}))


if __name__ == "__main__":
    main()

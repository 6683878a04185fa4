"""FP modules in training mode: the torch path (config.fp_train="torch") against the device path (prb_fp_train_* in
csrc/sa_train.cu), per level forward / backward time, launches, host syncs and peak memory, and whole RPNTrainer steps with
the switch off and on.

    python scripts/bench_fp_train.py [--steps 10] [--warmup 3] [--repeats 3] [--batch 16]

Levels: the RPN backbone's FP3-FP0 on B x 16384 points, each fed what the training step gives it (one forward without
grad, captured at the module).  Every time is measured --repeats times, the two variants alternating, and reported as
the list of repeats.  The "split" line puts the torch path's FP levels (forward + backward, each measured alone) next to
the whole torch RPNTrainer.step.  Prints one JSON line per measurement with the card name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200 import config  # noqa: E402


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


def host_syncs(fn):
    """synchronising CUDA calls torch reports while fn runs"""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(x.message) for x in w)


def fp_inputs(backbone, pc):
    """(unknown, known, skip, known_feats) of every FP module as the training forward calls it"""
    got = {}
    hooks = [m.register_forward_pre_hook(lambda mod, a, k=k: got.setdefault(k, tuple(t.detach() if t is not None else None for t in a)))
             for k, m in enumerate(backbone.FP_modules)]
    with torch.no_grad():
        backbone(pc)
    for h in hooks:
        h.remove()
    return [got[k] for k in range(len(backbone.FP_modules))]


def bench_levels(backbone, inputs, steps, warmup, repeats, name):
    """-> {variant: {level: median forward + backward ms}}"""
    med = {}
    for k in range(len(inputs) - 1, -1, -1):
        m = backbone.FP_modules[k]
        unknown, known, skip, kf = inputs[k]
        kf = kf.detach().requires_grad_(True)
        sk = skip.detach().requires_grad_(k > 0) if skip is not None else None
        variants = {
            "torch": lambda: m(unknown, known, sk, kf),
            "device": lambda: m._forward_train(unknown, known, sk, kf),
        }
        res = {v: [] for v in variants}
        for _ in range(repeats):
            for v, run in variants.items():
                with config.override(fp_train="torch"):
                    def fwd():
                        run()

                    def fwd_bwd():
                        m.zero_grad(set_to_none=True)
                        out = run()
                        out.backward(torch.ones_like(out))

                    f = timed(fwd, steps, warmup)
                    t = timed(fwd_bwd, steps, warmup)
                    res[v].append((f, t))
        for v, run in variants.items():
            def fwd_bwd():
                m.zero_grad(set_to_none=True)
                out = run()
                out.backward(torch.ones_like(out))
            with config.override(fp_train="torch"):
                lc = C.launch_count()
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                fwd_bwd()
                torch.cuda.synchronize()
                peak = torch.cuda.max_memory_allocated() - base
                launches = C.launch_count() - lc
                syncs = host_syncs(fwd_bwd)
            fw = sorted(r[0] for r in res[v])
            bw = sorted(r[1] - r[0] for r in res[v])
            tot = sorted(r[1] for r in res[v])
            med.setdefault(v, {})[k] = tot[len(tot) // 2]
            print(json.dumps(dict(bench="fp_level", level="rpn_fp%d" % k, impl=v, rows=int(unknown.size(0) * unknown.size(1)),
                                  known_rows=int(known.size(0) * known.size(1)), fwd_ms=[round(x, 3) for x in fw],
                                  bwd_ms=[round(x, 3) for x in bw], total_ms=[round(x, 3) for x in tot], lib_launches=launches,
                                  host_syncs=syncs, peak_mb=round(peak / 2 ** 20, 1), card=name)), flush=True)
    return med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_fp_train: no GPU")
    import synth
    from pointrcnn_b200.backbone import Pointnet2MSG
    from pointrcnn_b200.train.step import RPNTrainer, synthetic_labels
    dev = torch.device("cuda")
    name = card()

    torch.manual_seed(0)
    pc = torch.from_numpy(synth.u_kitti(args.batch, 16384, 123, channels=4)).to(dev)
    backbone = Pointnet2MSG(input_channels=1).to(dev).train()
    med = bench_levels(backbone, fp_inputs(backbone, pc), args.steps, args.warmup, args.repeats, name)

    cls, reg = synthetic_labels(pc, seed=1)
    trainers = {impl: RPNTrainer(input_channels=1, device=dev, seed=3, loss_impl="device", sa_train="device", fp_train=impl)
                for impl in ("torch", "device")}
    trainers["all_torch"] = RPNTrainer(input_channels=1, device=dev, seed=3, loss_impl="device", sa_train="torch", fp_train="torch")
    steps = {k: [] for k in trainers}
    for _ in range(args.repeats):
        for k, tr in trainers.items():
            steps[k].append(timed(lambda: tr.step(pc, cls, reg), args.steps, args.warmup))
    for k, ms in steps.items():
        sa, fp = ("torch", "torch") if k == "all_torch" else ("device", k)
        print(json.dumps(dict(bench="rpn_step", sa_train=sa, fp_train=fp, batch=args.batch, ms=sorted(round(x, 2) for x in ms),
                              card=name)), flush=True)
    step_ms = sorted(steps["all_torch"])[args.repeats // 2]
    fp_ms = sum(med["torch"].values())
    print(json.dumps(dict(bench="split", what="torch RPNTrainer.step vs its FP levels measured alone", step_ms=round(step_ms, 2),
                          fp_ms=round(fp_ms, 2), fp_share=round(fp_ms / step_ms, 3), card=name)), flush=True)


if __name__ == "__main__":
    main()

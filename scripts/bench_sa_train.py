"""SA modules in training mode: the torch path (config.sa_train="torch") against the device path (csrc/sa_train.cu), per
level forward / backward time, launches and peak memory, and whole trainer steps with each setting.

    python scripts/bench_sa_train.py [--steps 10] [--warmup 3] [--repeats 3] [--rpn-batch 16] [--rcnn-batch 4] [--profile DIR]

Levels: the RPN backbone's SA1-SA4 on B x 16384 points (inputs: the previous levels' outputs) and the RCNN stage's SA1-SA3
on B x 64 RoIs x 512 points.  Every time is measured --repeats times, torch and device alternating, and reported as the
list of repeats.  The "split" line puts the torch path's SA levels (forward + backward, each measured alone on the inputs
the step gives it) next to the whole torch RPNTrainer.step.  Prints one JSON line per measurement with the card name and
power limit.  --profile writes a torch.profiler table of one RPNTrainer.step per setting (a separate run: tracing slows
the host).
"""
import argparse
import json
import os
import subprocess
import sys

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


def level_inputs(modules, xyz, feats):
    """the (xyz, features) each module of a stack sees, from one forward without grad"""
    out = []
    with torch.no_grad():
        for m in modules:
            out.append((xyz, feats.contiguous() if feats is not None else None))
            xyz, feats = m(xyz, feats)
            if xyz is None:
                break
    return out


def bench_levels(tag, modules, inputs, steps, warmup, repeats, card_name):
    """-> {impl: summed median forward + backward ms over the levels}"""
    totals = {"torch": 0.0, "device": 0.0}
    for k, (m, (xyz, feats)) in enumerate(zip(modules, inputs)):
        f = feats.detach().requires_grad_(k > 0) if feats is not None else None
        res = {"torch": [], "device": []}
        for impl in ["torch", "device"] * repeats:
            with config.override(sa_train=impl):
                holder = {}

                # the device side runs _forward_train directly, so levels outside sa_train.FAST_MAX_WIDTH are measured too
                run = m._forward_train if impl == "device" else m

                def fwd():
                    holder["out"] = run(xyz, f, None)[1]

                def fwd_bwd():
                    m.zero_grad(set_to_none=True)
                    out = run(xyz, f, None)[1]
                    out.backward(torch.ones_like(out))

                fwd_ms = timed(fwd, steps, warmup)
                holder.clear()
                total_ms = timed(fwd_bwd, steps, warmup)
                res[impl].append((fwd_ms, total_ms))
                if len(res[impl]) < repeats:
                    continue
                lc = C.launch_count()
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                fwd_bwd()
                torch.cuda.synchronize()
                peak = torch.cuda.max_memory_allocated() - base
                fw = sorted(r[0] for r in res[impl])
                bw = sorted(r[1] - r[0] for r in res[impl])
                totals[impl] += sorted(r[1] for r in res[impl])[len(fw) // 2]
                print(json.dumps(dict(bench="sa_level", level="%s_sa%d" % (tag, k + 1), impl=impl, fwd_ms=[round(x, 3) for x in fw],
                                      bwd_ms=[round(x, 3) for x in bw], lib_launches=C.launch_count() - lc,
                                      peak_mb=round(peak / 2 ** 20, 1), card=card_name)), flush=True)
    return totals


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--rpn-batch", type=int, default=16)
    ap.add_argument("--rcnn-batch", type=int, default=4)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_sa_train: no GPU")
    import synth
    from oracle import rcnn_offline as RO
    from pointrcnn_b200.backbone import Pointnet2MSG
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer, synthetic_labels
    dev = torch.device("cuda")
    name = card()

    torch.manual_seed(0)
    pc = torch.from_numpy(synth.u_kitti(args.rpn_batch, 16384, 123, channels=4)).to(dev)
    backbone = Pointnet2MSG(input_channels=1).to(dev).train()
    xyz, feats = pc[..., :3].contiguous(), pc[..., 3:].transpose(1, 2).contiguous()
    rpn_sa = bench_levels("rpn", list(backbone.SA_modules), level_inputs(backbone.SA_modules, xyz, feats), args.steps, args.warmup,
                          args.repeats, name)

    scenes = [RO.synth_scene(50 + s, "mixed", n_feat=128) for s in range(args.rcnn_batch)]
    batch = RCNNOfflineSampler(device=dev).prepare_jit_batch(scenes)
    rc = RCNNTrainer(device=dev, seed=5, target_draw="device", loss_impl="device")
    captured = {}
    sa0 = rc.model.SA_modules[0]
    hook = sa0.register_forward_pre_hook(lambda mod, a: captured.setdefault("in", (a[0].detach(), a[1].detach())))
    with torch.no_grad():
        rc.model.forward_train(batch, target_draw="device")
    hook.remove()
    xyz, feats = captured["in"]
    bench_levels("rcnn", list(rc.model.SA_modules), level_inputs(rc.model.SA_modules, xyz, feats), args.steps, args.warmup, args.repeats,
                 name)

    cls, reg = synthetic_labels(pc, seed=1)
    trainers = {impl: (RPNTrainer(input_channels=1, device=dev, seed=3, loss_impl="device", sa_train=impl),
                       RCNNTrainer(device=dev, seed=5, target_draw="device", loss_impl="device", sa_train=impl)) for impl in ("torch", "device")}
    steps = {(k, impl): [] for k in ("rpn_step", "rcnn_step_jit") for impl in ("torch", "device")}
    for _ in range(args.repeats):
        for impl, (rpn, rcnn) in trainers.items():
            steps[("rpn_step", impl)].append(timed(lambda: rpn.step(pc, cls, reg), args.steps, args.warmup))
            steps[("rcnn_step_jit", impl)].append(timed(lambda: rcnn.step_jit(batch), args.steps, args.warmup))
    for (k, impl), ms in steps.items():
        print(json.dumps(dict(bench=k, impl=impl, batch=args.rpn_batch if k == "rpn_step" else args.rcnn_batch,
                              ms=sorted(round(x, 2) for x in ms), card=name)), flush=True)
    step_ms = sorted(steps[("rpn_step", "torch")])[args.repeats // 2]
    print(json.dumps(dict(bench="split", what="torch RPNTrainer.step vs its SA levels measured alone", step_ms=round(step_ms, 2),
                          sa_ms=round(rpn_sa["torch"], 2), sa_share=round(rpn_sa["torch"] / step_ms, 3), card=name)), flush=True)

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.profile, exist_ok=True)
        for impl in ("torch", "device"):
            tr = RPNTrainer(input_channels=1, device=dev, seed=3, loss_impl="device", sa_train=impl)
            tr.step(pc, cls, reg)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                tr.step(pc, cls, reg)
                torch.cuda.synchronize()
            with open(os.path.join(args.profile, "rpn_step_%s.txt" % impl), "w") as fh:
                fh.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40))


if __name__ == "__main__":
    main()

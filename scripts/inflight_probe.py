"""How much does running consecutive batches on alternating streams buy? (feasibility probe)"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch, bench
dev = torch.device("cuda:0")
net = bench.build_model(dev)
pool = [torch.from_numpy(bench.make_scenes(16 * i, 16)).to(dev) for i in range(8)]
with torch.no_grad():
    for F in (1, 2, 3):
        streams = [torch.cuda.Stream() for _ in range(F)]
        for i in range(6):
            with torch.cuda.stream(streams[i % F]): net(pool[i % 8])
        torch.cuda.synchronize()
        K = 24
        t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
        t0.record()
        for s in streams: s.wait_event(t0)
        for i in range(K):
            with torch.cuda.stream(streams[i % F]): net(pool[i % 8])
        for s in streams: torch.cuda.current_stream().wait_stream(s)
        t1.record(); torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / K
        print("inflight", F, "ms/batch %.3f" % ms, "scenes/s %.0f" % (16 / ms * 1e3), flush=True)

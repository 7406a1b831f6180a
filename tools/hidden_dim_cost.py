#!/usr/bin/env python
"""Train-step time of the C2 workload (1080x1920, V = 200, 1024 rays x 128 samples, uniform + jitter, rgb L1 + depth L1, Adam x3, whole-step
CUDA graph; bench.py's headline configuration) at model.hidden_dim 256, 128 and 64: one trainer per width, timed in alternating windows of
K steps (CUDA events), median over the windows.   python tools/hidden_dim_cost.py [K] [windows]"""
import json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import bench

K = int(sys.argv[1]) if len(sys.argv) > 1 else 30
NWIN = int(sys.argv[2]) if len(sys.argv) > 2 else 5
DIMS = (256, 128, 64)
dev = torch.device("cuda", 0); torch.cuda.set_device(0)
_, frames = bench.synth_frames(bench.H, bench.W, bench.HD, bench.WD, bench.N_FRAMES, bench.V, dev, with_ref=False)
trainers = {}
for D in DIMS:
    cfg = bench.make_cfg(bench.NRAYS)
    cfg["model"]["hidden_dim"] = D
    trainers[D] = bench.build_trainer(cfg, dev, bench.V)


def run(tr, n, start):
    for i in range(start, start + n):
        ld = tr.train_step(frames[i % len(frames)], it=i, epoch=0, scheduling_start=10000, render_path=None)
    return ld


for tr in trainers.values():
    run(tr, 30, 0)                                   # eager first step, capture, clocks settle
torch.cuda.synchronize()
times = {D: [] for D in DIMS}
for w in range(NWIN):
    for D, tr in trainers.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); run(tr, K, 30 + w * K); e1.record(); torch.cuda.synchronize()
        times[D].append(e0.elapsed_time(e1) / K)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {}
for D, v in times.items():
    med = float(np.median(v))
    out["d%d" % D] = {"ms_per_step_median": round(med, 4), "ms_per_step_min": round(min(v), 4), "ms_per_step_max": round(max(v), 4),
                      "ray_samples_per_s": round(bench.NRAYS * bench.S / (med / 1e3), 1)}
out.update(steps_per_window=K, windows=NWIN, gpu=q.splitlines()[0] if q else torch.cuda.get_device_name(0))
print(json.dumps(out))

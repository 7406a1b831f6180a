#!/usr/bin/env python
"""Step time of the training options that the whole-step CUDA graph runs (pose.learn_focal, training.depth_loss_type = invariant,
training.weight_dist_1st_loss / weight_dist_2nd_loss) on the C2 render step (1080 x 1920 frames, 1024 rays x 128 samples): for each
option the eager general path (Trainer(use_cuda_graph=False): torch autograd / median / Adam, kernels launched one by one) and the
captured graph, plus the default step's graph, timed in alternating windows of K steps (CUDA events) in one session, median over
the windows.  The card's name and power limit are queried in the same run.   python tools/graph_options_cost.py [K] [windows]"""
import json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import bench
import nope_nerf_b200.model as mdl

K = int(sys.argv[1]) if len(sys.argv) > 1 else 20
NWIN = int(sys.argv[2]) if len(sys.argv) > 2 else 7
dev = torch.device("cuda", 0); torch.cuda.set_device(0)
_, frames = bench.synth_frames(bench.H, bench.W, bench.HD, bench.WD, 4, bench.V, dev, with_ref=False)
OPTIONS = {"default": {}, "learn_focal": {"focal": True}, "invariant_depth": {"training": {"depth_loss_type": "invariant"}},
           "pose_smoothness": {"training": {"weight_dist_1st_loss": [0.1, 0.1], "weight_dist_2nd_loss": [0.1, 0.1]}},
           "all_three": {"focal": True, "training": {"depth_loss_type": "invariant", "weight_dist_1st_loss": [0.1, 0.1],
                                                     "weight_dist_2nd_loss": [0.1, 0.1]}}}


def make(opts, graph):
    cfg = bench.make_cfg(bench.NRAYS)
    cfg["training"].update(opts.get("training", {}))
    tr = bench.build_trainer(cfg, dev, bench.V)
    tr.use_cuda_graph = graph
    if opts.get("focal"):
        kx = float(frames[0]["img.camera_mat"][0, 0, 0]); ky = -float(frames[0]["img.camera_mat"][0, 1, 1])
        tr.focal_net = mdl.LearnFocal(True, False, order=2, init_focal=[kx, ky]).to(dev)
        tr.optimizer_focal = torch.optim.Adam(tr.focal_net.parameters(), lr=1e-3)
    return tr


trainers = {}
for name, opts in OPTIONS.items():
    for graph in ((True,) if name == "default" else (False, True)):
        trainers["%s/%s" % (name, "graph" if graph else "general")] = make(opts, graph)


def run(tr, n, start):
    for i in range(start, start + n):
        ld = tr.train_step(frames[i % 4], it=i, epoch=0, scheduling_start=10000, render_path=None)
    return ld


for n, tr in trainers.items():
    run(tr, 30, 0)                                   # eager first step, capture, clocks settle
    on_graph = any(v and v.graph is not None for v in tr._gsteps.values())
    assert on_graph == n.endswith("/graph"), n
torch.cuda.synchronize()
times = {n: [] for n in trainers}
for w in range(NWIN):
    for n, tr in trainers.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); run(tr, K, 30 + w * K); e1.record(); torch.cuda.synchronize()
        times[n].append(e0.elapsed_time(e1) / K)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {n: {"ms_per_step_median": round(float(np.median(v)), 4), "ms_per_step_min": round(min(v), 4), "ms_per_step_max": round(max(v), 4)}
       for n, v in times.items()}
out["speedup_graph_over_general"] = {o: round(out[o + "/general"]["ms_per_step_median"] / out[o + "/graph"]["ms_per_step_median"], 2)
                                     for o in OPTIONS if o != "default"}
out.update(steps_per_window=K, windows=NWIN, gpu=q.splitlines()[0] if q else torch.cuda.get_device_name(0))
print(json.dumps(out))

#!/usr/bin/env python
"""Cost of training.with_ssim = True + training.detach_ref_img = False on the C2 full-loss train step (1024 rays x 128 samples, point-cloud
+ warped-RGB terms, whole-step CUDA graph): the same step with the default options and with both options on, timed in alternating
windows of K steps (CUDA events), median over the windows; and the reference-image stage on its own (nnb_refstage at C2 size, 96 x 168
points), which in the step runs on a forked stream beside the render backward.   python tools/refopts_cost.py [K] [windows]"""
import json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import bench

K = int(sys.argv[1]) if len(sys.argv) > 1 else 50
NWIN = int(sys.argv[2]) if len(sys.argv) > 2 else 7
dev = torch.device("cuda", 0); torch.cuda.set_device(0)
_, frames = bench.synth_frames(bench.H, bench.W, bench.HD, bench.WD, 4, bench.V, dev, with_ref=True)
trainers = {}
for name, opts in (("full_loss", {}), ("full_loss_refopts", {"with_ssim": True, "detach_ref_img": False})):
    cfg = bench.make_cfg(bench.NRAYS, full_loss=True)
    cfg["training"].update(opts)
    trainers[name] = bench.build_trainer(cfg, dev, bench.V)


def run(tr, n, start):
    for i in range(start, start + n):
        ld = tr.train_step(frames[i % 4], it=i, epoch=0, scheduling_start=10000, render_path=None)
    return ld


for tr in trainers.values():
    run(tr, 30, 0)                                   # eager first step, capture, clocks settle
torch.cuda.synchronize()
times = {n: [] for n in trainers}
for w in range(NWIN):
    for n, tr in trainers.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); ld = run(tr, K, 30 + w * K); e1.record(); torch.cuda.synchronize()
        times[n].append(e0.elapsed_time(e1) / K)
# the stage alone, default flags vs both options (same inputs as the step's first frame pair, identity-ish poses)
from nope_nerf_b200 import ops
f0 = frames[0]
c2w, c2wr = torch.eye(4, device=dev), torch.eye(4, device=dev); c2wr[0, 3] = 0.05
dc, dr = torch.tensor([1.0, 0.0], device=dev), torch.tensor([1.02, 0.01], device=dev)
stage = {}
for n, kw in (("refstage", {}), ("refstage_refopts", dict(with_ssim=True, g_c2w_ref=torch.zeros(4, 4, device=dev), g_dist_ref=torch.zeros(2, device=dev)))):
    call = lambda: ops.refstage_raw(c2w, dc, c2wr, dr, f0["img.dpt"][0], f0["img.ref_dpts"][0], H=bench.H, W=bench.W, img_cur=f0["img"][0],
                                    img_ref=f0["img.ref_imgs"][0], kx=1.2, ky=-2.13, g_c2w=torch.zeros(4, 4, device=dev),
                                    g_dist=torch.zeros(2, device=dev), **kw)
    for _ in range(5): call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50): call()
    e1.record(); torch.cuda.synchronize()
    stage[n] = round(e0.elapsed_time(e1) / 50, 4)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {n: {"ms_per_step_median": round(float(np.median(v)), 4), "ms_per_step_min": round(min(v), 4), "ms_per_step_max": round(max(v), 4)}
       for n, v in times.items()}
out["extra_ms_median"] = round(out["full_loss_refopts"]["ms_per_step_median"] - out["full_loss"]["ms_per_step_median"], 4)
out["stage_ms"] = stage
out.update(steps_per_window=K, windows=NWIN, gpu=q.splitlines()[0] if q else torch.cuda.get_device_name(0))
print(json.dumps(out))

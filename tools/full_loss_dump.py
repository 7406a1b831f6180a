#!/usr/bin/env python
"""Parameters after K seeded full-loss training steps (bench.py's full_loss workload: C2 + point-cloud and warped-RGB terms, the
reference-image stage on its side stream) run as the whole-step CUDA graph, written as .npy files like bench.py --dump-outputs.
Every reduction of the step runs in a fixed order, so two builds that compute the same write the same bits: compare two runs'
directories file by file.   python tools/full_loss_dump.py OUT_DIR [K]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import bench

out_dir = sys.argv[1]
K = int(sys.argv[2]) if len(sys.argv) > 2 else 20
dev = torch.device("cuda", 0); torch.cuda.set_device(0)
_, frames = bench.synth_frames(bench.H, bench.W, bench.HD, bench.WD, 4, bench.V, dev, with_ref=True)
tr = bench.build_trainer(bench.make_cfg(bench.NRAYS, full_loss=True), dev, bench.V)
assert tr.use_cuda_graph
for i in range(K):
    ld = tr.train_step(frames[i % 4], it=i, epoch=0, scheduling_start=10000, render_path=None)
assert any(g is not None and g.use_ref and g.graph is not None for g in tr._gsteps.values()), "the full-loss step was not captured"
bench.dump_outputs(out_dir, tr, ld)
print("wrote", len(os.listdir(out_dir)), "files to", out_dir)

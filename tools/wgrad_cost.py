#!/usr/bin/env python
"""Per-kernel cost of the weight-gradient stage in the eager C2 train step (1024 rays x 128 samples, D = 256): torch.profiler with CUDA
activities over PK steps, device time per step of tc_wgrad<KN>, tc_wgrad_piece<64>, head_wgrad (simt_wgrad in older builds) and
wgrad_reduce, and for the tensor-core kernels the achieved bytes/s and tensor FLOP/s from the job shapes.  bench.py and tools/step_time.py time the whole stage as one interval.  NNB_LIB_PATH selects a
library variant (alternate the runs of two builds to compare them).   python tools/wgrad_cost.py [tag]

The rgb_layers.0 pieces, the encoding jobs and the head jobs are chained behind tc_wgrad<256>, so the kernel times overlap and
"wgrad_ms_per_step", their sum, is not the stage time.  "timeline" gives, from the kernels' device timestamps, per step: the stage's
wall interval (start of the first weight-gradient kernel to the end of the last wgrad_reduce) and the start and end of
tc_wgrad_piece<64>, tc_wgrad<64> and the head kernel relative to the end of tc_wgrad<256> (negative: before it ends), as medians over
the PK steps and per step.  A chained grid cannot end before the grid it was launched behind (its last CTA waits for it), so an end at
about 0 means its work was done inside tc_wgrad<256>."""
import json, os, re, statistics, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import bench
from nope_nerf_b200 import _lib as L

PK = 10


def tc_shapes(M, D):
    """per tensor-core launch of tc_wgrad_all: (bytes of dY and X if each is read once, bytes as issued (every 128-row slice of a job
    reads its X, every 64-column piece its whole dY rows and its X columns), tensor FLOP: three bf16 MMAs per logical multiply-add)"""
    launches = {"tc_wgrad<%d>" % D: ([D] * 8, D, D, False, 1),   # dY widths (layers 1..7, fc_feature), X width, Kk, X shared, pieces
                "tc_wgrad_piece<64>": ([D // 2], D, D, False, D // 64),   # rgb_layers.0 in 64-column pieces
                "tc_wgrad<64>": ([D, D], 64, 63, True, 1)}                # layers 0 and 4: one shared X (the encoding stash)
    out = {}
    for name, (nns, ldx, kk, shared_x, pieces) in launches.items():
        once = sum(M * nn * 4 for nn in nns) + M * ldx * 4 * (1 if shared_x else len(nns))
        issued = sum(M * (nn * pieces + (nn + 127) // 128 * ldx) * 4 for nn in nns)
        out[name] = (once, issued, sum(3 * 2 * M * nn * kk for nn in nns))
    return out


def timeline(trace_path, D):
    """per-step intervals of the stage from a chrome trace of the profiled steps (see the module docstring)"""
    with open(trace_path) as f:
        evs = json.load(f)["traceEvents"]
    ks = sorted((e["ts"], e["ts"] + e["dur"], e["name"]) for e in evs if e.get("ph") == "X" and e.get("cat") == "kernel")
    pat = re.compile(r"(tc_wgrad<\d+>|tc_wgrad_piece<\d+>|simt_wgrad|head_wgrad|wgrad_reduce)")
    big = "tc_wgrad<%d>" % D
    steps = []
    for i, (t0, t1, name) in enumerate(ks):
        if pat.search(name) is None or pat.search(name).group(1) != big:
            continue
        stage = {}
        for s0, s1, n in ks[i:]:   # the stage: the weight-gradient kernels from this tc_wgrad<D> up to the next other kernel
            m = pat.search(n)
            if m is None or (s0 > t0 and m.group(1) == big):
                break
            stage.setdefault(m.group(1), []).append((s0, s1))
        step = {"wall_ms": (max(e for v in stage.values() for _, e in v) - t0) / 1e3, "big_ms": (t1 - t0) / 1e3}
        for k in ("tc_wgrad_piece<64>", "tc_wgrad<64>", "head_wgrad", "simt_wgrad"):
            if k in stage and k != big:
                step[k + "_start_ms"] = (stage[k][0][0] - t1) / 1e3
                step[k + "_end_ms"] = (stage[k][-1][1] - t1) / 1e3
        steps.append(step)
    med = {k: round(statistics.median(s[k] for s in steps), 4) for k in steps[0]} if steps else {}
    return {"median": med, "per_step": [{k: round(v, 4) for k, v in s.items()} for s in steps]}


def main():
    dev = torch.device("cuda", 0); torch.cuda.set_device(0)
    tr = bench.build_trainer(bench.make_cfg(bench.NRAYS), dev, bench.V)
    _, frames = bench.synth_frames(bench.H, bench.W, bench.HD, bench.WD, 4, bench.V, dev, with_ref=False)
    step = lambda i: tr.train_step(frames[i % 4], it=i, epoch=0, scheduling_start=10000, render_path=None)
    tr.use_cuda_graph = False
    for i in range(5): step(i)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for i in range(PK): step(i)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        tl = timeline(path, 256)
    pat = re.compile(r"(tc_wgrad<\d+>|tc_wgrad_piece<\d+>|simt_wgrad|head_wgrad|wgrad_reduce)")
    agg = {}
    for ev in prof.key_averages():
        m = pat.search(ev.key)
        if not m:
            continue
        t = getattr(ev, "device_time_total", None)
        if t is None: t = ev.cuda_time_total
        a = agg.setdefault(m.group(1), [0.0, 0])
        a[0] += t; a[1] += ev.count
    M, D = bench.NRAYS * bench.S, 256
    shapes = tc_shapes(M, D)
    kernels = {}
    for name, (us, n) in sorted(agg.items()):
        ms = us / 1e3 / PK
        k = {"ms_per_step": round(ms, 4), "launches_per_step": n / PK}
        if name in shapes:
            once, issued, flop = shapes[name]
            k.update(gb_read_once=round(once / 1e9, 3), gb_issued=round(issued / 1e9, 3), tb_per_s_once=round(once / ms / 1e9, 3),
                     tensor_tflop=round(flop / 1e12, 4), tensor_tflop_per_s=round(flop / ms / 1e9, 1))
        kernels[name] = k
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"tag": sys.argv[1] if len(sys.argv) > 1 else "", "lib": os.path.basename(L.LIB_PATH), "gpu": q.splitlines()[0] if q else "",
                      "steps": PK, "wgrad_ms_per_step": round(sum(v["ms_per_step"] for v in kernels.values()), 4), "kernels": kernels,
                      "timeline": tl}))


if __name__ == "__main__":
    main()

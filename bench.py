#!/usr/bin/env python
"""bench.py — train-step ray-samples/s of the NoPe-NeRF hot path (BASELINE.json metric).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--engine tc|simt] [--scaling weak|strong]
                    [--dump-outputs DIR]

Workload (BASELINE.json configs[1], SURVEY.md 8(d) "C2"): Ignatius-shape scene, 1080x1920 frames,
V=200 poses, 1024 rays x 128 samples per step, uniform sampling + stratified jitter, softplus
density, photometric L1 + DPT depth L1 losses ("coarse-only" = the reference's only mode), fp32
master weights, torch.optim.Adam x3 exactly as train.py builds them.  One "step" = one complete
Trainer.train_step: pose exp-map, ray generation, sampling, encoding, 8x256 MLP, compositing, losses,
full backward (MLP + pose + depth-distortion gradients), [all-reduce], optimizer steps.

  value : whole-job ray-samples/s over EXACTLY K timed steps with the frame + DPT map already resident in HBM (after W warm-up
          steps and SETTLE_STEPS untimed steps that let clocks and power settle).  Every other timed window is K steps too.
  e2e   : same step through the reference-facing API with HOST (page-locked) frame tensors, as train.py's DataLoader
          (pin_memory=True) hands them over: host->device traffic (DPT map copy + in-place gather of the sampled
          pixels over PCIe) and the D2H read of the loss every step (train.py:212) are inside the timed region.
  full_loss / c3 / fwd_only / reference_cuda (N = 1): the full default loss set (point-cloud chamfer + warped RGB, training.py:280-365),
          the LLFF-shape NDC + dist_alpha configuration, one 1/8 row block of a 1080p novel view (config 4), and the UNMODIFIED
          reference's Trainer.train_step on the same GPU (oracle/_ref, made by build() where the reference tree exists).
  N > 1 : weak scaling — every GPU keeps the C2 per-GPU work (1024 rays x 128 samples): the step draws a global batch of
          1024*N rays, sharded rank::N (Trainer dp_mode='rays'), ONE NCCL all-reduce of the flat [gradients | loss]
          buffer per step; value = all ranks' ray-samples / max-over-ranks time.  A `strong` record (the fixed 1024-ray batch
          split over the GPUs) is added to the same line.
  --impl reference : the UNMODIFIED reference's Trainer.train_step (oracle/_ref) on the host cores, full 1024 x 128 batch on the
          same synthetic C2 data, all host threads (rank 0 only under torchrun).
  --dump-outputs DIR : after the headline window, a second trainer built from the same seeds runs the same timed path (W warm-up
          + K steps on the same frames); the outputs of its last step go to DIR/<name>.npy (float32 / float64): the loss terms the
          step returned and every parameter it updated (MLP, poses, distortions).  Inputs, seeds and step counts are fixed by the
          arguments, and every reduction of the step runs in a fixed order (no float atomics), so two runs of one build write the
          same bits and two builds can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

H, W, HD, WD, V, NRAYS, S = 1080, 1920, 384, 672, 200, 1024, 128
N_FRAMES = 8                      # distinct synthetic frames cycled through (each 24.9 MB + 1 MB DPT map)
FLOP_PER_SAMPLE_STEP = 3560448    # fwd + dgrad + wgrad (BASELINE.md section 2)
FLOP_PER_SAMPLE_FWD = 1186816
SETTLE_STEPS = 300                # untimed steps before the headline window (about 2 s at 8 ms per step: clocks and power settle)
# H100 SXM data sheet, dense FP16 / BF16 tensor rate and HBM3 bandwidth at the 700 W limit: a ceiling, not a measured rate
PEAK = dict(tflops=989.0, hbm_gbs=3350.0, source="H100 SXM data sheet (dense fp16, 700 W); see clocks for this card's limit")


class ClockSampler:
    def __init__(self, idx):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
            "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        try:
            self.p = subprocess.Popen(["nvidia-smi", "-i", str(idx), "--query-gpu=" + q, "--format=csv,noheader,nounits", "-lms", "50"],
                                      stdout=self.f, stderr=subprocess.DEVNULL)
        except Exception:
            self.p = None

    def stop(self):
        out = dict(sm_mhz=None, sm_max_mhz=None, reasons=[])
        if self.p is None:
            return out
        self.p.terminate()
        try:
            self.p.wait(timeout=5)
        except Exception:
            self.p.kill()
        self.f.flush(); self.f.seek(0)
        rows = [l.strip().split(",") for l in self.f.read().splitlines() if l.count(",") >= 6]
        os.unlink(self.f.name)
        if not rows:
            return out
        import statistics
        sm = [float(r[0]) for r in rows if r[0].strip().replace(".", "").isdigit()]
        pw = [float(r[2]) for r in rows if r[2].strip().replace(".", "").isdigit()]
        out["sm_mhz"] = statistics.median(sm) if sm else None
        out["sm_max_mhz"] = float(rows[0][1])
        out["power_w_median"] = statistics.median(pw) if pw else None
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for i, nm in enumerate(names):
            if any("Active" == r[3 + i].strip() for r in rows):
                out["reasons"].append(nm)
        out["samples"] = len(rows)
        return out


def make_cfg(n_rays, full_loss=False, c3=False):
    from _cfg import default_cfg
    cfg = default_cfg()
    if not full_loss:
        cfg["training"]["pc_weight"] = [0.0, 0.0]; cfg["training"]["rgb_s_weight"] = [0.0, 0.0]   # render + rgb + depth losses
    if c3:
        cfg["rendering"].update(sample_option="ndc", dist_alpha=True, depth_range=[0.0, 1.0])
    cfg["training"]["n_training_points"] = n_rays; cfg["rendering"]["num_points"] = S
    return cfg


def synth_frames(h, w, hd, wd, n, v, dev, with_ref):
    """seeded synthetic frames (U[0,1) pixels, DPT-range depth 0.6..7.2), page-locked host copies + device copies"""
    import torch
    g = torch.Generator().manual_seed(42)
    fx = 0.6 * w
    cam = torch.tensor([[2 * fx / w, 0, 0, 0], [0, -2 * fx / h, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
    raw = []
    pin = (lambda t: t.pin_memory()) if torch.cuda.is_available() else (lambda t: t)
    for f in range(n):
        raw.append((pin(torch.rand(1, 3, h, w, generator=g)), pin(torch.rand(1, hd, wd, generator=g) * 6.6 + 0.6)))
    host, devd = [], []
    dimg = [(a.to(dev), b.to(dev)) for a, b in raw] if dev is not None else None
    for f in range(n):
        idx = f * (v // n)
        d = {"img": raw[f][0], "img.idx": torch.tensor([idx]), "img.dpt": raw[f][1], "img.camera_mat": cam, "img.scale_mat": torch.eye(4)[None]}
        if with_ref:
            r = (f + 1) % n
            d.update({"img.ref_imgs": raw[r][0], "img.ref_dpts": raw[r][1], "img.ref_idxs": torch.tensor([idx + 1])})
        host.append(d)
        if dev is not None:
            dd = dict(d); dd["img"] = dimg[f][0]; dd["img.dpt"] = dimg[f][1]
            if with_ref:
                dd["img.ref_imgs"] = dimg[(f + 1) % n][0]; dd["img.ref_dpts"] = dimg[(f + 1) % n][1]
            devd.append(dd)
    return host, devd


def build_trainer(cfg, dev, v, dp_mode="rays"):
    import numpy as np
    import torch
    import nope_nerf_b200.model as mdl
    np.random.seed(42); torch.manual_seed(42)                     # train.py:22-23
    net = mdl.OfficialStaticNerf(cfg)
    rend = mdl.Renderer(net, cfg["rendering"], device=dev)
    model = mdl.get_model(rend, cfg, device=dev)
    pose = mdl.LearnPose(v, True, True, cfg).to(dev)
    dnet = mdl.Learn_Distortion(v, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.normal_(0, 0.05); pose.t.normal_(0, 0.05)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=0.0)          # train.py:58
    opt_p = torch.optim.Adam(pose.parameters(), lr=5e-4)                           # train.py:99
    opt_d = torch.optim.Adam(dnet.parameters(), lr=5e-4)                           # train.py:117
    return mdl.Trainer(model, opt, cfg["training"], device=dev, optimizer_pose=opt_p, pose_param_net=pose,
                       optimizer_distortion=opt_d, distortion_net=dnet, cfg_all=cfg, dp_mode=dp_mode, keep_graph=True)


# ------------------------------------------------------------------------------------------------
def run_ours(args):
    import torch
    import torch.distributed as dist
    rank = int(os.environ.get("RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1)); local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from nope_nerf_b200 import ops, _lib as L         # the library build() made; this script writes nothing into the tree
    ops.set_default_engine(args.engine)
    weak = args.scaling == "weak"
    n_local = NRAYS if weak else NRAYS // world
    trainer = build_trainer(make_cfg(n_local * world), dev, V)
    host, devd = synth_frames(H, W, HD, WD, N_FRAMES, V, dev, with_ref=False)

    def step(tr, data, it):
        return tr.train_step(data, it=it, epoch=0, scheduling_start=10000, render_path=None)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(tr, datas, K, Wm, sync_loss, settle=0):
        for i in range(Wm + settle):                        # warm-up, then untimed steps while clocks / power settle
            ld = step(tr, datas[i % len(datas)], i)
            if sync_loss and i < Wm: ld["loss"].item()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(K):
            ld = step(tr, datas[i % len(datas)], Wm + i)
            if sync_loss: ld["loss"].item()                           # train.py:212-214 reads the loss every step
        e1.record()
        barrier()
        ms = e0.elapsed_time(e1)
        t = torch.tensor([ms], device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.item(), ld

    K, Wm = args.steps, max(args.warmup, 3)
    # ---- profiled pass (events between the library's kernels; not part of the headline timing) ----
    import ctypes as C
    prof = {}
    graph_mode = trainer.use_cuda_graph
    trainer.use_cuda_graph = False                          # the profiled pass launches the same kernel sequence eagerly
    for i in range(3): step(trainer, devd[i % N_FRAMES], i)          # every rank takes part (the step all-reduces when world > 1)
    PK = 10
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(9 * PK)]
    for e in evs: e.record()
    torch.cuda.synchronize()
    arr = (C.c_void_p * len(evs))(*[e.cuda_event for e in evs])
    L.lib.nnb_profile_events(arr, len(evs))
    for i in range(PK): step(trainer, devd[i % N_FRAMES], i)
    torch.cuda.synchronize()
    L.lib.nnb_profile_events(None, 0)
    trainer.use_cuda_graph = graph_mode
    if rank == 0:
        names = ["weight_image", "field_fwd", "composite_fwd", None, "composite_bwd", "dgrad", "wgrad", "ray_bwd"]
        acc = {n: 0.0 for n in names if n}
        for s_ in range(PK):
            for j, n in enumerate(names):
                if n: acc[n] += evs[9 * s_ + j].elapsed_time(evs[9 * s_ + j + 1])
        prof = {n: v / PK for n, v in acc.items()}
    if world > 1:
        dist.barrier()
    # ---- headline: device-resident inputs, EXACTLY K timed steps after warm-up + settling ----
    cs = ClockSampler(local) if rank == 0 else None
    ms_burst, _ = timed(trainer, devd, K, Wm, sync_loss=False)               # right after warm-up: boost clocks (round-1 methodology)
    ms, ld = timed(trainer, devd, K, 0, sync_loss=False, settle=SETTLE_STEPS)  # headline: after the untimed settling steps
    if args.dump_outputs:
        # a second trainer from the same seeds runs the same timed path (W warm-up + K steps on the same frames): the dumped step
        # is W + K steps from a fixed start, so rounding differences between builds have had few Adam steps to grow
        tr_d = build_trainer(make_cfg(n_local * world), dev, V)
        _, ld_d = timed(tr_d, devd, K, Wm, sync_loss=False)
        if rank == 0:
            dump_outputs(args.dump_outputs, tr_d, ld_d)
        del tr_d
    ms_sus, _ = timed(trainer, devd, K, 0, sync_loss=False)
    clocks = cs.stop() if cs else {}
    launches = trainer.graph_kernel_nodes()
    # ---- e2e: host (pinned) frames, H2D inside the step, loss read back every step ----
    ms_e2e, _ = timed(trainer, host, K, max(Wm, N_FRAMES), sync_loss=True)   # warm-up touches every page-locked frame once (first-touch mapping)
    ms_e2e_sus, _ = timed(trainer, host, K, 0, sync_loss=True)
    ms_dev_item, _ = timed(trainer, devd, K, 0, sync_loss=True)             # breakdown: loss read-back alone
    ms_host_noitem, _ = timed(trainer, host, K, 0, sync_loss=False)         # breakdown: host frames alone
    extra = {}
    if world > 1 and weak:
        # strong scaling of the SAME 1024-ray batch (north_star): second trainer, rays split rank::world
        tr_s = build_trainer(make_cfg(NRAYS), dev, V)
        ms_s, _ = timed(tr_s, devd, K, 5, sync_loss=False)
        extra["strong"] = {"value": round(NRAYS * S * K / (ms_s / 1e3), 1), "unit": "ray-samples/s", "ms_per_step": round(ms_s / K, 4),
                           "global_rays": NRAYS, "rays_per_gpu": NRAYS // world, "steps": K}
        del tr_s
    if world > 1 and weak:
        # C5 (BASELINE.json configs[4]): 4096 rays x 128 samples over the GPUs, one view per rank, full default loss set, one exchange
        ops_c5 = make_cfg(4096 // world, full_loss=True)
        tr_c = build_trainer(ops_c5, dev, V, dp_mode="views")
        hostf, devf = synth_frames(H, W, HD, WD, 2 * world, V, dev, with_ref=True)
        mine = [devf[(2 * k + rank) % len(devf)] for k in range(2)]
        ms_c, ldc = timed(tr_c, mine, K, 5, sync_loss=False)
        extra["c5"] = {"value": round(4096 * S * K / (ms_c / 1e3), 1), "unit": "ray-samples/s", "ms_per_step": round(ms_c / K, 4), "global_rays": 4096,
                       "rays_per_gpu": 4096 // world, "steps": K,
                       "workload": "C5: 4096 rays x 128 samples, dp_mode='views' (one view per rank), rgb + depth + point-cloud + warped-RGB losses"}
        del tr_c, hostf, devf
    if world == 1:
        extra.update(single_gpu_records(dev, step, timed, args))
    if rank == 0:
        pk = PEAK
        samples_per_step = n_local * world * S
        value = samples_per_step * K / (ms / 1e3)
        e2e = samples_per_step * K / (ms_e2e / 1e3)
        # roofline of the dominant kernel (largest average duration in the profiled pass)
        flops = {"field_fwd": FLOP_PER_SAMPLE_FWD, "dgrad": FLOP_PER_SAMPLE_FWD, "wgrad": FLOP_PER_SAMPLE_FWD}
        dom = max((k for k in prof if k in flops), key=lambda k: prof[k]) if prof else None
        roof = None
        if dom:
            ach = flops[dom] * (n_local * S) / (prof[dom] / 1e3) / 1e12
            roof = {"bound": "tensor", "kernel": dom, "achieved": round(ach, 2), "peak": pk["tflops"], "unit": "TFLOP/s",
                    "frac": round(ach / pk["tflops"], 4), "peak_source": pk["source"], "algorithmic_flop_per_launch": flops[dom] * n_local * S,
                    "kernel_ms": {k: round(v, 4) for k, v in prof.items()},
                    "step_algorithmic_tflops": round(FLOP_PER_SAMPLE_STEP * n_local * S / (ms_sus / K / 1e3) / 1e12, 1),
                    "note": "algorithmic fp32-equivalent FLOPs; the tensor-core forward issues three split-fp16 wgmma per logical product"}
        line = {"metric": "train-step ray-samples/sec", "value": round(value, 1), "unit": "ray-samples/s", "n_gpus": world, "steps": K,
                "warmup": Wm, "ms_per_step": round(ms / K, 4), "higher_is_better": True, "scaling": "weak" if weak else "strong", "vs_baseline": None,
                "dtype": "fp32 (split fp16 hi+lo wgmma forward, split bf16 hi+lo wgmma backward, fp32 accumulate)" if args.engine == "tc" else "fp32",
                "data": "synthetic",
                "config": {"workload": "C2 Ignatius-shape 1080x1920, V=200, 1024 rays x 128 samples, uniform+jitter, rgb L1 + depth L1, Adam x3",
                           "global_rays": n_local * world, "rays_per_gpu": n_local, "samples_per_ray": S,
                           "parallelism": "dp%d (ray shards, 1 all-reduce)" % world,
                           "engine": args.engine, "frames_resident": N_FRAMES, "cuda_graph": bool(trainer.use_cuda_graph),
                           "l2_policy": "no flush: each step streams a >1 GB activation stash, far larger than the 50 MB L2",
                           "settle": "W warm-up steps + %d untimed steps before the K timed steps" % SETTLE_STEPS},
                "sustained": {"steps": K, "ms_per_step": round(ms_sus / K, 4), "value": round(samples_per_step * K / (ms_sus / 1e3), 1),
                              "note": "the next K steps, right after the headline window"},
                "burst": {"steps": K, "ms_per_step": round(ms_burst / K, 4), "value": round(samples_per_step * K / (ms_burst / 1e3), 1),
                          "note": "K steps timed right after the W warm-up steps, before clocks / power settle (how round 1 measured)"},
                "e2e": {"value": round(e2e, 1), "unit": "ray-samples/s", "ms_per_step": round(ms_e2e / K, 4),
                        "h2d_bytes_per_step": int(n_local * 3 * 32 + HD * WD * 4 + 64 + 16) * world, "d2h_bytes_per_step": 4 * world,
                        "sustained_ms_per_step": round(ms_e2e_sus / K, 4),
                        "breakdown_ms_per_step": {"device_frames_no_readback": round(ms_sus / K, 4), "device_frames_loss_item": round(ms_dev_item / K, 4),
                                                  "host_frames_no_readback": round(ms_host_noitem / K, 4), "host_frames_loss_item": round(ms_e2e_sus / K, 4)},
                        "h2d_note": "host frames are page-locked: the loss kernel gathers the 1024x3 sampled pixels in place over PCIe "
                                    "(one 32-B sector each) instead of copying the 24.9 MB frame; the 1 MB DPT map, camera_mat and idx are copied"},
                "gpu_launches": (launches["kernels"] if launches else 22) * K * world,
                "gpu_launches_note": ("kernel nodes of the captured step graph (cudaGraphGetNodes): %s" % launches) if launches else
                                     "static count (graph introspection unavailable)",
                "clocks": clocks, "roofline": roof, "loss": float(ld["loss"].item()), "impl": "ours"}
        line.update(extra)
        if world == 1 and not args.no_cpu_baseline:
            line["cpu_baseline"] = cpu_reference(steps=3, warm=1, budget_s=60.0)
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def single_gpu_records(dev, step, timed, args):
    """N = 1 extras: full default loss set, C3 (NDC + dist_alpha), forward-only row block (config 4), the reference on this GPU"""
    import torch
    from nope_nerf_b200 import ops
    out = {}
    # ---- full loss set: point-cloud chamfer (P = 96 x 168 = 16 128) + warped-RGB terms, training.py:280-365 ----
    tr_f = build_trainer(make_cfg(NRAYS, full_loss=True), dev, V)
    hostf, devf = synth_frames(H, W, HD, WD, 4, V, dev, with_ref=True)
    K = args.steps
    ms_f, ld = timed(tr_f, devf, K, 5, sync_loss=False)
    P = (HD // 4) * (WD // 4)
    X = torch.randn(P, 3, device=dev); Y = torch.randn(P, 3, device=dev) + 0.05
    keys = torch.empty(2 * P, dtype=torch.int64, device=dev); loss = torch.zeros(1, device=dev)
    from nope_nerf_b200 import _lib as L
    import ctypes as C
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for _ in range(3): L.lib.nnb_chamfer(L.ptr(X), P, L.ptr(Y), P, L.ptr(keys), None, None, L.ptr(loss), 1.0, None, None, st)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20): L.lib.nnb_chamfer(L.ptr(X), P, L.ptr(Y), P, L.ptr(keys), None, None, L.ptr(loss), 1.0, None, None, st)
    e1.record(); torch.cuda.synchronize()
    ch_ms = e0.elapsed_time(e1) / 20
    out["full_loss"] = {"ms_per_step": round(ms_f / K, 4), "value": round(NRAYS * S * K / (ms_f / 1e3), 1), "steps": K,
                        "loss_pc": float(ld["loss_pc"]), "loss_rgb_s": float(ld["loss_rgb_s"]), "points_per_cloud": P,
                        "chamfer_ms": round(ch_ms, 4), "chamfer_pairs_per_s": round(2.0 * P * P / (ch_ms / 1e3), 1),
                        "chamfer_note": "brute force, both directions in one launch: 2*P*P fp32 pair distances (SIMT)",
                        "workload": "C2 + pc_weight = rgb_s_weight = 1 (configs/default.yaml:95-101 before annealing), captured in the same CUDA graph"}
    del tr_f, hostf, devf
    torch.cuda.empty_cache()
    # ---- C3: LLFF fern shape, NDC + dist_alpha, depth loss on 1 - 1/d ----
    tr_c = build_trainer(make_cfg(NRAYS, c3=True), dev, 20)
    _, devc = synth_frames(756, 1008, 384, 512, 4, 20, dev, with_ref=False)
    ms_c, _ = timed(tr_c, devc, K, 5, sync_loss=False)
    out["c3"] = {"ms_per_step": round(ms_c / K, 4), "value": round(NRAYS * S * K / (ms_c / 1e3), 1), "steps": K,
                 "workload": "C3 fern shape 756x1008, V=20, 1024 rays x 128 samples, NDC + dist_alpha (single 128-sample pass: the reference has no hierarchical sampling)"}
    del tr_c, devc
    # ---- config 4: one 1/8 row block of a 1080x1920 novel view, forward only ----
    import nope_nerf_b200.model as mdl
    cfg = make_cfg(NRAYS); cfg["extract_images"] = {"resolution": (H, W)}
    net = mdl.OfficialStaticNerf(cfg); rend = mdl.Renderer(net, cfg["rendering"], device=dev)
    ex = mdl.Extract_Images(rend, cfg, device=dev, render_type="nope_nerf")
    c2w = torch.eye(4, device=dev); fx = 0.6 * W
    cam = torch.diag(torch.tensor([2 * fx / W, -2 * fx / H, -1.0, 1.0])).to(dev)
    rows = (0, H // 8)
    ex.render_frame(c2w, cam, H, W, rows=rows); torch.cuda.synchronize()
    e0.record()
    for _ in range(3): ex.render_frame(c2w, cam, H, W, rows=rows)
    e1.record(); torch.cuda.synchronize()
    ms_b = e0.elapsed_time(e1) / 3
    nr = (rows[1] - rows[0]) * W
    out["fwd_only"] = {"ms_per_row_block": round(ms_b, 3), "rays": nr, "value": round(nr * S / (ms_b / 1e3), 1), "unit": "ray-samples/s",
                       "frames_per_s_8gpu_est": round(1e3 / ms_b, 3),
                       "workload": "config 4: rows %d..%d of one 1080x1920 view x 128 samples, eval mode, prior = ones (Extract_Images.render_frame); "
                                   "8 GPUs render the 8 row blocks of a frame concurrently, no collective" % rows}
    # ---- the UNMODIFIED reference on this GPU (oracle/_ref): same C2 step ----
    out["reference_cuda"] = reference_on_device("cuda", steps=10, warm=3, budget_s=60.0)
    return out


def dump_outputs(out_dir, trainer, ld):
    """the last step's loss terms and the parameters it updated, as float32 (parameters) / float64 (losses) .npy files"""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    for k, v in ld.items():
        if torch.is_tensor(v) or isinstance(v, (int, float)):
            np.save(os.path.join(out_dir, "loss_%s.npy" % k), np.asarray(torch.as_tensor(v).detach().double().cpu().numpy()))
    mods = {"mlp": trainer.model, "pose": trainer.pose_param_net, "distortion": trainer.distortion_net}
    for mn, mod in mods.items():
        if mod is None:
            continue
        for pn, p in mod.named_parameters():
            np.save(os.path.join(out_dir, "%s.%s.npy" % (mn, pn)), p.detach().float().cpu().numpy())


# ------------------------------------------------------------------------------------------------
def reference_on_device(device, steps, warm, budget_s):
    """Trainer.train_step of the UNMODIFIED reference (oracle/_ref) on the C2 workload at the full 1024 x 128 batch"""
    import torch
    from oracle import ref_harness as RH
    if not RH.available():
        return {"unavailable": "oracle/_ref missing (oracle/vendor_ref.py copies a reference checkout there)"}
    cfg = RH.load_default_cfg()
    RH.set_cfg(cfg, {"training.pc_weight": [0.0, 0.0], "training.rgb_s_weight": [0.0, 0.0], "training.n_training_points": NRAYS,
                     "rendering.num_points": S, "training.vis_reprojection_every": 10 ** 9})
    import numpy as np
    np.random.seed(42); torch.manual_seed(42)
    rig = RH.RefRig(cfg, V, device)
    with torch.no_grad():
        rig.pose.r.normal_(0, 0.05); rig.pose.t.normal_(0, 0.05)
    host, _ = synth_frames(H, W, HD, WD, 2, V, None, with_ref=False)
    ts = []
    t_start = time.perf_counter()
    for i in range(warm + steps):
        if device != "cpu": torch.cuda.synchronize()
        t0 = time.perf_counter()
        ld = rig.train_step(host[i % 2], it=i + 1)
        float(ld["loss"].detach())                              # train.py:212 reads the loss every step
        if device != "cpu": torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
        if i == 0 and ts[0] > budget_s / 4:
            warm = 1                                            # very slow host: one warm-up step has to do
        if i >= warm and time.perf_counter() - t_start + ts[-1] > budget_s:
            break                                               # bounded run: at least one timed step, then stop inside the budget
    ts = sorted(ts[warm:])
    med = ts[len(ts) // 2]
    return {"value": round(NRAYS * S / med, 1), "unit": "ray-samples/s", "sec_per_step": round(med, 4), "steps_timed": len(ts),
            "kind": "reference", "device": device, "loss": float(ld["loss"].detach()),
            "sample": "unmodified reference Trainer.train_step (oracle/_ref), full 1024 rays x 128 samples per step on 1080x1920 host frames "
                      "(the reference copies the frame to the device every step), median of %d timed steps after %d warm-up" % (len(ts), warm)}


def cpu_reference(steps, warm, budget_s):
    import torch
    # intra-op threads: all cores up to 32 -- on the 128-core GPU box the reference's step (thousands of small ATen ops) measured 59.6 s
    # with 128 threads (r2 run 2); NNB_REF_THREADS overrides
    torch.set_num_threads(int(os.environ.get("NNB_REF_THREADS", min(os.cpu_count() or 1, 32))))
    from oracle import ref_harness as RH
    if RH.available():
        r = reference_on_device("cpu", steps, warm, budget_s)
        r["cores"] = torch.get_num_threads()
        return r
    # no vendored reference on this box: numpy port of the same step (oracle/nerf_oracle.py), bounded sample
    import numpy as np
    from oracle import nerf_oracle as O
    rng = np.random.default_rng(42)
    cfg = dict(O.DEFAULT_CFG); cfg["num_points"] = S
    state = dict(P=O.init_params(seed=42), r=rng.normal(0, .05, (V, 3)).astype(np.float32), t=rng.normal(0, .05, (V, 3)).astype(np.float32),
                 scales=np.ones((V, 1), np.float32), shifts=np.zeros((V, 1), np.float32))
    img = rng.uniform(0, 1, (3, H, W)).astype(np.float32); dpt = rng.uniform(.6, 7.2, (HD, WD)).astype(np.float32)
    fx = 0.6 * W; sample_rays = 256
    ts = []
    for i in range(1 + 2):
        ray_idx = rng.permutation(H * W)[:sample_rays]; noise = rng.uniform(0, 1, (sample_rays, S)).astype(np.float32)
        t0 = time.perf_counter()
        O.train_step(state, img, dpt, ray_idx, noise, 3, 2 * fx / W, -2 * fx / H, cfg)
        ts.append(time.perf_counter() - t0)
    sec = sorted(ts[1:])[0]
    return {"value": round(sample_rays * S / sec, 1), "unit": "ray-samples/s", "cores": os.cpu_count(), "kind": "port",
            "sample": "numpy port, %d rays x %d samples per step (1/%d of the batch)" % (sample_rays, S, NRAYS // sample_rays), "sec_per_step": round(sec, 3)}


def run_reference(args):
    rank = int(os.environ.get("RANK", 0))
    if rank != 0:
        return
    # torchrun pins OMP_NUM_THREADS=1 for its workers: the reference arm is ONE process that should use every host core
    n = int(os.environ.get("NNB_REF_THREADS", min(os.cpu_count() or 1, 32)))
    os.environ["OMP_NUM_THREADS"] = str(n); os.environ["MKL_NUM_THREADS"] = str(n)
    K, Wm = args.steps, args.warmup
    cb = cpu_reference(steps=K, warm=max(1, min(Wm, 2)), budget_s=150.0)
    line = {"metric": "train-step ray-samples/sec", "value": cb["value"], "unit": "ray-samples/s", "n_gpus": args.gpus, "steps": K, "warmup": Wm,
            "ms_per_step": round(cb["sec_per_step"] * 1e3, 2), "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "fp32",
            "data": "synthetic", "impl": "reference",
            "config": {"workload": "C2 Ignatius-shape 1080x1920, V=200, 1024 rays x 128 samples, uniform+jitter, rgb L1 + depth L1, Adam x3",
                       "global_rays": NRAYS, "samples_per_ray": S,
                       "note": "the reference's own Trainer.train_step on the host cores (oracle/_ref = unmodified copy of the reference tree); "
                               "steps_timed may be smaller than K: the run is bounded to ~150 s"},
            "cpu_baseline": cb, "e2e": {"value": cb["value"], "unit": "ray-samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--engine", default="tc", choices=["tc", "simt"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last step of the timed path (W warm-up + K steps from the seeded start) to DIR/<name>.npy")
    ap.add_argument("--scaling", default="weak", choices=["weak", "strong"],
                    help="N > 1: weak = 1024 rays per GPU (global batch 1024*N), strong = the 1024-ray batch split over the GPUs")
    a = ap.parse_args()
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)

"""Cost of Trainer(frame_grad=True): the captured training step with the differentiable frame's training pair (FrameRenderCall:
nnb_render_frame_train_fwd + nnb_render_frame_train_bwd) against the default step (nnb_render_fwd with NNB_STASH + nnb_render_bwd).
Shapes: the C2 step (1024 rays x 128 samples, bench.py's render-only configuration and frames) and N = 4096, S = 512, D = 256.
  * Trainer graph steps: one Trainer per path, steps alternated between the two over --rounds rounds of --steps steps each, median ms per
    step; the peak torch.cuda.max_memory_allocated over each Trainer's build and warm-up, above what was allocated before it.
  * The ops-level pair: FrameRenderCall + backward against render_frame_engine + nnb_render_frame_bwd (ops.render_frame_bwd), which
    evaluates the field once more, same inputs, alternated, median.
--engine simt compares Trainer(frame_grad=True, frame_grad_engine='simt') (ExactFrameRenderCall) with the default step on the exact-fp32
engine, at the C2 step and at S = 8, below the tensor-core range, and the ops-level pair on that engine.
--t-min t (tensor-core engine) adds Trainer(frame_grad=True, frame_grad_t_min=t) to the alternated graph steps, with the mean n_eval of
its training render, and replaces the ops-level comparison by the _tmin pair (ops.frame_render_call(t)) against the t_min = 0 pair on
three fields: the seeded surface field (both shapes), and test_gpu_render_frame_local's scattered (s256: 301 x 256) and translucent
(t100: 1024 x 100) plants at their own sizes.
The card's name and power limit are read in the same run (nvidia-smi query, read-only).  Without a CUDA device the tool fails."""
import argparse, gc, json, os, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from field_query_cost import card  # noqa: E402

SHAPES = {"tc": ((1024, 128), (4096, 512)), "simt": ((1024, 128), (1024, 8))}
FRAME_KW = {"tc": dict(frame_grad=True), "simt": dict(frame_grad=True, frame_grad_engine="simt")}


def build(N, S, frame_grad, dev, engine="tc", t_min=None):
    import bench
    import nope_nerf_b200.model as mdl
    cfg = bench.make_cfg(N)
    cfg["rendering"]["num_points"] = S
    np.random.seed(42); torch.manual_seed(42)
    net = mdl.OfficialStaticNerf(cfg)
    model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
    pose = mdl.LearnPose(bench.V, True, True, cfg).to(dev); dnet = mdl.Learn_Distortion(bench.V, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.normal_(0, 0.05); pose.t.normal_(0, 0.05)
    return mdl.Trainer(model, torch.optim.Adam(model.parameters(), lr=1e-3), cfg["training"], device=dev,
                       optimizer_pose=torch.optim.Adam(pose.parameters(), lr=5e-4), pose_param_net=pose,
                       optimizer_distortion=torch.optim.Adam(dnet.parameters(), lr=5e-4), distortion_net=dnet,
                       **(dict(FRAME_KW[engine], **({} if t_min is None else dict(frame_grad_t_min=t_min))) if frame_grad else {}))


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record(); e1.synchronize()
    return e0.elapsed_time(e1) / n


def trainer_steps(N, S, frames, rounds, steps, dev, engine="tc", t_min=None):
    trainers, peak, calls = {}, {}, []
    paths = (("stash", False, None), ("frame", True, None)) + ((("frame_tmin", True, t_min),) if t_min is not None else ())
    for key, fg, t in paths:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(); torch.cuda.reset_peak_memory_stats()
        tr = build(N, S, fg, dev, engine, t)
        if t is not None:   # keep the training renders' calls: the captured one's n_eval is rewritten by every replay
            from nope_nerf_b200 import ops
            base_call = ops.frame_render_call(t)
            rec = type("Recorded", (base_call,), {"__init__": lambda self, *a, **k: (calls.append(self), base_call.__init__(self, *a, **k))[1]})
            tr._train_render_call = lambda backward, rec=rec: rec if backward else ops.RenderCall
        for i in range(3):                                   # eager warm-up, capture, first replay
            tr.train_step(frames[i % len(frames)], it=i, epoch=0, scheduling_start=10000, render_path=None)
        torch.cuda.synchronize()
        peak[key] = torch.cuda.max_memory_allocated() - base
        trainers[key] = tr
    assert all(len([v for v in tr._gsteps.values() if v]) == 1 for tr in trainers.values()), "the graph step did not run"
    times = {k: [] for k in trainers}
    order = list(trainers)
    for r in range(rounds):
        for key in (order if r % 2 == 0 else order[::-1]):
            tr = trainers[key]
            times[key].append(timed(lambda i: tr.train_step(frames[i % len(frames)], it=i, epoch=0, scheduling_start=10000, render_path=None),
                                    steps))
    n_eval = None
    if calls:   # mean n_eval over `steps` untimed steps after the timed rounds (the field changes as it trains)
        tr, vals = trainers["frame_tmin"], []
        for i in range(steps):
            tr.train_step(frames[i % len(frames)], it=i, epoch=0, scheduling_start=10000, render_path=None)
            vals.append(float(calls[-1].n_eval.float().mean()))
        n_eval = dict(mean=float(np.mean(vals)), min=float(np.min(vals)), max=float(np.max(vals)))
    del trainers, calls
    gc.collect(); torch.cuda.empty_cache()
    return {k: float(np.median(v)) for k, v in times.items()}, peak, n_eval


def ops_pair_tmin(fields, t_min, rounds):
    """the _tmin pair against the t_min = 0 pair, alternated, median ms; fields: name -> (flat, c2w, cam, kw, g_rgb)"""
    from nope_nerf_b200 import ops, _lib as L
    out = {}
    for name, (flat, c2w, cam, kw, g_rgb) in fields.items():
        N, D = kw["N"], kw["hidden_dim"]
        zeros = torch.zeros(N, device="cuda")
        g_w = torch.zeros(L.num_params(D), device="cuda"); g_c = torch.zeros(4, 4, device="cuda")
        last = {}

        def run(cls):
            def fn(_):
                call = cls(flat, c2w, cam, engine=None, **kw)
                last[cls] = call
                call.backward(g_rgb, zeros, zeros, g_w, g_c)
            return fn
        tmin, plain = run(ops.frame_render_call(t_min)), run(ops.FrameRenderCall)
        for fn in (tmin, plain):
            fn(0); fn(0)
        torch.cuda.synchronize()
        n_eval = float(last[ops.frame_render_call(t_min)].n_eval.float().mean())
        times = {"tmin": [], "t0": []}
        for r in range(rounds):
            for key, fn in (("tmin", tmin), ("t0", plain)) if r % 2 == 0 else (("t0", plain), ("tmin", tmin)):
                times[key].append(timed(fn, 1))
        m = {k: float(np.median(v)) for k, v in times.items()}
        out[name] = dict(N=N, S=kw["S"], tmin_ms=m["tmin"], t0_ms=m["t0"], ratio=m["tmin"] / m["t0"], mean_n_eval=n_eval)
        print("ops pair %s (N=%d S=%d): t_min=%g %.2f ms, t_min=0 %.2f ms (x%.2f), mean n_eval %.1f"
              % (name, N, kw["S"], t_min, m["tmin"], m["t0"], m["tmin"] / m["t0"], n_eval), file=sys.stderr, flush=True)
    ops._pool.free.clear(); torch.cuda.empty_cache()
    return out


def seeded_field(N, S, D):
    from nope_nerf_b200 import ops
    from oracle import nerf_oracle as O
    rng = np.random.default_rng(0)
    cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    flat = cu(O.flatten_params(O.init_params(seed=7, D=D, hf_damp=True)))
    c2w = cu(O.make_c2w(np.array([0.02, -0.03, 0.01], np.float32), np.array([0.05, 0.0, -0.04], np.float32)))
    cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0])).cuda()
    H, W = 270, 480
    kw = dict(N=N, S=S, flags=ops.flags_from_cfg(dict(O.DEFAULT_CFG), "softplus"), near=0.01, far=10.0,
              ray_idx=cu(rng.permutation(H * W)[:N].astype(np.int64)), depth_map=cu(rng.uniform(0.6, 7.2, (48, 64)).astype(np.float32)),
              scale=torch.tensor([1.05]).cuda(), shift=torch.tensor([0.02]).cuda(), H=H, W=W, hidden_dim=D)
    return flat, c2w, cam, kw, cu(rng.normal(0, 1, (N, 3)).astype(np.float32))


def planted_field(name):
    import test_gpu_render_frame_local as FL
    from oracle import nerf_oracle as O
    P, inp, flags, D = FL.planted(name)
    return (FL._cu(O.flatten_params(P)), FL._cu(inp["c2w"]), FL._cu(inp["cam"]), FL._call_kw(inp, flags, D), FL._cu(inp["g_rgb"]))


def ops_pair(N, S, D, rounds, engine="tc"):
    from nope_nerf_b200 import ops, _lib as L
    from oracle import nerf_oracle as O
    rng = np.random.default_rng(0)
    cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    flat = cu(O.flatten_params(O.init_params(seed=7, D=D, hf_damp=True)))
    c2w = cu(O.make_c2w(np.array([0.02, -0.03, 0.01], np.float32), np.array([0.05, 0.0, -0.04], np.float32)))
    cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0])).cuda()
    H, W = 270, 480
    kw = dict(N=N, S=S, flags=ops.flags_from_cfg(dict(O.DEFAULT_CFG), "softplus"), near=0.01, far=10.0,
              ray_idx=cu(rng.permutation(H * W)[:N].astype(np.int64)), depth_map=cu(rng.uniform(0.6, 7.2, (48, 64)).astype(np.float32)),
              scale=torch.tensor([1.05]).cuda(), shift=torch.tensor([0.02]).cuda(), H=H, W=W, hidden_dim=D)
    g_rgb, g_dp, g_dg = cu(rng.normal(0, 1, (N, 3)).astype(np.float32)), torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    g_w = torch.zeros(L.num_params(D), device="cuda"); g_c = torch.zeros(4, 4, device="cuda")

    exact = engine == "simt"
    eng = L.ENGINE_SIMT if exact else L.ENGINE_TC

    def pair(_):
        call = (ops.ExactFrameRenderCall if exact else ops.FrameRenderCall)(flat, c2w, cam, engine=None, **kw)
        call.backward(g_rgb, g_dp, g_dg, g_w, g_c)

    def one_call(_):
        ops.render_frame_engine(flat, c2w, cam, engine=eng, **kw)
        ops.render_frame_bwd(flat, c2w, cam, g_rgb, g_dp, g_dg, g_w, g_c, engine=eng, **kw)

    for fn in (pair, one_call):
        fn(0); fn(0)
    torch.cuda.synchronize()
    times = {"pair": [], "fwd_plus_frame_bwd": []}
    for r in range(rounds):
        for key, fn in (("pair", pair), ("fwd_plus_frame_bwd", one_call)) if r % 2 == 0 else (("fwd_plus_frame_bwd", one_call), ("pair", pair)):
            times[key].append(timed(fn, 1))
    ops._pool.free.clear(); torch.cuda.empty_cache()
    return {k: float(np.median(v)) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20, help="graph steps per timed round")
    ap.add_argument("--engine", choices=("tc", "simt"), default="tc")
    ap.add_argument("--t-min", type=float, default=None, help="also time Trainer(frame_grad_t_min=t) and the _tmin ops pair")
    args = ap.parse_args()
    if args.t_min is not None and args.engine != "tc":
        sys.exit("train_frame_cost: --t-min runs on the tensor-core engine only")
    if not torch.cuda.is_available():
        sys.exit("train_frame_cost: needs a CUDA device (there is no CPU path and a CPU timing would say nothing about the GPU)")
    import bench
    from nope_nerf_b200 import ops, _lib as L
    ops.set_default_engine(args.engine)   # the engine of the default step
    dev = torch.device("cuda", 0); torch.cuda.set_device(0)
    name, limit = card()
    D = 256
    _, frames = bench.synth_frames(bench.H, bench.W, bench.HD, bench.WD, 4, bench.V, dev, with_ref=False)
    res = {"gpu": name, "power_limit": limit, "hidden_dim": D, "rounds": args.rounds, "steps": args.steps, "shapes": []}
    if args.engine == "simt":
        res["engine"] = "simt"
    if args.t_min is not None:
        res["t_min"] = args.t_min
    for N, S in SHAPES[args.engine]:
        step, peak, n_eval = trainer_steps(N, S, frames, args.rounds, args.steps, dev, args.engine, args.t_min)
        if args.t_min is not None:
            row = {"N": N, "S": S, "step_stash_ms": step["stash"], "step_frame_ms": step["frame"], "step_frame_tmin_ms": step["frame_tmin"],
                   "peak_stash_bytes": int(peak["stash"]), "peak_frame_bytes": int(peak["frame"]),
                   "peak_frame_tmin_bytes": int(peak["frame_tmin"]), "train_mean_n_eval": n_eval,
                   "ops_pair": ops_pair_tmin({"seeded": seeded_field(N, S, D)}, args.t_min, args.rounds)}
            res["shapes"].append(row)
            print("N=%d S=%d D=%d  graph step: stash %.2f ms, frame_grad %.2f ms, frame_grad t_min=%g %.2f ms (n_eval per step: mean %.1f, min %.1f, max %.1f); "
                  "peak %.2f / %.2f / %.2f GB" % (N, S, D, step["stash"], step["frame"], args.t_min, step["frame_tmin"], n_eval["mean"],
                                                n_eval["min"], n_eval["max"], peak["stash"] / 1e9,
                                      peak["frame"] / 1e9, peak["frame_tmin"] / 1e9), file=sys.stderr, flush=True)
            continue
        pair = ops_pair(N, S, D, args.rounds, args.engine)
        row = {"N": N, "S": S, "step_stash_ms": step["stash"], "step_frame_ms": step["frame"], "step_ratio": step["frame"] / step["stash"],
               "peak_stash_bytes": int(peak["stash"]), "peak_frame_bytes": int(peak["frame"]),
               "ops_pair_ms": pair["pair"], "ops_fwd_plus_frame_bwd_ms": pair["fwd_plus_frame_bwd"],
               "ops_ratio": pair["pair"] / pair["fwd_plus_frame_bwd"]}
        res["shapes"].append(row)
        print("N=%d S=%d D=%d  graph step: stash %.2f ms, frame_grad %.2f ms (x%.2f); peak %.2f GB -> %.2f GB | ops: train pair %.2f ms, "
              "render_frame_engine + nnb_render_frame_bwd %.2f ms (x%.2f)"
              % (N, S, D, step["stash"], step["frame"], row["step_ratio"], peak["stash"] / 1e9, peak["frame"] / 1e9, pair["pair"],
                 pair["fwd_plus_frame_bwd"], row["ops_ratio"]), file=sys.stderr, flush=True)
    if args.t_min is not None:
        res["ops_pair_plants"] = ops_pair_tmin({"scattered_s256": planted_field("s256"), "translucent_t100": planted_field("t100")},
                                               args.t_min, args.rounds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

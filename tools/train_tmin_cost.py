"""Cost of Trainer(train_t_min=t): the captured training step with early ray termination on the per-sample stash
(ops.stash_render_call: nnb_render_fwd_tmin + nnb_render_bwd_tmin) against the default step, the frame pair with early termination
(Trainer(frame_grad=True, frame_grad_t_min=t)) and train_t_min=0 (no ray stops: the packing's overhead over the default step).
Shapes: the C2 step (1024 rays x 128 samples, bench.py's render-only configuration and frames) at D = 256, 128 and 64, and 4096 x 512 at
D = 256.  Fields: bench.py's untrained field, and the seeded surface field (the weights of tools/train_frame_cost.py's seeded_field,
which stop every ray after its first chunk at t = 1e-4) loaded into the trainer's network.
One Trainer per configuration; graph steps alternated between them over --rounds rounds of --steps steps, median ms per step (at
4096 x 512, where two trainers' stashes do not fit in the card together, each configuration's rounds run alone in turn); the mean
n_eval of the training render over --steps untimed steps after the timed rounds; the peak torch.cuda.max_memory_allocated over each
Trainer's build and warm-up, above what was allocated before it.  The card's name and power limit are read in the same run
(nvidia-smi query, read-only).  Writes one JSON line to stdout.  Without a CUDA device the tool fails.
--engine simt measures the exact-fp32 engine instead (every render of the step on it, ops.set_default_engine('simt')): the default exact
step against Trainer(train_t_min=t, train_t_min_engine='simt') (ops.exact_stash_render_call) and the same at t = 0, at the C2 step for
D = 256 and 64 and at 1024 rays x 8 samples (D = 256), on the same two fields."""
import argparse, gc, json, os, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from field_query_cost import card  # noqa: E402
from train_frame_cost import timed  # noqa: E402

SIZES = ((1024, 128, 256), (4096, 512, 256), (1024, 128, 128), (1024, 128, 64))
SIMT_SIZES = ((1024, 128, 256), (1024, 128, 64), (1024, 8, 256))


def configs(t, engine="tc"):
    if engine == "simt":
        return {"default": {}, "stash_tmin": dict(train_t_min=t, train_t_min_engine="simt"),
                "stash_t0": dict(train_t_min=0.0, train_t_min_engine="simt")}
    return {"default": {}, "frame_tmin": dict(frame_grad=True, frame_grad_t_min=t), "stash_tmin": dict(train_t_min=t),
            "stash_t0": dict(train_t_min=0.0)}


def build(N, S, D, field, dev, kw):
    import bench
    import nope_nerf_b200.model as mdl
    from oracle import nerf_oracle as O
    cfg = bench.make_cfg(N)
    cfg["rendering"]["num_points"] = S
    cfg["model"]["hidden_dim"] = D
    np.random.seed(42); torch.manual_seed(42)
    net = mdl.OfficialStaticNerf(cfg)
    if field == "surface":
        net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=7, D=D, hf_damp=True).items()})
    model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
    pose = mdl.LearnPose(bench.V, True, True, cfg).to(dev); dnet = mdl.Learn_Distortion(bench.V, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.normal_(0, 0.05); pose.t.normal_(0, 0.05)
    return mdl.Trainer(model, torch.optim.Adam(model.parameters(), lr=1e-3), cfg["training"], device=dev,
                       optimizer_pose=torch.optim.Adam(pose.parameters(), lr=5e-4), pose_param_net=pose,
                       optimizer_distortion=torch.optim.Adam(dnet.parameters(), lr=5e-4), distortion_net=dnet, **kw)


def run(N, S, D, field, frames, t, rounds, steps, dev, keys, engine="tc"):
    trainers, peak, calls = {}, {}, {}
    step = lambda tr, i: tr.train_step(frames[i % len(frames)], it=i, epoch=0, scheduling_start=10000, render_path=None)
    for key, kw in configs(t, engine).items():
        if key not in keys:
            continue
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(); torch.cuda.reset_peak_memory_stats()
        tr = build(N, S, D, field, dev, kw)
        cls = tr._train_render_call(True)
        if getattr(cls, "t_min", None) is not None:   # keep the training renders' calls for n_eval
            calls[key] = []
            rec = type("Recorded", (cls,), {"__init__": lambda self, *a, _c=cls, _l=calls[key], **k: (_l.append(self), _c.__init__(self, *a, **k))[1]})
            tr._train_render_call = lambda backward, rec=rec, tr=tr: rec if backward else type(tr)._train_render_call(tr, False)
        for i in range(3):                                   # eager warm-up, capture, first replay
            step(tr, i)
        torch.cuda.synchronize()
        peak[key] = torch.cuda.max_memory_allocated() - base
        trainers[key] = tr
    assert all(len([v for v in tr._gsteps.values() if v]) == 1 for tr in trainers.values()), "the graph step did not run"
    times = {k: [] for k in trainers}
    order = list(trainers)
    for r in range(rounds):
        for key in (order if r % 2 == 0 else order[::-1]):
            times[key].append(timed(lambda i, tr=trainers[key]: step(tr, i), steps))
    n_eval = {}
    for key, lst in calls.items():
        vals = []
        for i in range(steps):
            step(trainers[key], i)
            vals.append(float(lst[-1].n_eval.float().mean()))
        n_eval[key] = float(np.mean(vals))
    return {k: float(np.median(v)) for k, v in times.items()}, peak, n_eval


def release():
    """frees what the last run() held (a recorded trainer refers to itself, so only the collector frees it) and the pooled workspaces"""
    from nope_nerf_b200 import ops
    gc.collect()
    ops._pool.free.clear()
    gc.collect(); torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20, help="graph steps per timed round")
    ap.add_argument("--t-min", type=float, default=1e-4)
    ap.add_argument("--sizes", default="all", help="'all' or 'c2' (the C2 step at D = 256 only)")
    ap.add_argument("--engine", default="tc", choices=("tc", "simt"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_tmin_cost.py needs a CUDA device")
    import bench
    from nope_nerf_b200 import ops
    if args.engine == "simt":
        ops.set_default_engine("simt")
    dev = torch.device("cuda")
    name, limit = card()
    _, frames = bench.synth_frames(bench.H, bench.W, bench.HD, bench.WD, 4, bench.V, dev, with_ref=False)
    out = dict(card=name, power_limit=limit, engine=args.engine, t_min=args.t_min, rounds=args.rounds, steps=args.steps, results=[])
    sizes = SIMT_SIZES if args.engine == "simt" else SIZES
    for N, S, D in (sizes if args.sizes == "all" else sizes[:1]):
        for field in ("bench", "surface"):
            # the stash of two 4096 x 512 trainers does not fit in 80 GB together: there each configuration runs alone, not alternated
            groups = [list(configs(0.0, args.engine))] if N * S <= 1024 * 128 else [[k] for k in configs(0.0, args.engine)]
            ms, peak, n_eval = {}, {}, {}
            for keys in groups:
                res = run(N, S, D, field, frames, args.t_min, args.rounds, args.steps, dev, keys, args.engine)
                for d, r in zip((ms, peak, n_eval), res):
                    d.update(r)
                release()
            row = dict(N=N, S=S, D=D, field=field, ms=ms, peak_mb={k: v / 2 ** 20 for k, v in peak.items()}, mean_n_eval=n_eval)
            out["results"].append(row)
            print("%s N=%d S=%d D=%d %s" % (name, N, S, D, field), " ".join("%s %.2f ms" % kv for kv in ms.items()),
                  "n_eval", {k: round(v, 1) for k, v in n_eval.items()},
                  "peak MB", {k: round(v / 2 ** 20) for k, v in peak.items()}, file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

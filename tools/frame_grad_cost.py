"""Cost of the differentiable frame: nnb_render_frame_bwd (forward with checkpoints, then reverse rounds over 32-sample chunks, each
evaluating its chunk again with a chunk-sized stash) against nnb_render_fwd (NNB_STASH) + nnb_render_bwd, gradients to the MLP and the
pose.  Shapes: the C2 training step (1024 rays x 128 samples) and N = 4096, S = 512, D = 256; each timed call is a whole forward +
backward, alternated between the two paths over --rounds rounds, median reported.  Workspace bytes of both paths are printed beside
them.  --engine simt times the exact-fp32 engine's forms instead (nnb_render_frame_bwd_engine against nnb_render_fwd + nnb_render_bwd on
NNB_ENGINE_SIMT) and adds one call of the frame backward alone at N = 4096, S = 1024, where the exact stash path cannot be sized.  The
card's name and power limit are read in the same run (nvidia-smi query, read-only).  Without a CUDA device the tool fails."""
import argparse, json, os, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from field_query_cost import card  # noqa: E402

SHAPES = ((1024, 128), (4096, 512))
FRAME_ONLY = {"simt": ((4096, 1024),), "tc": ()}   # shapes timed on the frame path alone


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--engine", choices=("tc", "simt"), default="tc")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("frame_grad_cost: needs a CUDA device (there is no CPU path and a CPU timing would say nothing about the GPU)")
    from nope_nerf_b200 import ops, _lib as L
    from oracle import nerf_oracle as O
    name, limit = card()
    D = args.dim
    res = {"gpu": name, "power_limit": limit, "hidden_dim": D, "rounds": args.rounds, "shapes": []}
    eng = L.ENGINE_SIMT if args.engine == "simt" else L.ENGINE_TC
    if args.engine == "simt":
        res["engine"] = "simt"
    for N, S in SHAPES + FRAME_ONLY[args.engine]:
        frame_only = (N, S) in FRAME_ONLY[args.engine]
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

        def stash():
            call = ops.RenderCall(flat, c2w, cam, stash=True, engine=eng, **kw)
            call.backward(g_rgb, g_dp, g_dg, g_w, g_c)

        def frame():
            ops.render_frame_bwd(flat, c2w, cam, g_rgb, g_dp, g_dg, g_w, g_c, engine=eng, **kw)

        paths = (("frame", frame),) if frame_only else (("stash", stash), ("frame", frame))
        times = {k: [] for k, _ in paths}
        for _, fn in paths:   # warm-up: module load, workspace allocation
            fn(); fn()
        torch.cuda.synchronize()
        for r in range(args.rounds):
            for key, fn in paths if r % 2 == 0 else paths[::-1]:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); fn(); e1.record(); e1.synchronize()
                times[key].append(e0.elapsed_time(e1))
        med = {k: float(np.median(v)) for k, v in times.items()}
        stash_ws = int(L.lib.nnb_workspace_bytes_dim(N, S, L.STASH, eng, D))
        frame_ws = int(L.lib.nnb_render_frame_bwd_workspace_bytes_engine(N, S, D, eng))
        if frame_only:
            row = {"N": N, "S": S, "frame_bwd_ms": med["frame"], "stash_ws_bytes": stash_ws, "frame_bwd_ws_bytes": frame_ws}
            res["shapes"].append(row)
            print("N=%d S=%d D=%d  frame_bwd %.2f ms  workspace %.2f GB (the stash path would need %.2f GB)"
                  % (N, S, D, med["frame"], frame_ws / 1e9, stash_ws / 1e9), file=sys.stderr, flush=True)
            ops._pool.free.clear(); torch.cuda.empty_cache()
            continue
        row = {"N": N, "S": S, "stash_fwd_bwd_ms": med["stash"], "frame_bwd_ms": med["frame"], "ratio": med["frame"] / med["stash"],
               "stash_ws_bytes": stash_ws, "frame_bwd_ws_bytes": frame_ws}
        res["shapes"].append(row)
        print("N=%d S=%d D=%d  render_fwd+bwd %.2f ms  frame_bwd %.2f ms (x%.2f)  workspace %.2f GB -> %.2f GB"
              % (N, S, D, med["stash"], med["frame"], row["ratio"], row["stash_ws_bytes"] / 1e9, row["frame_bwd_ws_bytes"] / 1e9),
              file=sys.stderr, flush=True)
        ops._pool.free.clear(); torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Cost of the differentiable normals on each engine (CUDA events, median of --reps after --warmup):
  * gradient() + its backward with gradients to p and every parameter: the exact engine (nnb_field_hvp) against
    gradient_grad(engine='tc', grad_engine='tc') (nnb_field_hvp_tc), at M = 2 048 / 16 384 / 131 072 / 524 288 points and
    model.hidden_dim 64 / 128 / 256;
  * the C2 Renderer.nope_nerf forward + backward (N = 1024 rays, S = 128 samples, D = 256) with normal_loss, on the exact engine and with
    Renderer(normal_engine='tc', normal_grad_engine='tc').
Every configuration is timed in each of --rounds rounds, the configurations alternating within a round; the JSON line gives the median
and the range over the rounds, with the card's name and power limit read in the same run (nvidia-smi query, read-only)."""
import argparse, json, os, sys
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from normals_cost import timed, card, net_for   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default="2048,16384,131072,524288")
    args = ap.parse_args()
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rounds": args.rounds}
    g = torch.Generator().manual_seed(0)
    steps = {}
    for D in (64, 128, 256):
        net, _ = net_for(D)
        for M in [int(x) for x in args.sizes.split(",")]:
            p0 = (torch.rand(M, 3, generator=g) * 2 - 1).cuda()
            for eng in ("exact", "tc"):
                kw = dict(engine="tc", grad_engine="tc") if eng == "tc" else {}

                def step(net=net, p0=p0, kw=kw):
                    p = p0.clone().requires_grad_(True)
                    net.gradient_grad(p, 0, **kw).norm(dim=-1).mean().backward()
                steps["gradient_fwd_bwd_M%d_D%d_%s_ms" % (M, D, eng)] = step
    N = 1024
    pix = (torch.rand(1, N, 2, generator=g) * 2 - 1).cuda()
    depth = (torch.rand(N, generator=g) * 3 + 1).cuda()
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], device="cuda")[None]
    for eng in ("exact", "tc"):
        net, rend = net_for(256, True)
        if eng == "tc":
            import nope_nerf_b200.model as mdl
            rend = mdl.Renderer(net, rend.cfg, device=torch.device("cuda"), normal_engine="tc", normal_grad_engine="tc")

        def step(rend=rend):
            c2w = torch.eye(4, device="cuda").requires_grad_(True)
            out = rend.nope_nerf(pix, depth, cam, None, None, add_noise=True, it=0, c2w=c2w)
            (out["rgb"].sum() + out["depth_pred"].sum() + out["normal"].mean()).backward()
        steps["render_C2_fwd_bwd_normal_loss_%s_ms" % eng] = step
    times = {k: [] for k in steps}
    for _ in range(args.rounds):
        for k, fn in steps.items():
            times[k].append(timed(fn, args.warmup, args.reps))
    for k, v in times.items():
        res[k] = {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

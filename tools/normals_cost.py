#!/usr/bin/env python
"""Cost of rendering.normal_loss and the differentiable OfficialStaticNerf.gradient (CUDA events, median of --reps after --warmup):
  * gradient() + its backward (nnb_field_hvp) at M = 2048 points, for model.hidden_dim 64 / 128 / 256;
  * the C2 Renderer.nope_nerf forward + backward (N = 1024 rays, S = 128 samples) with normal_loss off and on.
Every configuration is timed in each of --rounds rounds, the configurations alternating within a round; the JSON line gives the median
and the range over the rounds, with the card's name and power limit read in the same run (nvidia-smi query, read-only)."""
import argparse, json, os, subprocess, sys
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timed(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True,
                           timeout=60).stdout.strip().splitlines()[torch.cuda.current_device()]
        name, limit = [x.strip() for x in q.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def net_for(D, normal_loss=False):
    import nope_nerf_b200.model as mdl
    from oracle import nerf_oracle as O
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from _cfg import default_cfg
    cfg = default_cfg()
    cfg["model"]["hidden_dim"] = D; cfg["rendering"]["normal_loss"] = normal_loss; cfg["rendering"]["num_points"] = 128
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=1, D=D, hf_damp=True).items()})
    net = net.cuda()
    return net, mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rounds": args.rounds}
    g = torch.Generator().manual_seed(0)
    p0 = (torch.rand(2048, 3, generator=g) * 2 - 1).cuda()
    N, S = 1024, 128
    pix = (torch.rand(1, N, 2, generator=g) * 2 - 1).cuda()
    depth = (torch.rand(N, generator=g) * 3 + 1).cuda()
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], device="cuda")[None]
    steps = {}
    for D in (64, 128, 256):
        net, _ = net_for(D)

        def step(net=net):
            p = p0.clone().requires_grad_(True)
            net.gradient(p, 0).norm(dim=-1).mean().backward()
        steps["gradient_fwd_bwd_M2048_D%d_ms" % D] = step
    for nl in (False, True):
        net, rend = net_for(256, nl)

        def step(rend=rend):
            c2w = torch.eye(4, device="cuda").requires_grad_(True)
            out = rend.nope_nerf(pix, depth, cam, None, None, add_noise=True, it=0, c2w=c2w)
            loss = out["rgb"].sum() + out["depth_pred"].sum()
            if out["normal"] is not None:
                loss = loss + out["normal"].mean()
            loss.backward()
        steps["render_C2_fwd_bwd_normal_loss_%s_ms" % ("on" if nl else "off")] = step
    times = {k: [] for k in steps}
    for _ in range(args.rounds):
        for k, fn in steps.items():
            times[k].append(timed(fn, args.warmup, args.reps))
    for k, v in times.items():
        res[k] = {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

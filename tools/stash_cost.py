#!/usr/bin/env python
"""What the fp32 training stash costs the tensor-core field kernels, at the C2 shape (1024 rays x 128 samples) and hidden_dim 256, 128
and 64: device time of

  tc_field_fwd<D>  via nnb_render_fwd with NNB_STASH (h0..h7, feat, hr, enc, denc and the ReLU gate bits) and without it (neither);
  tc_dgrad<D>      via nnb_render_bwd with g_weights (the dY stash is written) and with g_weights = NULL (write_dy = 0: no dY stash).

The configurations alternate over R rounds in one process; each round times K calls of each with torch.profiler (CUDA activities) and
takes the kernel's device time per launch it recorded.  Medians over the rounds, and the spread (max - min).  The stash bytes per call come from the
layout (nnb_debug_layout is not needed: the widths are fixed by D).  NNB_LIB_PATH selects a library variant.
    python tools/stash_cost.py [tag] [K] [R]"""
import json, os, re, statistics, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from nope_nerf_b200 import ops, _lib as L

N, S, H, W = 1024, 128, 1080, 1920
DIMS = (256, 128, 64)


def stash_bytes(D, M):
    """fp32 floats per sample written by the forward (h0..h7, feat, hr, enc, denc) and by tc_dgrad (dy0..dy7, dfeat, dyr, dyc)"""
    return M * 4 * (9 * D + D // 2 + 64 + 32), M * 4 * (9 * D + D // 2 + 4)


def make_inputs(D, dev, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    w = (torch.randn(L.num_params(D), generator=g) * (1.0 / D ** 0.5)).to(dev)
    c2w = torch.eye(4).to(dev)
    cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0])).to(dev)
    ray_idx = torch.randperm(H * W, generator=g)[:N].to(torch.int64).to(dev)
    noise = torch.rand(N, S, generator=g).to(dev)
    dmap = (torch.rand(H // 8, W // 8, generator=g) * 6 + 0.6).to(dev)
    scale, shift = torch.ones(1, device=dev), torch.zeros(1, device=dev)
    g_rgb, g_dp, g_dg = (torch.randn(N, 3, generator=g) * 1e-3).to(dev), (torch.randn(N, generator=g) * 1e-3).to(dev), torch.zeros(N, device=dev)
    return w, c2w, cam, ray_idx, noise, dmap, scale, shift, g_rgb, g_dp, g_dg


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else ""
    K = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    R = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    dev = torch.device("cuda", 0); torch.cuda.set_device(0)
    flags = L.SOFTPLUS | L.USE_DIR
    inp = {D: make_inputs(D, dev, 7 + D) for D in DIMS}

    def call(D, stash):
        w, c2w, cam, ray_idx, noise, dmap, scale, shift = inp[D][:8]
        return ops.RenderCall(w, c2w, cam, N=N, S=S, flags=flags, engine=L.ENGINE_TC, near=0.01, far=10.0, ray_idx=ray_idx,
                              depth_map=dmap, scale=scale, shift=shift, noise=noise, H=H, W=W, stash=stash, hidden_dim=D)

    def fwd(D, stash):
        c = call(D, stash)
        if stash:
            c.release()

    def bwd(D, gw):
        c = call(D, True)
        g_rgb, g_dp, g_dg = inp[D][8:]
        g_c = torch.zeros(4, 4, device=dev)
        c.backward(g_rgb, g_dp, g_dg, torch.zeros(L.num_params(D), device=dev) if gw else None, g_c)

    configs = []
    for D in DIMS:
        configs += [("fwd", D, "stash", lambda D=D: fwd(D, True)), ("fwd", D, "no_stash", lambda D=D: fwd(D, False)),
                    ("dgrad", D, "dy_stash", lambda D=D: bwd(D, True)), ("dgrad", D, "no_dy_stash", lambda D=D: bwd(D, False))]
    for _, _, _, f in configs:   # warm every shape: module load, workspace pool, stage tables
        for _ in range(3): f()
    torch.cuda.synchronize()
    times = {(k, D, v): [] for k, D, v, _ in configs}
    for _ in range(R):
        for kind, D, var, f in configs:
            name = "tc_field_fwd<%d>" % D if kind == "fwd" else "tc_dgrad<%d>" % D
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(K): f()
                torch.cuda.synchronize()
            tot, cnt = 0.0, 0
            for ev in prof.key_averages():
                if re.search(r"\b%s" % re.escape(name), ev.key) and "(" in ev.key:
                    t = getattr(ev, "device_time_total", None)
                    tot += ev.cuda_time_total if t is None else t
                    cnt += ev.count
            if cnt < K // 2:   # the profiler can drop a few kernel records of a window; a window that lost most is not used
                raise RuntimeError("%s: %d launches of %s in %d calls" % (var, cnt, name, K))
            times[(kind, D, var)].append(tot / cnt / 1e3)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {}
    M = N * S
    for (kind, D, var), v in times.items():
        res.setdefault("D%d" % D, {})["%s_%s_ms" % (kind, var)] = round(statistics.median(v), 4)
        res["D%d" % D]["%s_%s_spread_ms" % (kind, var)] = round(max(v) - min(v), 4)
    for D in DIMS:
        r = res["D%d" % D]
        fb, db = stash_bytes(D, M)
        r["fwd_stash_gb"], r["dgrad_stash_gb"] = round(fb / 1e9, 3), round(db / 1e9, 3)
        r["fwd_stash_cost_ms"] = round(r["fwd_stash_ms"] - r["fwd_no_stash_ms"], 4)
        r["dgrad_stash_cost_ms"] = round(r["dgrad_dy_stash_ms"] - r["dgrad_no_dy_stash_ms"], 4)
    print(json.dumps({"tag": tag, "lib": os.path.basename(L.LIB_PATH), "gpu": q.splitlines()[0] if q else "", "calls_per_round": K,
                      "rounds": R, "M": M, "by_width": res}))


if __name__ == "__main__":
    main()

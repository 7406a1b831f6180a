#!/usr/bin/env python
"""Cost of explicit-point field queries (nnb_field_fwd) on the exact-fp32 engine, the tensor-core engine, and the tensor-core engine
with NNB_OCC_ONLY, for M points x model.hidden_dim D; and of one geometry frame (Renderer.phong_renderer: 512-step ray marching,
8 secant steps, normals, surface colour) with Renderer(field_engine=None) against field_engine='tc'.

CUDA events around each call.  Every shape is warmed up first; then every configuration is timed in each of --rounds rounds, the
configurations alternating within a round, and the JSON line gives the median and the range over the rounds.  FLOP per point come from
the layer shapes (2 per multiply-add of the layers the mode evaluates).  The card's name and power limit are read in the same run
(nvidia-smi query, read-only).  There is no CPU path: without a CUDA device the tool fails."""
import argparse, ctypes as C, json, os, subprocess, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = (4096, 16384, 131072, 524288, 3500000)
DIMS = (64, 128, 256)


def flop_per_point(D, occ_only):
    """2 x the multiply-adds of OfficialStaticNerf on one point (official_nerf.py:20-37); occ_only stops after fc_density"""
    trunk = 63 * D + 3 * D * D + (D + 63) * D + 3 * D * D + D
    colour = D * D + (D + 27) * (D // 2) + 3 * (D // 2)
    return 2 * (trunk + (0 if occ_only else colour))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True,
                           timeout=60).stdout.strip().splitlines()[torch.cuda.current_device()]
        name, limit = [x.strip() for x in q.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def once(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); b.synchronize()
    return a.elapsed_time(b)


def rounds_of(fns, warmup, reps, rounds):
    """fns: {name: callable}.  Returns {name: per-round medians of `reps` calls}, the names alternating within a round."""
    for f in fns.values():
        for _ in range(warmup):
            f()
    torch.cuda.synchronize()
    out = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            out[k].append(float(np.median([once(f) for _ in range(reps)])))
    return out


def summary(ts):
    return dict(median_ms=float(np.median(ts)), min_ms=float(min(ts)), max_ms=float(max(ts)))


def field_fn(L, ops, flat, D, p, d, flags, engine):
    M = p.shape[0]
    ws = torch.empty(L.lib.nnb_workspace_bytes_dim(M, 1, flags, engine, D), dtype=torch.uint8, device="cuda")
    out = torch.empty(M, 4, device="cuda")
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p); a.dirs = L.ptr(d); a.N = M; a.S = 1; a.flags = flags; a.engine = engine; a.hidden_dim = D
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    keep = (ws, out, flat, p, d)

    def call(a=a, out=out, keep=keep):
        L.check(L.lib.nnb_field_fwd(C.byref(a), L.ptr(out), ops._stream()), "nnb_field_fwd")
    return call


def geometry_frame(H, W, warmup, reps, rounds):
    """one phong_renderer frame of H x W pixels in chunks of 1024 pixels (the chunk size of render_visdata / render_geometry)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import _fullsize_cases as FC
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200.model import common as mc
    cfg = FC.default_cfg()
    state = FC.start_state(cfg, 4, 31, 95, geo=True)
    dev = torch.device("cuda")
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: v.clone() for k, v in state["net"].items()})
    data = FC.small_scene(H, W, V=4)
    pixels = mc.arange_pixels((H, W), 1)[1].cuda()
    cam = data["img.camera_mat"].cuda(); smat = data["img.scale_mat"].cuda()
    pose = mdl.LearnPose(4, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.copy_(state["r"]); pose.t.copy_(state["t"])
        wmat = torch.inverse(pose(1)).unsqueeze(0)
    fns = {}
    for name, fe in (("exact", None), ("tc", "tc")):
        rend = mdl.Renderer(net, cfg["rendering"], device=dev, field_engine=fe)

        def frame(rend=rend):
            for px in torch.split(pixels, 1024, dim=1):
                rend(px, None, cam, wmat, smat, "phong_renderer", it=0)
        fns[name] = frame
    ts = rounds_of(fns, warmup, reps, rounds)
    return {k: summary(v) for k, v in ts.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="*", default=list(SIZES))
    ap.add_argument("--dims", type=int, nargs="*", default=list(DIMS))
    ap.add_argument("--frame", type=int, nargs=2, default=[270, 480], metavar=("H", "W"), help="geometry frame size; 0 0 skips it")
    ap.add_argument("--frame-reps", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("field_query_cost: needs a CUDA device (there is no CPU path and a CPU timing would say nothing about the GPU)")
    from nope_nerf_b200 import _lib as L, ops
    from oracle import nerf_oracle as O
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rounds": args.rounds, "reps": args.reps, "field": [], "flop_per_point": {}}
    g = torch.Generator().manual_seed(0)
    for D in args.dims:
        res["flop_per_point"][str(D)] = {"full": flop_per_point(D, False), "occ_only": flop_per_point(D, True)}
        flat = torch.from_numpy(O.flatten_params(O.init_params(seed=1, D=D))).cuda()
        for M in args.sizes:
            p = (torch.rand(M, 3, generator=g) * 3 - 1.5).cuda()
            d = torch.nn.functional.normalize(torch.randn(M, 3, generator=g), dim=1).cuda()
            fns = {"simt": field_fn(L, ops, flat, D, p, d, L.SOFTPLUS, L.ENGINE_SIMT),
                   "tc": field_fn(L, ops, flat, D, p, d, L.SOFTPLUS, L.ENGINE_TC),
                   "tc_occ": field_fn(L, ops, flat, D, p, None, L.SOFTPLUS | L.OCC_ONLY, L.ENGINE_TC)}
            ts = rounds_of(fns, args.warmup, args.reps, args.rounds)
            row = {"D": D, "M": M}
            for k, v in ts.items():
                s = summary(v)
                s["tflops"] = flop_per_point(D, k == "tc_occ") * M / (s["median_ms"] * 1e-3) / 1e12   # algorithmic FLOP of the mode / time
                row[k] = s
            row["simt_over_tc"] = row["simt"]["median_ms"] / row["tc"]["median_ms"]
            row["simt_over_tc_occ"] = row["simt"]["median_ms"] / row["tc_occ"]["median_ms"]
            res["field"].append(row)
            print("D=%3d M=%8d  simt %9.3f ms  tc %9.3f ms (x%.2f)  tc occ-only %9.3f ms (x%.2f)"
                  % (D, M, row["simt"]["median_ms"], row["tc"]["median_ms"], row["simt_over_tc"], row["tc_occ"]["median_ms"], row["simt_over_tc_occ"]),
                  file=sys.stderr)
            del fns, p, d
            torch.cuda.empty_cache()
    H, W = args.frame
    if H > 0 and W > 0:
        fr = geometry_frame(H, W, 1, args.frame_reps, args.rounds)
        res["geometry_frame"] = {"H": H, "W": W, "hidden_dim": 256, **fr, "exact_over_tc": fr["exact"]["median_ms"] / fr["tc"]["median_ms"]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

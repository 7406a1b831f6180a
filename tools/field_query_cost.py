#!/usr/bin/env python
"""Cost of explicit-point field queries (nnb_field_fwd) on the exact-fp32 engine, the tensor-core engine, and the tensor-core engine
with NNB_OCC_ONLY, for M points x model.hidden_dim D; and of one geometry frame (Renderer.phong_renderer: 512-step ray marching,
8 secant steps, normals, surface colour) with Renderer(field_engine=None), with field_engine='tc' through the torch march over
explicit-point queries (Renderer._ray_marching_torch), and with field_engine='tc' as it runs (the fused march, nnb_ray_march); for the
fused march also the share of the frame's rays that take part in each 128-step round, and one ray_march call over the whole frame
instead of 1024-pixel chunks.

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


def geometry_frame(H, W, D, warmup, reps, rounds):
    """one phong_renderer frame of H x W pixels in chunks of 1024 pixels (the chunk size of render_visdata / render_geometry).  The
    field is the seeded geometry field of the tests at width D (tests/_fullsize_cases.start_state(geo=True), net seed 31): the share of
    rays each round of the fused march still carries depends on it."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import _fullsize_cases as FC
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import field
    from nope_nerf_b200.model import common as mc
    cfg = FC.default_cfg()
    cfg["model"]["hidden_dim"] = D
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
    class TorchMarch(mdl.Renderer):   # field_engine's queries through the torch march, as before the fused march existed
        def ray_marching(self, ray0, ray_direction, model, c=None, tau=0.5, n_steps=[128, 129], n_secant_steps=8, depth_range=[0., 2.4],
                         max_points=3500000, rad=1.0):
            n = int(torch.randint(n_steps[0], n_steps[1], (1,)).item())
            return self._ray_marching_torch(ray0, ray_direction, model, n, n_secant_steps, depth_range, max_points, rad, self.field_engine)

    fns = {}
    for name, cls, fe in (("exact", mdl.Renderer, None), ("tc_torch_march", TorchMarch, "tc"), ("tc", mdl.Renderer, "tc")):
        rend = cls(net, cfg["rendering"], device=dev, field_engine=fe)

        def frame(rend=rend):
            for px in torch.split(pixels, 1024, dim=1):
                rend(px, None, cam, wmat, smat, "phong_renderer", it=0)
        fns[name] = frame
    # the march of the whole frame as one nnb_ray_march call (no renderer around it), and what it reports about the rounds
    net = net.to(dev).eval()
    for q in net.parameters():
        q.requires_grad_(False)
    with torch.no_grad():
        cw, rv = rend._rays_world(pixels, cam, wmat, smat)
        far = rend._sphere_far(cw[:, 0], rv, cfg["rendering"]["radius"]).reshape(-1).contiguous()
    ray0, dirs = cw.reshape(-1, 3).contiguous(), rv.reshape(-1, 3).contiguous()
    frac = torch.linspace(0, 1, steps=512, device=dev)
    fns["march_one_call"] = lambda: field.ray_march(net, ray0, dirs, far, frac, 0.0, 8, 0.5)
    ts = rounds_of(fns, warmup, reps, rounds)
    depth, first, _, counts = field.ray_march(net, ray0, dirs, far, frac, 0.0, 8, 0.5, want_bracket=True)
    n = ray0.shape[0]
    out = {k: summary(v) for k, v in ts.items()}
    out["rays"] = n
    out["rays_hit_share"] = float(counts[0]) / n
    out["rays_in_round_share"] = [1.0] + [float(c) / n for c in counts[1:-1].tolist()]   # round k = steps 128 k .. 128 k + 127
    out["tiles_evaluated_over_all_steps"] = (n + int(counts[1:-1].sum())) / (n * 4.0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="*", default=list(SIZES))
    ap.add_argument("--dims", type=int, nargs="*", default=list(DIMS))
    ap.add_argument("--frame", type=int, nargs=2, default=[270, 480], metavar=("H", "W"), help="geometry frame size; 0 0 skips it")
    ap.add_argument("--frame-reps", type=int, default=1)
    ap.add_argument("--frame-dims", type=int, nargs="*", default=[256, 128, 64])
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
        res["geometry_frame"] = []
        for D in args.frame_dims:
            fr = geometry_frame(H, W, D, 1, args.frame_reps, args.rounds)
            res["geometry_frame"].append({"H": H, "W": W, "hidden_dim": D, **fr, "exact_over_tc": fr["exact"]["median_ms"] / fr["tc"]["median_ms"],
                                          "tc_torch_march_over_tc": fr["tc_torch_march"]["median_ms"] / fr["tc"]["median_ms"]})
    print(json.dumps(res))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Cost of one volumetric frame (Extract_Images.render_frame, the renderer of generate_images and Eval_Images.eval_images) two ways, at
H x W pixels, S samples per ray and model.hidden_dim D:
  render_fwd: Extract_Images.render_frame as by default (nnb_render_fwd on the tensor-core engine: 32-byte records per sample, then
              composite_fwd);
  frame:      ops.render_frame (nnb_render_frame: compositing fused into the tensor-core forward) at t_min = 0, 1e-4 and 1e-3.
With --engine simt both run on the exact-fp32 engine instead: render_fwd is Extract_Images.render_frame with Renderer(engine=ENGINE_SIMT)
(nnb_render_fwd on that engine) and frame is ops.render_frame_engine(engine=ENGINE_SIMT) (nnb_render_frame_engine).  The default is tc.
Two fields: 'surface' (the seeded geometry field of the tests, with opaque surfaces) and 'hf' (init_params(seed=7, hf_damp=True), nearly
transparent).  CUDA events around each frame; every call is warmed up first; the calls alternate within each of --rounds rounds, and the
JSON line gives the median and [min, max] over the rounds.  Also reported: mean n_eval, the share of stopped rays, max |rgb - rgb(t_min=0)|,
the PSNR of each frame against the t_min = 0 frame, whether t_min = 0 equals the default path bit for bit, and both paths' workspace
bytes.  The card's name and power limit are read in the same run (nvidia-smi query, read-only).  Without a CUDA device the tool fails."""
import argparse, json, math, os, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from field_query_cost import card, rounds_of, summary  # noqa: E402
from geometry_normals_cost import geometry_net  # noqa: E402

FRAMES = ((540, 960), (1080, 1920))
DIMS = (64, 128, 256)
T_MINS = (0.0, 1e-4, 1e-3)


def make_extract(field, D, S, H, W):
    import nope_nerf_b200.model as mdl
    from oracle import nerf_oracle as O
    from _cfg import default_cfg
    dev = torch.device("cuda")
    if field == "surface":
        net, cfg, _ = geometry_net(D)
    else:
        cfg = default_cfg(); cfg["model"]["hidden_dim"] = D
        net = mdl.OfficialStaticNerf(cfg)
        net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=7, D=D, hf_damp=True).items()})
    cfg["rendering"]["num_points"] = S
    cfg["extract_images"] = {"resolution": (H, W)}
    return mdl.Extract_Images(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev, render_type="nope_nerf")


def frame_cost(field, H, W, D, S, rounds, engine="tc"):
    from nope_nerf_b200 import ops, _lib as L
    ex = make_extract(field, D, S, H, W)
    rend, net = ex.renderer, ex.renderer.model
    eng = {"tc": L.ENGINE_TC, "simt": L.ENGINE_SIMT}[engine]
    if engine == "simt":
        rend.engine = eng
    c2w = torch.eye(4, device="cuda")
    c2w[:3, 3] = torch.tensor([0.05, 0.0, -0.04])
    cam = torch.diag(torch.tensor([1.2, -2.1, -1.0, 1.0])).cuda()
    n = H * W
    ray_idx = torch.arange(n, device="cuda")
    kw = dict(N=n, S=S, flags=ops.flags_from_cfg(rend.cfg, net.occ_activation, eval_=True), engine=eng, near=rend.depth_range[0],
              far=rend.depth_range[1], ray_idx=ray_idx, depth_map=torch.ones(1, 1, device="cuda"), H=H, W=W, hidden_dim=D)
    flat = net.flat_weights()
    frames = {}

    def default():
        frames["render_fwd"] = ex.render_frame(c2w, cam, H, W)[0]
    fns = {"render_fwd": default}
    for t in T_MINS:
        def fn(t=t):
            frames[t] = (ops.render_frame if engine == "tc" else ops.render_frame_engine)(flat, c2w, cam, t_min=t, want_stats=True, **kw)
        fns["frame_%g" % t] = fn
    ts = rounds_of(fns, 1, 1, rounds)
    out = {k: summary(v) for k, v in ts.items()}
    ref = frames[0.0][0]
    out["t0_bit_equal"] = bool(torch.equal(frames["render_fwd"].reshape(-1, 3), ref))
    for t in T_MINS:
        rgb, n_eval = frames[t][0], frames[t][4]
        mse = float(((rgb.double() - ref.double()) ** 2).mean())
        out["frame_%g" % t].update(mean_n_eval=float(n_eval.double().mean()), stopped=float((n_eval < S).double().mean()),
                                   max_abs_drgb=float((rgb - ref).abs().max()), psnr_vs_t0=(math.inf if mse == 0 else -10 * math.log10(mse)),
                                   over_render_fwd=out["frame_%g" % t]["median_ms"] / out["render_fwd"]["median_ms"])
    out["workspace_render_fwd"] = int(L.lib.nnb_workspace_bytes_dim(n, S, kw["flags"], eng, D))
    out["workspace_frame"] = int(L.lib.nnb_render_frame_workspace_bytes_engine(n, S, D, eng))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--dims", type=int, nargs="*", default=list(DIMS))
    ap.add_argument("--fields", nargs="*", default=["surface", "hf"])
    ap.add_argument("--frames", type=int, nargs="*", default=[x for f in FRAMES for x in f], metavar="H W")
    ap.add_argument("--engine", choices=["tc", "simt"], default="tc")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("frame_cost: needs a CUDA device (there is no CPU path and a CPU timing would say nothing about the GPU)")
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "engine": args.engine, "rounds": args.rounds, "S": args.samples, "frames": []}
    for H, W in zip(args.frames[0::2], args.frames[1::2]):
        for D in args.dims:
            for field in args.fields:
                fr = frame_cost(field, H, W, D, args.samples, args.rounds, args.engine)
                res["frames"].append({"field": field, "H": H, "W": W, "hidden_dim": D, **fr})
                print("%s %-7s %dx%d D=%3d S=%d  render_fwd %.1f ms  frame t0 %.1f ms (x%.3f)  1e-4 %.1f ms  1e-3 %.1f ms (n_eval %.1f)"
                      % (args.engine, field, H, W, D, args.samples, fr["render_fwd"]["median_ms"], fr["frame_0"]["median_ms"], fr["frame_0"]["over_render_fwd"],
                         fr["frame_0.0001"]["median_ms"], fr["frame_0.001"]["median_ms"], fr["frame_0.001"]["mean_n_eval"]),
                      file=sys.stderr, flush=True)
                torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

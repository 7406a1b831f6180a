#!/usr/bin/env python
"""Cost of the geometry view's normals and of its chunking.

(a) OfficialStaticNerf.gradient(p) (detached normals, d logit / d p) on the exact-fp32 engine (engine=None: nnb_field_fwd + nnb_field_bwd)
    and on tensor cores (engine='tc': nnb_field_vjp, occupancy-only) for M points x model.hidden_dim D.
(b) one phong_renderer frame of H x W pixels at each D in three configurations: Renderer(field_engine='tc') in 1024-pixel chunks (the
    configuration before normal_engine existed), plus normal_engine='tc' in 1024-pixel chunks (rendering.GEOMETRY_CHUNK, what
    Extract_Images.render_geometry runs), plus chunks of LARGE_CHUNK pixels.  The JSON line says whether the last two frames are
    bit-identical: they are not in general, because the camera rays of Renderer._rays_world depend on the chunk (rendering.py).

CUDA events around each call; every shape is warmed up first; the configurations alternate within each of --rounds rounds and the JSON
line gives the median and range over the rounds.  The card's name and power limit are read in the same run (nvidia-smi query,
read-only).  There is no CPU path: without a CUDA device the tool fails."""
import argparse, json, os, sys
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from field_query_cost import card, rounds_of, summary  # noqa: E402

SIZES = (4096, 16384, 131072, 524288)
LARGE_CHUNK = 65536   # pixels per call of the third frame configuration (the workspaces stay well under 1 GB at 1080 x 1920)
DIMS = (64, 128, 256)


def geometry_net(D):
    """the seeded geometry field of the tests at width D (tests/_fullsize_cases.start_state(geo=True), net seed 31)"""
    import _fullsize_cases as FC
    import nope_nerf_b200.model as mdl
    cfg = FC.default_cfg()
    cfg["model"]["hidden_dim"] = D
    state = FC.start_state(cfg, 4, 31, 95, geo=True)
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: v.clone() for k, v in state["net"].items()})
    return net.cuda(), cfg, state


def frame_cost(H, W, D, warmup, reps, rounds):
    import _fullsize_cases as FC
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200.model import common as mc
    from nope_nerf_b200.model.rendering import GEOMETRY_CHUNK
    net, cfg, state = geometry_net(D)
    dev = torch.device("cuda")
    data = FC.small_scene(H, W, V=4)
    pixels = mc.arange_pixels((H, W), 1)[1].cuda()
    cam = data["img.camera_mat"].cuda(); smat = data["img.scale_mat"].cuda()
    pose = mdl.LearnPose(4, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.copy_(state["r"]); pose.t.copy_(state["t"])
        wmat = torch.inverse(pose(1)).unsqueeze(0)
    rends = {"field_tc": mdl.Renderer(net, cfg["rendering"], device=dev, field_engine="tc"),
             "field_tc_normal_tc": mdl.Renderer(net, cfg["rendering"], device=dev, field_engine="tc", normal_engine="tc")}
    chunks = {"field_tc": GEOMETRY_CHUNK, "field_tc_normal_tc": GEOMETRY_CHUNK, "field_tc_normal_tc_large_chunks": LARGE_CHUNK}
    rends["field_tc_normal_tc_large_chunks"] = rends["field_tc_normal_tc"]
    frames = {}

    def make(name):
        def frame():
            with torch.no_grad():
                frames[name] = torch.cat([rends[name](px, None, cam, wmat, smat, "phong_renderer", it=0)["rgb"]
                                          for px in torch.split(pixels, chunks[name], dim=1)], dim=1)
        return frame
    ts = rounds_of({k: make(k) for k in rends}, warmup, reps, rounds)
    out = {k: summary(v) for k, v in ts.items()}
    out["chunks"] = chunks
    out["large_chunks_bit_identical"] = bool(torch.equal(frames["field_tc_normal_tc"], frames["field_tc_normal_tc_large_chunks"]))
    out["normal_tc_max_abs_diff"] = float((frames["field_tc"] - frames["field_tc_normal_tc"]).abs().max())
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
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("geometry_normals_cost: needs a CUDA device (there is no CPU path and a CPU timing would say nothing about the GPU)")
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rounds": args.rounds, "reps": args.reps, "gradient": []}
    g = torch.Generator().manual_seed(0)
    for D in args.dims:
        net, _, _ = geometry_net(D)
        for M in args.sizes:
            p = (torch.rand(M, 3, generator=g) * 2 - 1).cuda()

            def grad(engine, p=p, net=net):
                with torch.no_grad():
                    net.gradient(p, 0, engine=engine)
            ts = rounds_of({"exact": lambda: grad(None), "tc": lambda: grad("tc")}, args.warmup, args.reps, args.rounds)
            row = {"D": D, "M": M, **{k: summary(v) for k, v in ts.items()}}
            row["exact_over_tc"] = row["exact"]["median_ms"] / row["tc"]["median_ms"]
            res["gradient"].append(row)
            print("gradient D=%3d M=%7d  exact %8.3f ms  tc %8.3f ms (x%.2f)" % (D, M, row["exact"]["median_ms"], row["tc"]["median_ms"],
                                                                            row["exact_over_tc"]), file=sys.stderr)
            del p
            torch.cuda.empty_cache()
    H, W = args.frame
    if H > 0 and W > 0:
        res["geometry_frame"] = []
        for D in args.dims:
            fr = frame_cost(H, W, D, 1, args.frame_reps, args.rounds)
            res["geometry_frame"].append({"H": H, "W": W, "hidden_dim": D, **fr})
            print("frame %dx%d D=%3d  %s" % (H, W, D, {k: round(v["median_ms"], 1) for k, v in fr.items() if isinstance(v, dict) and "median_ms" in v}),
                  file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

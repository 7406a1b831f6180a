#!/usr/bin/env python
"""Cost of one geometry-view frame on the exact-fp32 engine, at H x W pixels and model.hidden_dim D, four ways:
  (a) chunked:        Renderer() through phong_renderer in rendering.GEOMETRY_CHUNK-pixel calls (the default geometry view);
  (b) chunked_fused:  the same with Renderer(fused_march=True) (the march of each chunk in one nnb_ray_march call on the exact engine);
  (c) frame_simt:     Renderer(geometry_frame=True, geometry_frame_engine='simt').phong_frame on the whole frame (one exact call);
  (d) frame_tc:       Renderer(geometry_frame=True).phong_frame, the tensor-core frame, for reference.
Also the whole-frame march alone, the torch march (Renderer._ray_marching_torch on the exact engine) against field.ray_march(engine=
'simt') on the frame's rays, and the share of rays in each round of the fused march.  Method of geometry_frame_cost.py: the seeded
geometry fields of the tests, CUDA events around each frame, every shape warmed up, configurations alternating within each of --rounds
rounds, median and [min, max] over the rounds, the card's name and power limit read in the same run.  No CPU path."""
import argparse, json, os, sys
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from field_query_cost import card, rounds_of, summary  # noqa: E402
from geometry_normals_cost import geometry_net  # noqa: E402


def frame_cost(H, W, D, rounds, configs):
    import _fullsize_cases as FC
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import field
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
    R = lambda **kw: mdl.Renderer(net, cfg["rendering"], device=dev, **kw)
    r_a, r_b, r_c, r_d = R(), R(fused_march=True), R(geometry_frame=True, geometry_frame_engine="simt"), R(geometry_frame=True)
    frames = {}

    def chunked(rend, key):
        def f():
            with torch.no_grad():
                frames[key] = torch.cat([rend.phong_renderer(px, cam, wmat, smat, 0)["rgb"] for px in torch.split(pixels, GEOMETRY_CHUNK, dim=1)], 1)
        return f

    def whole(rend, key):
        def f():
            frames[key] = rend.phong_frame(pixels, cam, wmat, smat, 0)["rgb"]
        return f
    fns = {"chunked": chunked(r_a, "chunked"), "chunked_fused": chunked(r_b, "chunked_fused"), "frame_simt": whole(r_c, "frame_simt"),
           "frame_tc": whole(r_d, "frame_tc")}
    fns = {k: v for k, v in fns.items() if k in configs}
    # the march alone on the frame's own rays
    T = mdl.Renderer._ray_transform(cam, wmat, smat, dev)
    frac = torch.linspace(0, 1, 512, device=dev)
    _, _, it = field.geometry_frame(net, T, pixels, frac, float(cfg["rendering"]["radius"]), want_intermediates=True, engine="simt")
    ray0, rd, far = it["ray0"], it["ray_dir"], it["far"]
    rend_t = R()
    rend_t._sphere_far = lambda cam_loc, d, r: far.view(1, -1)
    marches = {}

    def m_torch():
        with torch.no_grad():
            marches["torch"] = rend_t._ray_marching_torch(ray0[None], rd[None], net, 512, 8, [0., 2.4], 3500000, 1.0, None)[0]

    def m_fused():
        marches["fused"] = field.ray_march(net, ray0, rd, far, frac, 0.0, 8, 0.5, engine="simt")
    if "chunked" in configs:
        fns["march_torch"] = m_torch
    fns["march_fused"] = m_fused
    ts = rounds_of(fns, 1, 1, rounds)
    out = {k: summary(v) for k, v in ts.items()}
    if "march_torch" in marches and "fused" in marches:
        out["march_bits_equal"] = bool(torch.equal(marches["torch"].view(torch.int32), marches["fused"].view(torch.int32)))
    counts = field.ray_march(net, ray0, rd, far, frac, 0.0, 8, 0.5, want_bracket=True, engine="simt")[3].tolist()
    n = ray0.shape[0]
    out["rays_per_round"] = [1.0] + [c / n for c in counts[1:]]
    out["share_hit"] = counts[0] / n
    if "chunked" in frames:
        for k in ("chunked_fused", "frame_simt", "frame_tc"):
            if k in frames:
                diff = (frames["chunked"] - frames[k]).abs().reshape(-1, 3).max(1).values
                out["frac_pixels_off_2_255_" + k] = float((diff > 2.0 / 255).float().mean())
        if "chunked_fused" in frames:
            out["chunked_fused_bits_equal"] = bool(torch.equal(frames["chunked"], frames["chunked_fused"]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dims", type=int, nargs="*", default=[64, 128, 256])
    ap.add_argument("--frame", type=int, nargs=2, default=[270, 480], metavar=("H", "W"))
    ap.add_argument("--configs", nargs="*", default=["chunked", "chunked_fused", "frame_simt", "frame_tc"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("exact_geometry_cost: needs a CUDA device (there is no CPU path and a CPU timing would say nothing about the GPU)")
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rounds": args.rounds, "frames": []}
    H, W = args.frame
    for D in args.dims:
        r = frame_cost(H, W, D, args.rounds, args.configs)
        r.update(H=H, W=W, D=D)
        res["frames"].append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

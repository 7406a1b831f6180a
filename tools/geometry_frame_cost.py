#!/usr/bin/env python
"""Cost of one geometry-view frame two ways, at H x W pixels and model.hidden_dim D:
  chunked: Renderer(field_engine='tc', normal_engine='tc') through phong_renderer in rendering.GEOMETRY_CHUNK-pixel calls (what
           Extract_Images.render_geometry and Trainer.render_visdata run by default);
  frame:   Renderer.phong_frame on the whole frame (nnb_geometry_frame: rays per pixel, march, normals, colour and shading in one call).
CUDA events around each frame; every shape is warmed up first; the two alternate within each of --rounds rounds, and the JSON line gives
the median and [min, max] over the rounds.  The frames are compared too: they differ only where the chunked path's batched-matmul rays
round differently (the share of pixels that differ by more than 2/255 is reported).  The card's name and power limit are read in the same
run (nvidia-smi query, read-only).  There is no CPU path: without a CUDA device the tool fails."""
import argparse, json, os, sys
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from field_query_cost import card, rounds_of, summary  # noqa: E402
from geometry_normals_cost import geometry_net  # noqa: E402

FRAMES = ((270, 480), (1080, 1920))
DIMS = (64, 128, 256)


def frame_cost(H, W, D, rounds):
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
    rend = mdl.Renderer(net, cfg["rendering"], device=dev, field_engine="tc", normal_engine="tc")
    frames = {}

    def chunked():
        with torch.no_grad():
            frames["chunked"] = torch.cat([rend.phong_renderer(px, cam, wmat, smat, 0)["rgb"]
                                           for px in torch.split(pixels, GEOMETRY_CHUNK, dim=1)], dim=1)

    def frame():
        frames["frame"] = rend.phong_frame(pixels, cam, wmat, smat, 0)["rgb"]
    ts = rounds_of({"chunked": chunked, "frame": frame}, 1, 1, rounds)
    out = {k: summary(v) for k, v in ts.items()}
    out["chunked_over_frame"] = out["chunked"]["median_ms"] / out["frame"]["median_ms"]
    diff = (frames["chunked"] - frames["frame"]).abs().reshape(-1, 3).max(1).values
    out["frac_pixels_off_2_255"] = float((diff > 2.0 / 255).float().mean())
    out["frac_surface"] = float((frames["frame"].reshape(-1, 3) < 1).any(1).float().mean())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dims", type=int, nargs="*", default=list(DIMS))
    ap.add_argument("--frames", type=int, nargs="*", default=[x for f in FRAMES for x in f], metavar="H W")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("geometry_frame_cost: needs a CUDA device (there is no CPU path and a CPU timing would say nothing about the GPU)")
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rounds": args.rounds, "frames": []}
    for H, W in zip(args.frames[0::2], args.frames[1::2]):
        for D in args.dims:
            fr = frame_cost(H, W, D, args.rounds)
            res["frames"].append({"H": H, "W": W, "hidden_dim": D, **fr})
            print("frame %dx%d D=%3d  chunked %.1f ms  frame %.1f ms (x%.1f)" % (H, W, D, fr["chunked"]["median_ms"], fr["frame"]["median_ms"],
                                                                               fr["chunked_over_frame"]), file=sys.stderr, flush=True)
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

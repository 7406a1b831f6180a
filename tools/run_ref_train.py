#!/usr/bin/env python
"""Run the UNMODIFIED reference train.py (oracle/_ref/train.py, lines 18-352) against the nope_nerf_b200 drop-in
(BASELINE.json configs[0], SURVEY.md 8(d) "C1": the train.py plumbing run).

    python tools/run_ref_train.py WORKDIR [--impl ours|reference] [--device cuda]

What this script does, and nothing else:
  1. writes a fixture scene in the loader's on-disk layout (SURVEY.md appendix B) under WORKDIR/data/Test/images:
     images/*.png, dpt/depth_<stem>.npz['pred'], intrinsics.npz['K']   (configs/Test/images.yaml: customized_focal, no COLMAP poses)
  2. loads configs/Test/images.yaml over configs/default.yaml with the reference's own dl.load_config and shrinks the
     schedule (2 epochs of 9 views, 256 rays x 64 samples, checkpoint / visualisation / print every few iterations)
  3. applies the INTEGRATION.md binding: the reference's `model` package with its hot-path classes redirected to
     nope_nerf_b200.model (CheckpointIO, model.common.backup / mse2psnr stay the reference's)
  4. calls the reference's train.train(cfg) — its DataLoader / OurDataset, optimizers, CheckpointIO, LR schedule, scale/shift logging,
     render_visdata call, `reset_parameters()` on every nn.Linear at scheduling_start (train.py:342-344) all run as written.
Harness shims (oracle/ref_harness.install_stubs): PIL-backed `imageio`, empty matplotlib / timm / lpips / skimage, and a recording
`torch.utils.tensorboard.SummaryWriter` (tensorboard is not installed in this image).  Prints one JSON line."""
import argparse
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def write_scene(base, V=10, H=48, W=64, hd=24, wd=32, seed=0):
    """appendix B layout; smooth random frames (so that the warped-RGB / point-cloud terms see structure)"""
    import torch
    from PIL import Image
    g = torch.Generator().manual_seed(seed)
    up = lambda t, size: torch.nn.functional.interpolate(t, size, mode="bilinear", align_corners=False)
    os.makedirs(os.path.join(base, "images"), exist_ok=True); os.makedirs(os.path.join(base, "dpt"), exist_ok=True)
    low = torch.rand(1, 3, 6, 8, generator=g); dlow = torch.rand(1, 1, 6, 8, generator=g)
    for v in range(V):
        low = (low + 0.08 * torch.randn(1, 3, 6, 8, generator=g)).clamp(0, 1)          # slowly changing "video"
        dlow = (dlow + 0.05 * torch.randn(1, 1, 6, 8, generator=g)).clamp(0, 1)
        img = (up(low, (H, W))[0].permute(1, 2, 0).numpy() * 255).astype(np.uint8)
        Image.fromarray(img).save(os.path.join(base, "images", "%03d.png" % v))
        dpt = (up(dlow, (hd, wd))[0] * 3.0 + 2.0).numpy().astype(np.float32)              # (1, hd, wd), DPT range
        np.savez(os.path.join(base, "dpt", "depth_%03d.npz" % v), pred=dpt)
    fx = 0.6 * W
    np.savez(os.path.join(base, "intrinsics.npz"), K=np.array([[fx, 0, W / 2], [0, fx, H / 2], [0, 0, 1]], np.float32))


class _Writer:
    """stand-in for torch.utils.tensorboard.SummaryWriter: records the scalars train.py logs"""
    log = []

    def __init__(self, *a, **k):
        pass

    def add_scalar(self, tag, value, step=None):
        try:
            v = float(value)
        except Exception:
            v = float(np.asarray(value).reshape(-1)[0])
        _Writer.log.append((tag, v, step))

    def add_image(self, *a, **k):
        pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workdir"); ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--normal-loss", action="store_true", help="rendering.normal_loss: True (the renderer computes the normal term)")
    a = ap.parse_args()
    import torch
    from oracle import ref_harness as RH
    assert RH.available(), "oracle/_ref missing (oracle/vendor_ref.py)"
    work = os.path.abspath(a.workdir)
    scene = os.path.join(work, "data", "Test", "images")
    write_scene(scene)
    RH.install_stubs()
    tb = types.ModuleType("torch.utils.tensorboard"); tb.SummaryWriter = _Writer
    sys.modules["torch.utils.tensorboard"] = tb
    REF = RH.REF
    sys.path.insert(0, REF)
    import dataloading as dl                                            # the reference's loader, unchanged
    cfg = dl.load_config(os.path.join(REF, "configs", "Test", "images.yaml"), os.path.join(REF, "configs", "default.yaml"))
    cfg["dataloading"].update(path=os.path.join(work, "data", "Test"), n_workers=0, resize_factor=None)
    cfg["training"].update(out_dir=os.path.join(work, "out"), n_training_points=256, print_every=1, visualize_every=7, checkpoint_every=5,
                           backup_every=-1, validate_every=-1, eval_pose_every=-1, eval_img_every=1, scheduling_start=1, scheduling_epoch=1,
                           scheduling_mode="reset", vis_resolution=[24, 32], vis_geo=False, log_scale_shift_per_view=True, length_smooth=1)
    cfg["rendering"]["num_points"] = 64
    cfg["rendering"]["normal_loss"] = bool(a.normal_loss)
    os.makedirs(cfg["training"]["out_dir"], exist_ok=True)
    # ---- the INTEGRATION.md binding: reference `model` package, hot-path classes redirected ----
    mdl = RH.import_reference("cuda" if torch.cuda.is_available() else "cpu")
    calls = {"train_step": 0, "render_visdata": 0}
    if a.impl == "ours":
        import nope_nerf_b200.model as ours
        for name in ("nope_nerf", "Trainer", "Renderer", "get_model", "OfficialStaticNerf", "LearnPose", "LearnFocal", "Trainer_pose", "Learn_Distortion"):
            setattr(mdl, name, getattr(ours, name))
        T = ours.Trainer
    else:
        T = mdl.Trainer
    o_step, o_vis = T.train_step, T.render_visdata

    def step(self, *x, **k):
        calls["train_step"] += 1
        return o_step(self, *x, **k)

    def vis(self, *x, **k):
        calls["render_visdata"] += 1
        return o_vis(self, *x, **k)
    T.train_step, T.render_visdata = step, vis
    import train as ref_train                                           # oracle/_ref/train.py, unmodified
    assert os.path.abspath(ref_train.__file__).startswith(REF)
    ref_train.train(cfg)
    if torch.cuda.is_available(): torch.cuda.synchronize()
    out = cfg["training"]["out_dir"]
    losses = [v for (t, v, s) in _Writer.log if t == "train/loss"]
    psnr = [v for (t, v, s) in _Writer.log if t == "train/psnr"]
    scal = sorted({t for (t, v, s) in _Writer.log})
    vis_dirs = sorted(d for d in os.listdir(os.path.join(out, "rendering")) if d.endswith("_vis"))
    ck = {f: os.path.getsize(os.path.join(out, f)) for f in ("model.pt", "model_pose.pt", "model_distortion.pt") if os.path.exists(os.path.join(out, f))}
    sd = torch.load(os.path.join(out, "model.pt"), map_location="cpu", weights_only=False) if "model.pt" in ck else {}
    res = {"impl": a.impl, "trainer_class": "%s.%s" % (T.__module__, T.__name__), "train_steps": calls["train_step"], "render_visdata_calls": calls["render_visdata"],
           "loss_first": losses[0] if losses else None, "loss_last": losses[-1] if losses else None, "losses_finite": bool(np.all(np.isfinite(losses))),
           "n_loss_logs": len(losses), "train_psnr_per_epoch": psnr, "scalar_tags": scal, "vis_dirs": vis_dirs,
           "vis_files": sorted(os.listdir(os.path.join(out, "rendering", vis_dirs[0]))) if vis_dirs else [], "checkpoints": ck,
           "checkpoint_keys": sorted(sd.keys())[:8], "n_model_tensors": len(sd.get("model", {})), "checkpoint_it": sd.get("it"),
           "model_keys_shapes": [[k, list(v.shape)] for k, v in sorted(sd.get("model", {}).items())],
           "optimizer_state_entries": len(sd.get("optimizer", {}).get("state", {})),
           "optimizer_state_keys": sorted(next(iter(sd["optimizer"]["state"].values())).keys()) if sd.get("optimizer", {}).get("state") else [],
           "optimizer_step": float(next(iter(sd["optimizer"]["state"].values()))["step"]) if sd.get("optimizer", {}).get("state") else None}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""PSNR parity of the product against the LIVE reference (oracle/_ref = unmodified copy of the reference tree) on a GPU
(BASELINE.json: "matched PSNR (+-0.1 dB)", train.py:277-295 reports PSNR from l2_mean).

    python tools/psnr_parity.py [--steps 2000] [--seeds 3] [--out gpurun_out/psnr_parity.json]

Teacher scene (SURVEY.md 8(d)): V views of a fixed random OfficialStaticNerf (seed 7) at known smooth poses, rendered by the
REFERENCE renderer in eval mode; the DPT prior of a view is the teacher's rendered depth.  Per seed, three students start from
the same parameters (the reference's torch init under that seed, r = t = 0), see the same view order, and train K steps of
render + rgb L1 + depth L1:
  ref    the reference's own Trainer.train_step on cuda                        (oracle/ref_harness.RefRig)
  eager  nope_nerf_b200 Trainer(use_cuda_graph=False, pixel_sampler='randperm') same RNG call order as the reference
  graph  nope_nerf_b200 Trainer()  (default: whole-step CUDA graph, in-graph hash pixel sampler -> different draws)
All three arms re-seed the device generator identically before training.  Rounding differences grow along a training
trajectory (gate flips, Adam's sign-like first steps), so the arms are compared through what BASELINE.json names: the PSNR of
every training view rendered from the student's own learned pose (each arm with its own renderer), plus the train PSNR
(-10 log10 l2_mean, train.py:277) averaged over the last 100 steps.  The reference's own seed-to-seed spread is printed next
to the differences.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_harness as RH  # noqa: E402


def psnr(a, b):
    return float(-10.0 * torch.log10(((a.float() - b.float()) ** 2).mean()))


def ref_render(rmdl, model, c2w, cam, H, W, dpt, dev):
    """reference render_visdata's loop (model/training.py:100-125): eval mode, no jitter, 1024-pixel chunks"""
    from model.common import arange_pixels
    world_mat = torch.inverse(c2w).unsqueeze(0)
    p_idx = torch.arange(H * W, device=dev)
    _, pixels = arange_pixels(resolution=(H, W))
    pixels = pixels.to(dev)
    rgb, dep = [], []
    with torch.no_grad():
        for px, pi in zip(torch.split(pixels, 1024, dim=1), torch.split(p_idx, 1024, dim=0)):
            out = model(px, pi, cam, world_mat, torch.eye(4, device=dev)[None], "nope_nerf", add_noise=False, eval_mode=True, it=0,
                        depth_img=dpt, img_size=(H, W))
            rgb.append(out["rgb"]); dep.append(out["depth_pred"])
    return torch.cat(rgb, dim=1).view(H, W, 3), torch.cat(dep, dim=0).view(H, W)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000); ap.add_argument("--seeds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "psnr_parity.json"))
    ap.add_argument("--arms", default="eager,graph", help="comma list of: eager, graph, eager_simt (exact-fp32 engine), eager_torchadam "
                    "(torch.optim.Adam.step instead of the fused one)")
    a = ap.parse_args()
    ARMS = {"eager": dict(use_cuda_graph=False, pixel_sampler="randperm"), "graph": dict(),
            "eager_simt": dict(use_cuda_graph=False, pixel_sampler="randperm", _engine="simt"),
            "eager_torchadam": dict(use_cuda_graph=False, pixel_sampler="randperm", fused_adam=False)}
    arms = [(n, dict(ARMS[n])) for n in a.arms.split(",")]
    assert RH.available(), "oracle/_ref missing (oracle/vendor_ref.py)"
    dev = torch.device("cuda")
    H, W, hd, wd, V, N, S = 60, 80, 60, 80, 6, 512, 64
    kx, ky = 1.2, -1.6
    cam = torch.diag(torch.tensor([kx, ky, -1.0, 1.0]))[None].to(dev)
    cfg = RH.load_default_cfg()
    RH.set_cfg(cfg, {"training.pc_weight": [0.0, 0.0], "training.rgb_s_weight": [0.0, 0.0], "training.n_training_points": N,
                     "rendering.num_points": S, "training.vis_reprojection_every": 10 ** 9})
    rmdl = RH.import_reference("cuda")
    # ---- teacher scene, rendered by the reference ----
    torch.manual_seed(7)
    t_rig = RH.RefRig(cfg, V, "cuda")
    with torch.no_grad():
        # a default-init field renders a nearly uniform grey volume: amplify the teacher's heads so the scene has structure
        # (mostly empty space with coloured blobs); the students keep the reference's stock initialisation
        t_rig.net.fc_density.weight.mul_(12.0); t_rig.net.fc_density.bias.fill_(-1.5)
        t_rig.net.fc_rgb.weight.mul_(12.0)
        for v in range(V):
            t_rig.pose.r[v] = torch.tensor([0.02 * v, -0.015 * v, 0.01 * v]); t_rig.pose.t[v] = torch.tensor([0.05 * v, 0.02 * v, -0.03 * v])
    ones = torch.ones(1, 1, hd, wd, device=dev)
    frames = []
    for v in range(V):
        rgb, depth = ref_render(rmdl, t_rig.model, t_rig.pose(v).detach(), cam, H, W, ones, dev)
        frames.append((rgb.permute(2, 0, 1).contiguous()[None], depth.contiguous()[None]))       # (1,3,H,W), (1,hd,wd)
    del t_rig

    def data_of(v):
        return {"img": frames[v][0], "img.idx": torch.tensor([v]), "img.dpt": frames[v][1], "img.camera_mat": cam.cpu(),
                "img.scale_mat": torch.eye(4)[None]}

    import nope_nerf_b200.model as mdl
    results = []
    eval_at = set(range(max(a.steps - 400, 1), a.steps + 1, 100)) | {a.steps}       # PSNR = mean over the last checkpoints (Adam at a
    for seed in range(a.seeds):                                                     # constant lr keeps the final state jittering)
        order = [int(x) for x in torch.randint(0, V, (a.steps,), generator=torch.Generator().manual_seed(100 + seed))]
        torch.manual_seed(42 + seed)
        rig = RH.RefRig(cfg, V, "cuda")
        init = rig.state()
        rec = {"seed": seed}
        # ---- ref ----
        torch.manual_seed(1000 + seed)
        t0 = time.perf_counter(); l2 = []; ckpt = []

        def ref_eval():
            ps = []
            for v in range(V):
                img, _ = ref_render(rmdl, rig.model, rig.pose(v).detach(), cam, H, W, frames[v][1][None], dev)
                ps.append(psnr(img, frames[v][0][0].permute(1, 2, 0)))
            return ps
        for it, v in enumerate(order):
            ld = rig.train_step(data_of(v), it=it + 1, epoch=0, scheduling_start=10 ** 9)
            l2.append(float(ld["l2_mean"].detach()))
            if it + 1 in eval_at:
                st_rng = torch.cuda.get_rng_state(); ckpt.append(ref_eval()); torch.cuda.set_rng_state(st_rng)
        torch.cuda.synchronize(); rec["ref_s_per_step"] = (time.perf_counter() - t0) / a.steps
        rec["ref"] = {"psnr_views": [round(x, 3) for x in ckpt[-1]], "psnr_mean": float(np.mean(ckpt)), "psnr_final": float(np.mean(ckpt[-1])),
                      "train_psnr_last500": float(-10 * np.log10(np.mean(l2[-500:])))}
        del rig
        # ---- product, two modes ----
        for arm, kw0 in arms:
            kw = dict(kw0)
            from nope_nerf_b200 import ops as _ops
            _ops.set_default_engine(kw.pop("_engine", "tc"))
            pcfg = json.loads(json.dumps(cfg)); pcfg["extract_images"] = {"resolution": (H, W)}
            net = mdl.OfficialStaticNerf(pcfg)
            net.load_state_dict({k: v.clone() for k, v in init["net"].items()})
            rend = mdl.Renderer(net, pcfg["rendering"], device=dev)
            model = mdl.get_model(rend, pcfg, device=dev)
            pose = mdl.LearnPose(V, True, True, pcfg).to(dev); dist = mdl.Learn_Distortion(V, True, True, pcfg).to(dev)
            tr = pcfg["training"]
            trainer = mdl.Trainer(model, torch.optim.Adam(model.parameters(), lr=tr["learning_rate"]), tr, device=dev,
                                  optimizer_pose=torch.optim.Adam(pose.parameters(), lr=tr["pose_lr"]), pose_param_net=pose,
                                  optimizer_distortion=torch.optim.Adam(dist.parameters(), lr=tr["distortion_lr"]), distortion_net=dist, **kw)
            ex = mdl.Extract_Images(rend, pcfg, device=dev, render_type="nope_nerf")

            def our_eval():
                ps = []
                for v in range(V):
                    with torch.no_grad():
                        img, _ = ex.render_frame(pose(v).detach(), cam[0], H, W)
                    ps.append(psnr(img.reshape(H, W, 3), frames[v][0][0].permute(1, 2, 0)))
                return ps
            torch.manual_seed(1000 + seed)
            t0 = time.perf_counter(); l2 = []; ckpt = []
            for it, v in enumerate(order):
                ld = trainer.train_step(data_of(v), it=it + 1, epoch=0, scheduling_start=10 ** 9, render_path=None)
                l2.append(ld["l2_mean"])
                if it + 1 in eval_at:
                    ckpt.append(our_eval())                   # (the evaluation draws no random numbers)
            l2 = [float(x) for x in torch.stack([x.detach().reshape(()) for x in l2]).cpu()]
            torch.cuda.synchronize(); s_per = (time.perf_counter() - t0) / a.steps
            rec[arm] = {"psnr_views": [round(x, 3) for x in ckpt[-1]], "psnr_mean": float(np.mean(ckpt)), "psnr_final": float(np.mean(ckpt[-1])),
                        "train_psnr_last500": float(-10 * np.log10(np.mean(l2[-500:]))), "s_per_step": s_per,
                        "dpsnr_vs_ref_db": float(np.mean(ckpt) - rec["ref"]["psnr_mean"]),
                        "dtrain_psnr_vs_ref_db": float(-10 * np.log10(np.mean(l2[-500:])) - rec["ref"]["train_psnr_last500"])}
            del trainer, ex
        results.append(rec)
        print(json.dumps(rec), flush=True)
    refs = np.array([r["ref"]["psnr_mean"] for r in results])
    se = lambda x: float(np.std(x, ddof=1) / np.sqrt(len(x))) if len(x) > 1 else float("nan")
    summ = {"steps": a.steps, "seeds": a.seeds, "scene": "teacher scene %dx%d, V=%d, %d rays x %d samples, render + rgb L1 + depth L1" % (H, W, V, N, S),
            "psnr": "mean over all views and the checkpoints at steps %s" % sorted(eval_at),
            "ref_psnr_mean": float(refs.mean()), "ref_psnr_seed_std": float(refs.std(ddof=1)) if len(refs) > 1 else None,
            "ref_train_psnr_last500_mean": float(np.mean([r["ref"]["train_psnr_last500"] for r in results]))}
    for arm, _ in arms:
        d = np.array([r[arm]["dpsnr_vs_ref_db"] for r in results]); dt = np.array([r[arm]["dtrain_psnr_vs_ref_db"] for r in results])
        summ[arm] = {"dpsnr_mean_db": float(d.mean()), "dpsnr_standard_error_db": se(d), "dpsnr_per_seed_db": [round(float(x), 3) for x in d],
                     "psnr_mean": float(np.mean([r[arm]["psnr_mean"] for r in results])),
                     "dtrain_psnr_mean_db": float(dt.mean()), "dtrain_psnr_standard_error_db": se(dt),
                     "train_psnr_last500_mean": float(np.mean([r[arm]["train_psnr_last500"] for r in results]))}
    out = {"summary": summ, "runs": results}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(summ))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Stored reference results of tests/test_gpu_fullsize_ref.py: runs the UNMODIFIED reference (oracle/_ref) on cuda on the inputs
of tests/_fullsize_cases.py and writes what each test compares against to tests/golden/fullsize_*.npz.

    python tools/make_golden_fullsize.py [--out DIR]    # needs oracle/_ref and a GPU; DIR defaults to tests/golden

The reference starts from the parameters tests/_fullsize_cases.start_state builds; the script first checks that they are the
reference's own torch init under the same seed, so the stored results are those of the reference's usual start."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_harness as RH  # noqa: E402
import _fullsize_cases as FC  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def rel(a, b):
    a = a.detach().double().reshape(-1); b = b.detach().double().reshape(-1)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def save(name, **arrs):
    path = os.path.join(OUT, "fullsize_%s.npz" % name)
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrs.items()})
    print(name, os.path.getsize(path), "bytes")


def np_(t):
    return t.detach().float().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def rig_with(cfg_ref, V, state, net_seed):
    """the reference's rig on `state`, after checking that its own init under `net_seed` is state's undamped net"""
    torch.manual_seed(net_seed)
    own = RH.RefRig(cfg_ref, V, "cuda").net.state_dict()
    plain = FC.start_state(FC.default_cfg(), 1, net_seed, 0)["net"]
    assert all(torch.equal(own[k].cpu(), plain[k]) for k in own), "reference init differs from the seeded start state"
    return RH.RefRig(cfg_ref, V, "cuda", state=state)


class patched_draws:
    """torch.randperm / torch.rand return the stored ray_idx / jitter draws (same coupling on both sides of a test)"""
    def __init__(self, HW, N, S, ray_idx, noise):
        self.a = (HW, N, S, ray_idx, noise)

    def __enter__(self):
        HW, N, S, ray_idx, noise = self.a
        self.rp, self.r = torch.randperm, torch.rand
        rp, r = self.rp, self.r
        torch.randperm = lambda n, *a, **k: ray_idx if n == HW else rp(n, *a, **k)
        torch.rand = lambda *a, **k: noise.to(torch.get_default_dtype()) if tuple(a) == (1, N, S) else r(*a, **k)

    def __exit__(self, *exc):
        torch.randperm, torch.rand = self.rp, self.r


def train_cases():
    for name, c in FC.CASES.items():
        cfg_ref = FC.case_cfg(c, RH.load_default_cfg()); V = c["V"]
        state = FC.start_state(FC.case_cfg(c), V, 1234, 99, damp=c.get("damp", False))
        rig = rig_with(cfg_ref, V, state, 1234)
        data = FC.frames(c, 7, 5)
        H, W, N, S = c["H"], c["W"], c["N"], c["S"]
        g = torch.Generator().manual_seed(77)
        ray_idx = torch.randperm(H * W, generator=g)[:N].cuda(); noise = torch.rand(1, N, S, generator=g).cuda()
        with patched_draws(H * W, N, S, ray_idx, noise):
            ld_ref = rig.train_step(data)
            gref = dict(r=rig.pose.r.grad.clone(), t=rig.pose.t.grad.clone(),
                        scales=rig.dist.global_scales.grad.clone() if rig.dist.global_scales.grad is not None else torch.zeros(V, 1).cuda(),
                        shifts=rig.dist.global_shifts.grad.clone(), params=torch.cat([p.grad.reshape(-1) for p in rig.net.parameters()]))
            with RH.fp64_mode():   # the reference's own rounding envelope: the same unmodified code under float64 defaults
                rig64 = RH.RefRig(cfg_ref, V, "cuda", state=state)
                data64 = {k: (v.double() if v.is_floating_point() else v) for k, v in data.items()}
                rig64.train_step(data64)
                g64 = dict(r=rig64.pose.r.grad, t=rig64.pose.t.grad, shifts=rig64.dist.global_shifts.grad,
                           scales=rig64.dist.global_scales.grad if rig64.dist.global_scales.grad is not None else torch.zeros(V, 1).cuda(),
                           params=torch.cat([p.grad.reshape(-1) for p in rig64.net.parameters()]))
                env = {k: rel(gref[k], g64[k]) for k in gref}
                del rig64
        idx = FC.param_sample_idx(gref["params"].numel()).cuda()
        out = {"loss_" + k: float(ld_ref[k]) for k in ("loss", "loss_rgb", "loss_depth", "l2_mean", "loss_pc", "loss_rgb_s")}
        out.update({"g_" + k: np_(gref[k]) for k in ("r", "t", "scales", "shifts")})
        out.update({"env_" + k: env[k] for k in env})
        out.update(params_sample=np_(gref["params"][idx]), params_absmax=float(gref["params"].abs().max()), digest=FC.state_digest(state))
        save("train_" + name, **out)


def render_cases():
    for name in ("C2_render", "C3_ndc"):
        c = FC.CASES[name]; cfg_ref = FC.case_cfg(c, RH.load_default_cfg()); V = c["V"]; idx = 3
        state = FC.start_state(FC.case_cfg(c), V, 4321, 98)
        rig = rig_with(cfg_ref, V, state, 4321)
        data = FC.frames(c, idx, 6)
        H, W, N = c["H"], c["W"], c["N"]
        ray_idx = torch.randperm(H * W, generator=torch.Generator().manual_seed(3))[:N].cuda()
        import model.common as mc                                          # the REFERENCE's helpers (oracle/_ref on sys.path)
        pix = mc.arange_pixels((H, W), 1)[1].cuda()[:, ray_idx]
        cam = data["img.camera_mat"].cuda(); smat = data["img.scale_mat"].cuda(); dpt = data["img.dpt"].cuda().unsqueeze(1)
        with torch.no_grad():
            c2w = rig.pose(idx); sc, sh = rig.dist(idx)
            out = rig.model(pix, ray_idx, cam, torch.inverse(c2w).unsqueeze(0), smat, "nope_nerf", it=0, eval_mode=False, depth_img=dpt * sc + sh,
                            add_noise=False, img_size=(H, W))
        save("render_" + name, rgb=np_(out["rgb"]), depth_pred=np_(out["depth_pred"]), depth_gt=np_(out["depth_gt"]),
             pixels=np_(pix), digest=FC.state_digest(state))


def small_cases(tmp):
    lp = lambda a, b, normalize=True: (a - b).abs().mean()             # stand-in for the LPIPS network (same callable on both sides)
    H, W, V = 48, 64, 4
    # ---- Eval_Images.eval_images ----
    cfg = RH.load_default_cfg(); cfg["extract_images"] = {"resolution": [H, W]}
    state = FC.start_state(FC.default_cfg(), V, 21, 97)
    rig = rig_with(cfg, V, state, 21)
    data = FC.small_scene(H, W, V=V)
    c2ws = torch.stack([rig.pose(i) for i in range(V)]).detach()
    import model.eval_images as rei                                   # the REFERENCE's module (oracle/_ref on sys.path)
    ev = rei.Eval_Images(rig.rend, cfg, use_learnt_poses=True, use_learnt_focal=False, device=torch.device("cuda"), render_type="nope_nerf", c2ws=c2ws)
    d = ev.eval_images(data, os.path.join(tmp, "ev"), None, lp, None)
    save("eval_images", mse=float(d["mse"]), psnr=float(d["psnr"]), ssim=float(d["ssim"]), lpips=float(d["lpips"]), img=np.asarray(d["img"]),
         depth=np.asarray(d["depth"]), depth_gt_shape=np.asarray(tuple(d["depth_gt"].shape)), digest=FC.state_digest(state))
    # ---- Trainer.render_visdata (nope_nerf view) ----
    cfg = RH.load_default_cfg(); cfg["training"]["vis_geo"] = False
    state = FC.start_state(FC.default_cfg(), V, 22, 96)
    rig = rig_with(cfg, V, state, 22)
    os.makedirs(os.path.join(tmp, "vis"), exist_ok=True)
    img = rig.trainer.render_visdata(FC.small_scene(H, W, V=V), (H, W), 0, os.path.join(tmp, "vis"))
    save("render_visdata", img=np.asarray(img), digest=FC.state_digest(state))
    # ---- geometry field: infer_occ / gradient, phong renderer ----
    cfg = RH.load_default_cfg()
    state = FC.start_state(FC.default_cfg(), V, 31, 95, geo=True)
    rig = rig_with(cfg, V, state, 31)
    p = ((torch.rand(4096, 3, generator=torch.Generator().manual_seed(8)) - 0.5) * 6.0).cuda()
    _, s_ref = rig.net.infer_occ(p)
    g_ref = rig.net.gradient(p.clone(), 0).detach()
    save("infer_occ", logit=np_(s_ref), grad=np_(g_ref), grad_shape=np.asarray(g_ref.shape), digest=FC.state_digest(state))
    Hs, Ws = 24, 32
    data = FC.small_scene(Hs, Ws, V=V)
    import model.common as mc
    pixels = mc.arange_pixels((Hs, Ws), 1)[1].cuda()
    cam = data["img.camera_mat"].cuda(); smat = data["img.scale_mat"].cuda()

    def shade(view):
        with torch.no_grad():
            c2w = rig.pose(view)
        o = rig.model(pixels, None, cam, torch.inverse(c2w).unsqueeze(0), smat, "phong_renderer", it=0, eval_mode=True, depth_img=None,
                      add_noise=False, img_size=(Hs, Ws))
        return o["rgb"].detach().reshape(-1, 3), o["rgb_surf"].detach().reshape(-1, 3)
    view = 1
    for v in range(V):          # a view whose camera sits in free space and sees a surface (random field: not every pose does)
        if float((shade(v)[1].abs().sum(1) > 0).float().mean()) > 0.02:
            view = v; break
    rgb, surf = shade(view)
    data["img.idx"] = torch.tensor([view])
    os.makedirs(os.path.join(tmp, "geo"), exist_ok=True)
    img = rig.trainer.render_visdata(data, (Hs, Ws), 0, os.path.join(tmp, "geo"))   # default config: vis_geo = True
    save("phong", view=view, rgb=np_(rgb), rgb_surf=np_(surf), img=np.asarray(img), digest=FC.state_digest(state))
    # ---- invariant depth loss, one train step ----
    N, S = 256, 64
    cfg = RH.load_default_cfg()
    FC.set_cfg(cfg, {"training.depth_loss_type": "invariant", "training.pc_weight": [0.0, 0.0], "training.rgb_s_weight": [0.0, 0.0],
                     "training.n_training_points": N, "rendering.num_points": S, "training.vis_reprojection_every": 10 ** 9})
    state = FC.start_state(FC.default_cfg(), V, 77, 94)
    rig = rig_with(cfg, V, state, 77)
    data = FC.small_scene(H, W, V=V)
    g = torch.Generator().manual_seed(78)
    ray_idx = torch.randperm(H * W, generator=g)[:N].cuda(); noise = torch.rand(1, N, S, generator=g).cuda()
    with patched_draws(H * W, N, S, ray_idx, noise):
        ld = rig.train_step(data)
    save("invariant_depth", loss=float(ld["loss"]), loss_depth=float(ld["loss_depth"]), g_r=np_(rig.pose.r.grad), g_t=np_(rig.pose.t.grad),
         g_shifts=np_(rig.dist.global_shifts.grad), digest=FC.state_digest(state))


if __name__ == "__main__":
    import tempfile
    assert RH.available() and torch.cuda.is_available(), "needs oracle/_ref and a GPU"
    if "--out" in sys.argv:
        OUT = os.path.abspath(sys.argv[sys.argv.index("--out") + 1])
    os.makedirs(OUT, exist_ok=True)
    RH.import_reference("cuda")
    train_cases()
    render_cases()
    with tempfile.TemporaryDirectory() as tmp:
        small_cases(tmp)

#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the UNMODIFIED reference (torch CPU, fp32).

Needs a reference checkout ($NOPE_NERF_REFERENCE, default ../reference beside this repository):  python tools/make_golden.py
The GPU box never runs this; it only reads the committed .npz fixtures.

Harness-side shims (reference files untouched, SURVEY.md section 8(c)):
  * empty stub modules for imageio / matplotlib / timm (imported at module scope by
    model/training.py:7, model/common.py:4, DPT/dpt/vit.py:3; no arithmetic),
  * torch.Tensor.cuda -> identity (hard-coded .cuda() in model/losses.py:84,162-194),
  * model.common.transform_to_world default device -> cpu (model/common.py:113).
Weights are numpy-seeded (oracle.init_params) so fixtures stay small: only inputs,
outputs and gradient digests are stored.
"""
import os, sys, types
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("NOPE_NERF_REFERENCE", os.path.join(os.path.dirname(ROOT), "reference"))
sys.path.insert(0, ROOT)


def install_stubs():
    for name in ("imageio", "matplotlib", "matplotlib.pyplot", "timm", "lpips", "skimage", "skimage.metrics"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            sys.modules[name] = m
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.modules["skimage"].metrics = sys.modules["skimage.metrics"]


def import_reference():
    import torch
    install_stubs()
    if REF not in sys.path:
        sys.path.insert(0, REF)
    torch.Tensor.cuda = lambda self, *a, **k: self
    import model as mdl
    import model.common as mc
    import model.training as mt
    _orig = mc.transform_to_world

    def ttw(pixels, depth, camera_mat, world_mat=None, scale_mat=None, invert=True, device=torch.device("cpu")):
        return _orig(pixels, depth, camera_mat, world_mat, scale_mat, invert, device)
    mc.transform_to_world = ttw
    mt.transform_to_world = ttw
    return mdl


def digest(name, g, rng_seed=0, k=64):
    """Small fingerprint of a big gradient tensor: sum, L2 norm, |.|max and k fixed samples."""
    g = np.asarray(g, dtype=np.float64).reshape(-1)
    idx = np.random.default_rng(abs(hash(name)) % (2 ** 31) if False else rng_seed).integers(0, g.size, size=min(k, g.size))
    return dict(sum=g.sum(), l2=np.sqrt((g * g).sum()), amax=np.abs(g).max(), idx=idx, val=g[idx])


def base_cfg():
    import yaml
    with open(os.path.join(REF, "configs", "default.yaml")) as f:
        return yaml.safe_load(f)


def build_model(mdl, cfg, P):
    import torch
    net = mdl.OfficialStaticNerf(cfg)
    sd = {k: torch.from_numpy(np.array(v)) for k, v in P.items()}
    net.load_state_dict(sd)
    rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cpu"))
    model = mdl.nope_nerf(cfg, rend, None, device=torch.device("cpu"))
    return net, rend, model


def case_render(mdl, name, overrides, N, S, H, W, hd, wd, eval_mode, add_noise, seed, pose_mode, prior="dpt", hf_damp=False, hidden_dim=256):
    """nope_nerf.forward (model/network.py:19-33 -> model/rendering.py:36-167) + autograd grads; hidden_dim = model.hidden_dim."""
    import torch
    from oracle import nerf_oracle as O
    cfg = base_cfg()
    for k, v in overrides.items():
        sec, key = k.split(".")
        cfg[sec][key] = v
    cfg["rendering"]["num_points"] = S
    cfg["model"]["hidden_dim"] = hidden_dim
    P = O.init_params(seed=seed, D=hidden_dim, white_bkgd=cfg["rendering"]["white_background"], hf_damp=hf_damp)
    net, rend, model = build_model(mdl, cfg, P)
    rng = np.random.default_rng(seed + 1)
    V = 5
    if pose_mode == "zero":
        r = np.zeros((V, 3), np.float32); t = np.zeros((V, 3), np.float32)
    else:
        r = rng.normal(0, 0.05, (V, 3)).astype(np.float32); t = rng.normal(0, 0.05, (V, 3)).astype(np.float32)
    init = None
    if pose_mode == "init":
        init = np.tile(np.eye(4, dtype=np.float32), (V, 1, 1))
        for v in range(V):
            init[v] = O.make_c2w(rng.normal(0, 0.3, 3).astype(np.float32), rng.normal(0, 0.2, 3).astype(np.float32))
    pose = mdl.LearnPose(V, True, True, cfg, init_c2w=None if init is None else torch.from_numpy(init))
    with torch.no_grad():
        pose.r.copy_(torch.from_numpy(r)); pose.t.copy_(torch.from_numpy(t))
    cam_id = 2
    fx = 0.6 * W
    kx, ky = 2 * fx / W, -2 * fx / H
    kxy = torch.tensor([kx, ky], dtype=torch.float32, requires_grad=True)        # d/dK as LearnFocal needs it (training.py:247-252)
    z4 = torch.zeros(4); one = torch.ones(1)
    camera_mat = torch.cat([kxy[0:1], z4, kxy[1:2], z4, -one, z4, one]).view(1, 4, 4)
    scale_mat = torch.eye(4).unsqueeze(0)
    if prior == "dpt":
        dpt = rng.uniform(0.6, 7.2, (hd, wd)).astype(np.float32)
    else:
        dpt = np.ones((hd, wd), np.float32)
    ray_idx = rng.permutation(H * W)[:N].astype(np.int64)
    scale = torch.tensor(1.07, requires_grad=True); shift = torch.tensor(-0.03, requires_grad=True)
    depth_img = (torch.from_numpy(dpt)[None, None] * scale + shift)
    c2w = pose(cam_id)
    c2w.retain_grad()
    world_mat = torch.inverse(c2w).unsqueeze(0)
    p_full = mdl.common.arange_pixels((H, W), 1)[1] if hasattr(mdl, "common") else None
    import model.common as mc
    p_full = mc.arange_pixels((H, W), 1)[1]
    p = p_full[:, torch.from_numpy(ray_idx)]
    noise = None
    if add_noise:
        torch.manual_seed(1000 + seed)
        noise = torch.rand(1, N, S).numpy()[0].copy()
        torch.manual_seed(1000 + seed)
    if eval_mode:
        net.eval()
    out = model(p, torch.from_numpy(ray_idx), camera_mat, world_mat, scale_mat, "nope_nerf", it=0,
                eval_mode=eval_mode, depth_img=depth_img, add_noise=add_noise, img_size=(H, W))
    g_rgb = rng.normal(0, 1, (1, N, 3)).astype(np.float32)
    nm = out["depth_pred"].shape[0]
    g_dp = rng.normal(0, 1, (nm,)).astype(np.float32); g_dg = rng.normal(0, 1, (nm,)).astype(np.float32)
    scalar = (out["rgb"] * torch.from_numpy(g_rgb)).sum() + (out["depth_pred"] * torch.from_numpy(g_dp)).sum() \
        + (out["depth_gt"] * torch.from_numpy(g_dg)).sum()
    scalar.backward()
    rec = dict(N=N, S=S, H=H, W=W, seed=seed, cam_id=cam_id, kx=kx, ky=ky, eval_mode=eval_mode, hf_damp=hf_damp, hidden_dim=hidden_dim,
               add_noise=add_noise, r=r, t=t, dpt=dpt, ray_idx=ray_idx, scale=1.07, shift=-0.03,
               pixels=p[0].detach().numpy(), c2w=c2w.detach().numpy(),
               g_rgb=g_rgb[0], g_dp=g_dp, g_dg=g_dg,
               rgb=out["rgb"][0].detach().numpy(), depth_pred=out["depth_pred"].detach().numpy(),
               depth_gt=out["depth_gt"].detach().numpy(), z_vals=out["z_vals"].detach().numpy(),
               alpha=out["alpha"].detach().numpy(),
               grad_c2w=c2w.grad.numpy(), grad_r=pose.r.grad.numpy(), grad_t=pose.t.grad.numpy(),
               grad_scale=scale.grad.numpy(), grad_shift=shift.grad.numpy(), grad_kxy=kxy.grad.numpy())
    if init is not None:
        rec["init_c2w"] = init
    if noise is not None:
        rec["noise"] = noise
    for k, v in overrides.items():
        rec["cfg." + k] = np.array(v)
    for n, prm in net.named_parameters():
        d = digest(n, prm.grad.numpy())
        for kk, vv in d.items():
            rec["pg.%s.%s" % (n, kk)] = vv
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **rec)
    print("wrote", name, "rgb[0]", rec["rgb"][0], "grad_r", rec["grad_r"][cam_id])


def case_mlp(mdl, name, M, dist_alpha, occ, seed, hidden_dim=256):
    """OfficialStaticNerf.forward (model/official_nerf.py:69-96) + grads wrt inputs/params."""
    import torch
    from oracle import nerf_oracle as O
    cfg = base_cfg(); cfg["rendering"]["dist_alpha"] = dist_alpha; cfg["model"]["occ_activation"] = occ
    cfg["model"]["hidden_dim"] = hidden_dim
    P = O.init_params(seed=seed, D=hidden_dim)
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in P.items()})
    rng = np.random.default_rng(seed + 7)
    pts = rng.uniform(-4, 4, (M, 3)).astype(np.float32); dirs = rng.normal(0, 1, (M, 3)).astype(np.float32)
    dirs /= np.linalg.norm(dirs, axis=-1, keepdims=True)
    tp = torch.from_numpy(pts).requires_grad_(True); td = torch.from_numpy(dirs).requires_grad_(True)
    rgb, a = net(tp, td, return_addocc=True)
    g_rgb = rng.normal(0, 1, (M, 3)).astype(np.float32); g_a = rng.normal(0, 1, (M, 1)).astype(np.float32)
    ((rgb * torch.from_numpy(g_rgb)).sum() + (a * torch.from_numpy(g_a)).sum()).backward()
    rec = dict(M=M, seed=seed, dist_alpha=dist_alpha, occ=occ, hidden_dim=hidden_dim, pts=pts, dirs=dirs, g_rgb=g_rgb, g_a=g_a[:, 0],
               rgb=rgb.detach().numpy(), a=a.detach().numpy()[:, 0], g_pts=tp.grad.numpy(), g_dirs=td.grad.numpy(),
               enc=__import__("model.official_nerf", fromlist=["x"]).encode_position(torch.from_numpy(pts), 10, True).numpy())
    for n, prm in net.named_parameters():
        for kk, vv in digest(n, prm.grad.numpy()).items():
            rec["pg.%s.%s" % (n, kk)] = vv
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **rec)
    print("wrote", name)


def case_pose(mdl, name):
    """LearnPose.forward (model/poses.py:23-31) incl. r = 0 and init_c2w."""
    import torch
    rng = np.random.default_rng(5)
    V = 4
    r = rng.normal(0, 0.4, (V, 3)).astype(np.float32); r[0] = 0
    t = rng.normal(0, 0.4, (V, 3)).astype(np.float32)
    init = np.tile(np.eye(4, dtype=np.float32), (V, 1, 1))
    from oracle import nerf_oracle as O
    for v in range(V):
        init[v] = O.make_c2w(rng.normal(0, 0.5, 3).astype(np.float32), rng.normal(0, 0.5, 3).astype(np.float32))
    G = rng.normal(0, 1, (V, 4, 4)).astype(np.float32)
    rec = dict(r=r, t=t, init=init, G=G)
    for use_init in (0, 1):
        pose = mdl.LearnPose(V, True, True, None, init_c2w=torch.from_numpy(init) if use_init else None)
        with torch.no_grad():
            pose.r.copy_(torch.from_numpy(r)); pose.t.copy_(torch.from_numpy(t))
        c2ws = []
        for v in range(V):
            c = pose(v); c2ws.append(c.detach().numpy())
            (c * torch.from_numpy(G[v])).sum().backward()
        rec["c2w_%d" % use_init] = np.stack(c2ws)
        rec["gr_%d" % use_init] = pose.r.grad.numpy().copy(); rec["gt_%d" % use_init] = pose.t.grad.numpy().copy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **rec)
    print("wrote", name)


def case_train_step(mdl, name, with_ref, steps, N, S, H, W, hd, wd, seed, last_view=False, learn_focal=False, training=None,
                    hidden_dim=256):
    """Trainer.train_step (model/training.py:67-97) for `steps` iterations on one synthetic pair; `training` overrides keys of
    cfg['training'] (stored as cfg.training.<key>); hidden_dim = model.hidden_dim (stored as hidden_dim)."""
    import torch
    from oracle import nerf_oracle as O
    cfg = base_cfg()
    cfg["training"].update(training or {})
    cfg["rendering"]["num_points"] = S; cfg["training"]["n_training_points"] = N
    if not with_ref:
        cfg["training"]["pc_weight"] = [0.0, 0.0]; cfg["training"]["rgb_s_weight"] = [0.0, 0.0]
    cfg["training"]["vis_reprojection_every"] = 10 ** 9
    cfg["model"]["hidden_dim"] = hidden_dim
    P = O.init_params(seed=seed, D=hidden_dim)
    net, rend, model = build_model(mdl, cfg, P)
    V = 4
    rng = np.random.default_rng(seed + 3)
    r0 = rng.normal(0, 0.05, (V, 3)).astype(np.float32); t0 = rng.normal(0, 0.05, (V, 3)).astype(np.float32)
    pose = mdl.LearnPose(V, True, True, cfg)
    dist = mdl.Learn_Distortion(V, True, True, cfg)
    with torch.no_grad():
        pose.r.copy_(torch.from_numpy(r0)); pose.t.copy_(torch.from_numpy(t0))
        dist.global_scales.copy_(torch.from_numpy(rng.uniform(0.9, 1.1, (V, 1)).astype(np.float32)))
        dist.global_shifts.copy_(torch.from_numpy(rng.uniform(-0.1, 0.1, (V, 1)).astype(np.float32)))
    sc0 = dist.global_scales.detach().numpy().copy(); sh0 = dist.global_shifts.detach().numpy().copy()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    opt_p = torch.optim.Adam(pose.parameters(), lr=5e-4)
    opt_d = torch.optim.Adam(dist.parameters(), lr=5e-4)
    fx = 0.6 * W
    kx, ky = 2 * fx / W, -2 * fx / H
    focal = opt_f = None
    if learn_focal:                                      # train.py:140-147: init_focal = [K00, -K11], order 2, Adam(focal_lr)
        focal = mdl.LearnFocal(True, False, order=2, init_focal=[kx * 1.03, -ky * 0.98])
        opt_f = torch.optim.Adam(focal.parameters(), lr=cfg["training"]["focal_lr"])
    trainer = mdl.Trainer(model, opt, cfg["training"], device=torch.device("cpu"), optimizer_pose=opt_p,
                          pose_param_net=pose, optimizer_distortion=opt_d, distortion_net=dist, optimizer_focal=opt_f,
                          focal_net=focal)
    cam = np.array([[kx, 0, 0, 0], [0, ky, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], np.float32)
    idx = V - 1 if last_view else 1
    ref_idx = idx - 1 if last_view else idx + 1
    img = rng.uniform(0, 1, (1, 3, H, W)).astype(np.float32); ref = rng.uniform(0, 1, (1, 3, H, W)).astype(np.float32)
    # smooth-ish prior so chamfer nearest neighbours are not degenerate
    dpt = rng.uniform(0.6, 7.2, (1, hd, wd)).astype(np.float32); rdpt = rng.uniform(0.6, 7.2, (1, hd, wd)).astype(np.float32)
    data = {"img": torch.from_numpy(img), "img.idx": torch.tensor([idx]), "img.dpt": torch.from_numpy(dpt),
            "img.camera_mat": torch.from_numpy(cam)[None], "img.scale_mat": torch.eye(4)[None],
            "img.ref_imgs": torch.from_numpy(ref), "img.ref_dpts": torch.from_numpy(rdpt),
            "img.ref_idxs": torch.tensor([ref_idx])}
    rec = dict(N=N, S=S, H=H, W=W, V=V, seed=seed, idx=idx, ref_idx=ref_idx, kx=kx, ky=ky, img=img[0], ref=ref[0],
               dpt=dpt[0], rdpt=rdpt[0], r0=r0, t0=t0, scales0=sc0, shifts0=sh0, steps=steps, with_ref=with_ref, hidden_dim=hidden_dim)
    for k, v in (training or {}).items():
        rec["cfg.training." + k] = np.array(v)
    if learn_focal:
        rec["focal0"] = np.array([focal.fx.item(), focal.fy.item()], np.float32)
    for it in range(steps):
        torch.manual_seed(500 + it)
        ray_idx = torch.randperm(H * W)[:N].numpy().copy()
        noise = torch.rand(1, N, S).numpy()[0].copy()
        torch.manual_seed(500 + it)
        ld = trainer.train_step(data, it=it + 1, epoch=0, scheduling_start=10000, render_path="/tmp")
        rec["ray_idx_%d" % it] = ray_idx; rec["noise_%d" % it] = noise
        for k, v in ld.items():
            rec["loss_%d.%s" % (it, k)] = np.asarray(v.detach().numpy() if hasattr(v, "detach") else v, dtype=np.float32)
        rec["grad_r_%d" % it] = pose.r.grad.numpy().copy(); rec["grad_t_%d" % it] = pose.t.grad.numpy().copy()
        gz = lambda prm: np.zeros(tuple(prm.shape), np.float32) if prm.grad is None else prm.grad.numpy().copy()
        rec["grad_scales_%d" % it] = gz(dist.global_scales)   # None when the view's scale is the fixed constant
        rec["grad_shifts_%d" % it] = gz(dist.global_shifts)
        if learn_focal:
            rec["grad_focal_%d" % it] = np.array([focal.fx.grad.item(), focal.fy.grad.item()], np.float32)
        for n, prm in net.named_parameters():
            for kk, vv in digest(n, prm.grad.numpy()).items():
                rec["pg_%d.%s.%s" % (it, n, kk)] = vv
    rec["r_end"] = pose.r.detach().numpy(); rec["t_end"] = pose.t.detach().numpy()
    rec["scales_end"] = dist.global_scales.detach().numpy(); rec["shifts_end"] = dist.global_shifts.detach().numpy()
    if learn_focal:
        rec["focal_end"] = np.array([focal.fx.item(), focal.fy.item()], np.float32)
    for n, prm in net.named_parameters():
        for kk, vv in digest(n, prm.detach().numpy()).items():
            rec["pend.%s.%s" % (n, kk)] = vv
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **rec)
    print("wrote", name, {k: float(v) for k, v in ld.items() if hasattr(v, "item") and v.numel() == 1})


def case_chamfer(mdl, name, P, Q, seed):
    """Loss.get_pc_loss 'dense' (model/losses.py:114-148) + autograd on two random point clouds (incl. one exact duplicate pair
    and one tie, which torch.argmin resolves to the first index)."""
    import torch
    from model.losses import Loss
    cfg = base_cfg()
    rng = np.random.default_rng(seed)
    X = rng.normal(0, 1, (P, 3)).astype(np.float32); Y = rng.normal(0, 1, (Q, 3)).astype(np.float32)
    Y[5] = X[7]                      # zero distance: the norm's sub-gradient is 0 there
    Y[11] = Y[3]                     # duplicated target: ties -> first index
    Xt = torch.from_numpy(X)[None].requires_grad_(True); Yt = torch.from_numpy(Y)[None].requires_grad_(True)
    loss = Loss(cfg["training"]).get_pc_loss(Xt, Yt)
    loss.backward()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), X=X, Y=Y, loss=np.float32(loss.item()),
                        gX=Xt.grad[0].numpy(), gY=Yt.grad[0].numpy())
    print("wrote", name, float(loss))


def case_normals(mdl, name, overrides, D, N, S, H, W, hd, wd, seed):
    """rendering.normal_loss: True (model/rendering.py:133-141, OfficialStaticNerf.gradient with create_graph): the reference's
    nope_nerf forward in fp32 and again in fp64 on the same draws (the sample jitter and the neighbour offsets, recorded from the fp32
    run), diff_norm and the gradients of a fixed random weighting of it with respect to the MLP (sampled entries), r, t, the camera
    matrix's kx / ky, scale and shift."""
    import torch
    from oracle import nerf_oracle as O
    cfg = base_cfg()
    for k, v in overrides.items():
        sec, key = k.split(".")
        cfg[sec][key] = v
    cfg["rendering"]["num_points"] = S
    cfg["rendering"]["normal_loss"] = True
    cfg["model"]["hidden_dim"] = D
    P = O.init_params(seed=seed, D=D, white_bkgd=cfg["rendering"]["white_background"], hf_damp=True)
    rng = np.random.default_rng(seed + 1)
    V, cam_id = 4, 1
    r = rng.normal(0, 0.05, (V, 3)).astype(np.float32); t = rng.normal(0, 0.05, (V, 3)).astype(np.float32)
    fx = 0.6 * W
    kx, ky = 2 * fx / W, -2 * fx / H
    dpt = rng.uniform(0.6, 7.2, (hd, wd)).astype(np.float32)
    ray_idx = rng.permutation(H * W)[:N].astype(np.int64)
    import model.common as mc
    pix = mc.arange_pixels((H, W), 1)[1][:, torch.from_numpy(ray_idx)]

    draws = []

    def run(dtype):
        torch.set_default_dtype(dtype)
        real_rand, real_rand_like = torch.rand, torch.rand_like
        k = [0]

        def replay(real):
            def f(*a, **kw):
                if dtype == torch.float32:
                    v = real(*a, **kw); draws.append(v.detach().clone()); return v
                v = draws[k[0]].to(dtype); k[0] += 1
                return v
            return f
        torch.rand, torch.rand_like = replay(real_rand), replay(real_rand_like)
        try:
            net, rend, model = build_model(mdl, cfg, P)
            net.to(dtype)
            pose = mdl.LearnPose(V, True, True, cfg).to(dtype)
            with torch.no_grad():
                pose.r.copy_(torch.from_numpy(r)); pose.t.copy_(torch.from_numpy(t))
            kxy = torch.tensor([kx, ky], dtype=dtype, requires_grad=True)
            z4 = torch.zeros(4); one = torch.ones(1)
            camera_mat = torch.cat([kxy[0:1], z4, kxy[1:2], z4, -one, z4, one]).view(1, 4, 4)
            scale = torch.tensor(1.07, dtype=dtype, requires_grad=True); shift = torch.tensor(-0.03, dtype=dtype, requires_grad=True)
            depth_img = torch.from_numpy(dpt).to(dtype)[None, None] * scale + shift
            world_mat = torch.inverse(pose(cam_id)).unsqueeze(0)
            out = model(pix.to(dtype), torch.from_numpy(ray_idx), camera_mat, world_mat, torch.eye(4).unsqueeze(0), "nope_nerf", it=0,
                        eval_mode=False, depth_img=depth_img, add_noise=True, img_size=(H, W))
        finally:
            torch.rand, torch.rand_like = real_rand, real_rand_like
        dn = out["normal"]
        wts = torch.from_numpy(np.random.default_rng(seed + 2).normal(0, 1, dn.shape[0])).to(dtype)
        (dn * wts).sum().backward()
        res = dict(diff_norm=dn.detach().numpy().astype(np.float64), wts=wts.numpy().astype(np.float64),
                   grad_r=pose.r.grad[cam_id].numpy().astype(np.float64), grad_t=pose.t.grad[cam_id].numpy().astype(np.float64),
                   grad_kxy=kxy.grad.numpy().astype(np.float64), grad_scale=scale.grad.numpy().astype(np.float64),
                   grad_shift=shift.grad.numpy().astype(np.float64))
        for n_, prm in net.named_parameters():
            g_ = torch.zeros_like(prm) if prm.grad is None else prm.grad          # biases and the rgb branch do not enter diff_norm
            res["pg." + n_] = g_.numpy().reshape(-1).astype(np.float64)
        torch.set_default_dtype(torch.float32)
        return res

    r32 = run(torch.float32)
    r64 = run(torch.float64)
    uniform = cfg["rendering"]["sample_option"] == "uniform"
    rec = dict(N=N, S=S, H=H, W=W, hd=hd, wd=wd, seed=seed, hidden_dim=D, cam_id=cam_id, kx=kx, ky=ky, r=r, t=t, dpt=dpt, ray_idx=ray_idx,
               scale=1.07, shift=-0.03, pixels=pix[0].numpy(), wts=r32["wts"].astype(np.float32),
               noise=draws[0].numpy()[0] if uniform else np.zeros((N, S), np.float32), nbr=draws[1 if uniform else 0].numpy())
    for k, v in overrides.items():
        rec["cfg." + k] = np.array(v)
    sel = np.random.default_rng(seed + 3)
    for key in r32:
        if key == "wts":
            continue
        a32, a64 = r32[key], r64[key]
        if key.startswith("pg.") and a32.size > 256:
            idx = np.sort(sel.choice(a32.size, 256, replace=False))
            rec[key + ".idx"] = idx; a32, a64 = a32[idx], a64[idx]
        rec[key + ".f32"] = a32.astype(np.float32); rec[key + ".f64"] = a64
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **rec)
    print("wrote", name, "valid", rec["diff_norm.f32"].shape[0], "|dn32-dn64|", np.abs(r32["diff_norm"] - r64["diff_norm"]).max(),
          "grad_t", rec["grad_t.f32"], rec["grad_t.f64"])


def main():
    mdl = import_reference()
    os.makedirs(os.path.join(ROOT, "tests", "golden"), exist_ok=True)
    which = sys.argv[1:] or ["mlp", "pose", "render", "chamfer", "train"]
    if "mlp" in which:
        case_mlp(mdl, "mlp_alpha_softplus", 96, False, "softplus", 11)
        case_mlp(mdl, "mlp_sigma_relu", 96, True, "relu", 12)
    if "pose" in which:
        case_pose(mdl, "pose_expmap")
    if "render" in which:
        case_render(mdl, "render_tanks_noise", {}, N=24, S=128, H=30, W=40, hd=12, wd=21, eval_mode=False,
                    add_noise=True, seed=21, pose_mode="rand")
        case_render(mdl, "render_tanks_r0", {}, N=32, S=32, H=30, W=40, hd=12, wd=21, eval_mode=False,
                    add_noise=True, seed=22, pose_mode="zero")
        case_render(mdl, "render_eval_ones", {}, N=32, S=64, H=27, W=48, hd=27, wd=48, eval_mode=True,
                    add_noise=False, seed=23, pose_mode="init", prior="ones")
        case_render(mdl, "render_ndc_distalpha", {"rendering.sample_option": "ndc", "rendering.dist_alpha": True,
                                                  "rendering.depth_range": [0.0, 1.0]},
                    N=24, S=128, H=30, W=40, hd=16, wd=20, eval_mode=False, add_noise=True, seed=24, pose_mode="rand")
        case_render(mdl, "render_oddflags", {"rendering.white_background": True, "rendering.use_ray_dir": False,
                                             "rendering.normalise_ray": False, "model.occ_activation": "relu"},
                    N=32, S=32, H=30, W=40, hd=12, wd=21, eval_mode=False, add_noise=False, seed=25, pose_mode="rand")
    if "render" in which or "damped" in which:
        # well-conditioned twins (oracle.init_params(hf_damp=True)): gradients gated at 1e-4 without an envelope term
        case_render(mdl, "render_tanks_noise_damped", {}, N=24, S=128, H=30, W=40, hd=12, wd=21, eval_mode=False,
                    add_noise=True, seed=21, pose_mode="rand", hf_damp=True)
        case_render(mdl, "render_ndc_distalpha_damped", {"rendering.sample_option": "ndc", "rendering.dist_alpha": True,
                                                         "rendering.depth_range": [0.0, 1.0]},
                    N=24, S=128, H=30, W=40, hd=16, wd=20, eval_mode=False, add_noise=True, seed=24, pose_mode="rand", hf_damp=True)
        case_render(mdl, "render_oddflags_damped", {"rendering.white_background": True, "rendering.use_ray_dir": False,
                                                    "rendering.normalise_ray": False, "model.occ_activation": "relu"},
                    N=32, S=32, H=30, W=40, hd=12, wd=21, eval_mode=False, add_noise=False, seed=25, pose_mode="rand", hf_damp=True)
        case_render(mdl, "render_eval_ones_damped", {}, N=32, S=64, H=27, W=48, hd=27, wd=48, eval_mode=True,
                    add_noise=False, seed=23, pose_mode="init", prior="ones", hf_damp=True)
    if "chamfer" in which:
        case_chamfer(mdl, "chamfer_dense", 193, 160, 41)
    if "train" in which:
        case_train_step(mdl, "train_render_only", False, steps=2, N=48, S=32, H=24, W=32, hd=16, wd=24, seed=31)
        case_train_step(mdl, "train_full_losses", True, steps=2, N=48, S=32, H=24, W=32, hd=16, wd=24, seed=32)
        case_train_step(mdl, "train_full_lastview", True, steps=1, N=48, S=32, H=24, W=32, hd=16, wd=24, seed=33,
                        last_view=True)
    if "focal" in which or "train" in which:
        case_train_step(mdl, "train_learn_focal", True, steps=2, N=48, S=32, H=24, W=32, hd=16, wd=24, seed=34, learn_focal=True)
    if "refopts" in which:
        # training.with_ssim / training.detach_ref_img: False; a 32x48 DPT map gives an 8x12 low-resolution grid with interior columns
        case_train_step(mdl, "train_full_ssim", True, steps=2, N=48, S=32, H=24, W=32, hd=32, wd=48, seed=35, training={"with_ssim": True})
        case_train_step(mdl, "train_full_undetached", True, steps=2, N=48, S=32, H=24, W=32, hd=32, wd=48, seed=36,
                        training={"detach_ref_img": False})
        case_train_step(mdl, "train_full_undetached_lastview", True, steps=1, N=48, S=32, H=24, W=32, hd=32, wd=48, seed=37, last_view=True,
                        training={"detach_ref_img": False})
        case_train_step(mdl, "train_full_ssim_undetached_shiftfirst", True, steps=1, N=48, S=32, H=24, W=32, hd=32, wd=48, seed=38,
                        training={"with_ssim": True, "detach_ref_img": False, "shift_first": True})

    if "hidden" in which:
        # model.hidden_dim 128 and 64: the field's trunk / rgb hidden layers D and D/2 wide (official_nerf.py:11-37)
        for D in (128, 64):
            case_mlp(mdl, "mlp_alpha_softplus_d%d" % D, 96, False, "softplus", 11, hidden_dim=D)
            for damp in (False, True):
                sfx = "_d%d%s" % (D, "_damped" if damp else "")
                case_render(mdl, "render_tanks_noise" + sfx, {}, N=24, S=128, H=30, W=40, hd=12, wd=21, eval_mode=False,
                            add_noise=True, seed=21, pose_mode="rand", hf_damp=damp, hidden_dim=D)
                case_render(mdl, "render_ndc_distalpha" + sfx, {"rendering.sample_option": "ndc", "rendering.dist_alpha": True,
                                                                "rendering.depth_range": [0.0, 1.0]},
                            N=24, S=128, H=30, W=40, hd=16, wd=20, eval_mode=False, add_noise=True, seed=24, pose_mode="rand", hf_damp=damp,
                            hidden_dim=D)
            case_train_step(mdl, "train_full_losses_d%d" % D, True, steps=2, N=48, S=32, H=24, W=32, hd=16, wd=24, seed=32, hidden_dim=D)

    if "samples" in which:
        # rendering.num_points outside {32, 64, 128, 256}: rays that straddle the 64-row blocks of the tensor-core engine, and S > 256
        for damp in (False, True):
            sfx = "_damped" if damp else ""
            case_render(mdl, "render_tanks_noise_s48" + sfx, {}, N=32, S=48, H=30, W=40, hd=12, wd=21, eval_mode=False,
                        add_noise=True, seed=51, pose_mode="rand", hf_damp=damp)
            case_render(mdl, "render_ndc_distalpha_s96" + sfx, {"rendering.sample_option": "ndc", "rendering.dist_alpha": True,
                                                                "rendering.depth_range": [0.0, 1.0]},
                        N=24, S=96, H=30, W=40, hd=16, wd=20, eval_mode=False, add_noise=True, seed=52, pose_mode="rand", hf_damp=damp)
            case_render(mdl, "render_eval_ones_s200" + sfx, {}, N=24, S=200, H=27, W=48, hd=27, wd=48, eval_mode=True,
                        add_noise=False, seed=53, pose_mode="init", prior="ones", hf_damp=damp)
            case_render(mdl, "render_tanks_noise_s300" + sfx, {}, N=24, S=300, H=30, W=40, hd=12, wd=21, eval_mode=False,
                        add_noise=True, seed=54, pose_mode="rand", hf_damp=damp)
        case_train_step(mdl, "train_full_losses_s48", True, steps=2, N=48, S=48, H=24, W=32, hd=16, wd=24, seed=55)
        case_train_step(mdl, "train_render_only_s300", False, steps=2, N=24, S=300, H=24, W=32, hd=16, wd=24, seed=56)

    if "normals" in which:
        # rendering.normal_loss: True -- diff_norm and its gradients through the second derivative of the field
        for D in (64, 256):
            case_normals(mdl, "normals_uniform_d%d" % D, {}, D=D, N=64, S=32, H=30, W=40, hd=12, wd=21, seed=61)
            case_normals(mdl, "normals_ndc_d%d" % D, {"rendering.sample_option": "ndc", "rendering.dist_alpha": True,
                                                      "rendering.depth_range": [0.0, 1.0]},
                         D=D, N=64, S=32, H=30, W=40, hd=16, wd=20, seed=62)


if __name__ == "__main__":
    main()

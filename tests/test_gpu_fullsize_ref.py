"""Full-size parity against the reference on cuda, through its stored results (tests/golden/fullsize_*.npz, written by
tools/make_golden_fullsize.py from the UNMODIFIED reference run on cuda).  BASELINE.json's configs at their REAL sizes:

  C2  1080x1920, DPT 384x672, V=200, 1024 rays x 128 samples, uniform + jitter, rgb L1 + depth L1            (+ full loss set)
  C3  756x1008,  DPT 384x512, V=20,  1024 rays x 128 samples, NDC + dist_alpha, depth loss on 1 - 1/d
  C5  1080x1920, 4096 rays x 128 samples (one rank's view of the 8-view batch), full loss set

Both sides start from the same parameters (the reference's own torch init under a fixed seed, tests/_fullsize_cases.py), see the
same frame pair, the same `ray_idx` (torch.randperm is patched to return a stored draw) and the same jitter (torch.rand likewise),
and run ONE Trainer.train_step.  Compared: every loss scalar, the pose / distortion gradients the step leaves in .grad, a fixed
seeded sample of the MLP gradient, and the rendered rgb / depth of a forward-only call.  The gradient gate is max(1e-4, 3 x
envelope), envelope = |reference fp32 - reference fp64| (the reference itself re-run in float64 on the same inputs = its own
rounding, dominated by ReLU-gate switches, see tests/test_oracle_golden.py::test_render_gate_matched_and_kxy)."""
import os

import numpy as np
import pytest
import torch

from _util import ROOT
import _fullsize_cases as FC

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, "tests", "golden")
REPORT = {}


def _golden(name, state=None):
    g = dict(np.load(os.path.join(GOLDEN, "fullsize_%s.npz" % name)))
    if state is not None:   # the stored results belong to this starting state
        assert abs(FC.state_digest(state) - float(g["digest"])) <= 1e-9 * max(1.0, abs(float(g["digest"]))), name
    return g


def _report(key, **vals):
    import json
    REPORT[key] = {k: float(v) for k, v in vals.items()}
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "parity_fullsize_report.json"), "w") as f:
        json.dump(REPORT, f, indent=1, sort_keys=True)


def rel(a, b):
    a = torch.as_tensor(a).detach().double().reshape(-1).cpu(); b = torch.as_tensor(b).detach().double().reshape(-1).cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def cosine(a, b):
    a = torch.as_tensor(a).detach().double().reshape(-1).cpu(); b = torch.as_tensor(b).detach().double().reshape(-1).cpu()
    return float((a @ b) / (a.norm() * b.norm()).clamp_min(1e-300))


def _ours(cfg, V, state, use_cuda_graph=False):
    import nope_nerf_b200.model as mdl
    dev = torch.device("cuda")
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: v.clone() for k, v in state["net"].items()})
    rend = mdl.Renderer(net, cfg["rendering"], device=dev)
    model = mdl.get_model(rend, cfg, device=dev)
    pose = mdl.LearnPose(V, True, True, cfg).to(dev); dist = mdl.Learn_Distortion(V, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.copy_(state["r"]); pose.t.copy_(state["t"]); dist.global_scales.copy_(state["scales"]); dist.global_shifts.copy_(state["shifts"])
    tr = cfg["training"]
    opt = torch.optim.Adam(model.parameters(), lr=tr["learning_rate"]); opt_p = torch.optim.Adam(pose.parameters(), lr=tr["pose_lr"])
    opt_d = torch.optim.Adam(dist.parameters(), lr=tr["distortion_lr"])
    trainer = mdl.Trainer(model, opt, tr, device=dev, optimizer_pose=opt_p, pose_param_net=pose, optimizer_distortion=opt_d, distortion_net=dist,
                          use_cuda_graph=use_cuda_graph)
    return trainer, net, pose, dist, model


def _patch_draws(monkeypatch, HW, N, S, ray_idx, noise):
    real_randperm, real_rand = torch.randperm, torch.rand
    monkeypatch.setattr(torch, "randperm", lambda n, *a, **k: ray_idx if n == HW else real_randperm(n, *a, **k))
    monkeypatch.setattr(torch, "rand", lambda *a, **k: noise.to(torch.get_default_dtype()) if tuple(a) == (1, N, S) else real_rand(*a, **k))


@pytest.mark.parametrize("name,eng", [(n, "tc") for n in FC.CASES] + [("C2_render", "simt")])   # exact-fp32 engine: one full-size case
def test_train_step_vs_live_reference(name, eng, monkeypatch):
    from nope_nerf_b200 import ops
    ops.set_default_engine(eng)
    c = FC.CASES[name]; cfg = FC.case_cfg(c); V = c["V"]
    state = FC.start_state(cfg, V, 1234, 99, damp=c.get("damp", False))
    gold = _golden("train_" + name, state)
    data = FC.frames(c, 7, 5)
    H, W, N, S = c["H"], c["W"], c["N"], c["S"]
    g = torch.Generator().manual_seed(77)
    ray_idx = torch.randperm(H * W, generator=g)[:N].cuda(); noise = torch.rand(1, N, S, generator=g).cuda()
    _patch_draws(monkeypatch, H * W, N, S, ray_idx, noise)
    trainer, net, pose, dist, _ = _ours(cfg, V, state)
    ld = trainer.train_step(data, it=1, epoch=0, scheduling_start=10000, render_path="/tmp")
    torch.cuda.synchronize()
    gours = dict(r=pose.r.grad, t=pose.t.grad, scales=dist.global_scales.grad, shifts=dist.global_shifts.grad)
    params = torch.cat([p.grad.reshape(-1) for p in net.parameters()])
    p_sample = params[FC.param_sample_idx(params.numel()).cuda()].double().cpu()
    e = {}
    for k in ("loss", "loss_rgb", "loss_depth", "l2_mean", "loss_pc", "loss_rgb_s"):
        ref = float(gold["loss_" + k]); got = float(ld[k])
        e["loss_" + k] = abs(got - ref) / max(abs(ref), 1e-6) if ref != 0 else abs(got)
    for k in gours:
        e["g_" + k] = rel(gours[k], gold["g_" + k]); e["env_" + k] = float(gold["env_" + k])
    ref_sample = torch.as_tensor(gold["params_sample"]).double()
    e["g_params"] = float((p_sample - ref_sample).abs().max()) / float(gold["params_absmax"]); e["env_params"] = float(gold["env_params"])
    e["cos_params"] = 1.0 - cosine(p_sample, ref_sample)
    _report("%s/%s" % (name, eng), **e)
    for k in ("loss", "loss_rgb", "loss_depth", "l2_mean", "loss_pc", "loss_rgb_s"):
        assert e["loss_" + k] < 1e-5, (k, e)
    # d t = sum of d p over all 131 072 samples, each carrying the 2^9-amplified fp32 rounding of the encoding adjoint: the exact-fp32
    # engine sits at 9e-5, the reference's own fp32 at 3e-5 of its fp64 twin -> 2e-4 floor for d t only
    for k in ("r", "t", "scales", "shifts"):
        floor = 1e-4 if (k != "t" or c.get("damp")) else 2e-4
        assert e["g_" + k] < max(floor, 3 * e["env_" + k]), (k, e)
    assert e["g_params"] < max(5e-4, 3 * e["env_params"]), e
    assert e["cos_params"] < 1e-6, e


@pytest.mark.parametrize("name", ["C2_render", "C3_ndc"])
def test_render_outputs_vs_live_reference(name):
    """nope_nerf.forward at full size: rgb, depth_pred, depth_gt <= 1e-4 of the reference (same ray_idx, no jitter so that the two
    sides need no RNG coupling; eval_mode False keeps the training-path arithmetic)."""
    from nope_nerf_b200 import ops
    from nope_nerf_b200.model import common as mc
    ops.set_default_engine("tc")
    c = FC.CASES[name]; cfg = FC.case_cfg(c); V = c["V"]; idx = 3
    state = FC.start_state(cfg, V, 4321, 98)
    gold = _golden("render_" + name, state)
    data = FC.frames(c, idx, 6)
    H, W, N = c["H"], c["W"], c["N"]
    ray_idx = torch.randperm(H * W, generator=torch.Generator().manual_seed(3))[:N].cuda()
    trainer, net, pose, dist, model = _ours(cfg, V, state)
    pix = mc.arange_pixels((H, W), 1)[1].cuda()[:, ray_idx]
    assert rel(pix, gold["pixels"]) == 0.0
    cam = data["img.camera_mat"].cuda(); smat = data["img.scale_mat"].cuda()
    dpt = data["img.dpt"].cuda().unsqueeze(1)
    with torch.no_grad():
        c2w = pose(idx); sc, sh = dist(idx)
        out = model(pix, ray_idx, cam, torch.inverse(c2w).unsqueeze(0), smat, "nope_nerf", it=0, eval_mode=False, depth_img=dpt * sc + sh,
                    add_noise=False, img_size=(H, W))
    e = dict(rgb=rel(out["rgb"], gold["rgb"]), depth_pred=rel(out["depth_pred"], gold["depth_pred"]),
             depth_gt=rel(out["depth_gt"], gold["depth_gt"]))
    _report("render/%s" % name, **e)
    assert max(e.values()) < 1e-4, e


def test_eval_images_vs_live_reference(tmp_path):
    """Eval_Images.eval_images (model/eval_images.py:46-137): the reference's chunked Renderer loop + pytorch_ssim against ONE
    render_frame call + on-device PSNR / SSIM; same learnt poses, same weights"""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    ops.set_default_engine("tc")
    H, W, V = 48, 64, 4
    cfg = FC.default_cfg()
    cfg["extract_images"] = {"resolution": [H, W]}
    state = FC.start_state(cfg, V, 21, 97)
    gold = _golden("eval_images", state)
    data = FC.small_scene(H, W, V=V)
    lp = lambda a, b, normalize=True: (a - b).abs().mean()             # stand-in for the LPIPS network (same callable on both sides)
    trainer, net, pose, dist, model = _ours(cfg, V, state)
    c2ws = torch.stack([pose(i) for i in range(V)]).detach()
    ev = mdl.Eval_Images(model.renderer, cfg, use_learnt_poses=True, use_learnt_focal=False, device=torch.device("cuda"), render_type="nope_nerf", c2ws=c2ws)
    d = ev.eval_images(data, str(tmp_path / "ours"), None, lp, None)
    e = dict(mse=abs(d["mse"] - float(gold["mse"])) / float(gold["mse"]), psnr=abs(d["psnr"] - float(gold["psnr"])),
             ssim=abs(d["ssim"] - float(gold["ssim"])), lpips=abs(d["lpips"] - float(gold["lpips"])) / float(gold["lpips"]),
             img=float(np.abs(d["img"].astype(np.int32) - gold["img"].astype(np.int32)).max()),
             depth=float(np.abs(d["depth"].astype(np.int32) - gold["depth"].astype(np.int32)).max()))
    _report("eval_images", **e)
    assert e["mse"] < 1e-4 and e["psnr"] < 1e-3 and e["ssim"] < 1e-5 and e["lpips"] < 1e-4 and e["img"] <= 1 and e["depth"] <= 1, e
    assert tuple(d["depth_gt"].shape) == tuple(gold["depth_gt_shape"]) and os.path.exists(str(tmp_path / "ours" / "img_out" / "0001.png"))


def test_render_visdata_vs_live_reference(tmp_path):
    """Trainer.render_visdata (model/training.py:100-163, nope_nerf view): uint8 frame of the reference's 1024-pixel chunk loop against
    the single-call drop-in; files written with the reference's names"""
    from nope_nerf_b200 import ops
    ops.set_default_engine("tc")
    H, W, V = 48, 64, 4
    cfg = FC.default_cfg()
    cfg["training"]["vis_geo"] = False                                 # the phong geometry view is checked below
    state = FC.start_state(cfg, V, 22, 96)
    gold = _golden("render_visdata", state)
    data = FC.small_scene(H, W, V=V)
    (tmp_path / "ours").mkdir()
    trainer, net, pose, dist, model = _ours(cfg, V, state)
    img = trainer.render_visdata(data, (H, W), 0, str(tmp_path / "ours"))
    diff = int(np.abs(img.astype(np.int32) - gold["img"].astype(np.int32)).max())
    _report("render_visdata", max_uint8_diff=diff)
    assert img.shape == gold["img"].shape == (H, W, 3) and diff <= 1, diff
    for f in ("0001_img.png", "0001_depth.png"):
        assert os.path.exists(str(tmp_path / "ours" / f)), f


def test_infer_occ_and_gradient_vs_live_reference():
    """OfficialStaticNerf.infer_occ / gradient (official_nerf.py:46-67: normals of the geometry view = -d logit / d p by autograd in the
    reference, the data-gradient chain of nnb_field_bwd here)"""
    cfg = FC.default_cfg()
    state = FC.start_state(cfg, 4, 31, 95, geo=True)
    gold = _golden("infer_occ", state)
    trainer, net, pose, dist, model = _ours(cfg, 4, state)
    p = ((torch.rand(4096, 3, generator=torch.Generator().manual_seed(8)) - 0.5) * 6.0).cuda()
    _, s = net.infer_occ(p)
    g_our = net.gradient(p.clone(), 0).detach()
    e = dict(logit=rel(s, gold["logit"]), grad=rel(g_our, gold["grad"]), shape=float(tuple(g_our.shape) == tuple(gold["grad_shape"])))
    _report("infer_occ_gradient", **e)
    assert e["shape"] == 1.0 and e["logit"] < 1e-5 and e["grad"] < 1e-4, e


def test_phong_renderer_vs_live_reference(tmp_path):
    """Renderer.phong_renderer (rendering.py:198-271: 512-step ray marching + 8 secant steps + normals + shading) and the geometry view
    of Trainer.render_visdata (training.py:146-161).  A pixel whose occupancy sits at the threshold may resolve to another march step on
    the other implementation: at most 1 % of the pixels may differ by more than 2 / 255."""
    from nope_nerf_b200.model import common as mc
    cfg = FC.default_cfg(); assert cfg["training"]["vis_geo"] is True
    H, W, V = 24, 32, 4
    state = FC.start_state(cfg, V, 31, 95, geo=True)
    gold = _golden("phong", state)
    trainer, net, pose, dist, model = _ours(cfg, V, state)
    data = FC.small_scene(H, W, V=V)
    pixels = mc.arange_pixels((H, W), 1)[1].cuda()
    cam = data["img.camera_mat"].cuda(); smat = data["img.scale_mat"].cuda()
    view = int(gold["view"])   # the reference's first view whose camera sits in free space and sees a surface
    with torch.no_grad():
        c2w = pose(view)
    o = model(pixels, None, cam, torch.inverse(c2w).unsqueeze(0), smat, "phong_renderer", it=0, eval_mode=True, depth_img=None, add_noise=False,
              img_size=(H, W))
    rgb, surf = o["rgb"].detach().reshape(-1, 3).cpu(), o["rgb_surf"].detach().reshape(-1, 3).cpu()
    rgb_ref, surf_ref = torch.as_tensor(gold["rgb"]), torch.as_tensor(gold["rgb_surf"])
    data["img.idx"] = torch.tensor([view])
    hit_ref = (surf_ref.abs().sum(1) > 0)
    bad = ((rgb_ref - rgb).abs().max(1).values > 2.0 / 255) | ((surf_ref - surf).abs().max(1).values > 2.0 / 255)
    e = dict(frac_bad=float(bad.float().mean()), frac_surface=float(hit_ref.float().mean()),
             med_rgb=float((rgb_ref - rgb).abs().median()), med_surf=float((surf_ref - surf).abs().median()))
    _report("phong_renderer", **e)
    assert 0.02 < e["frac_surface"] <= 1.0, e                  # the scene has a visible surface
    assert e["frac_bad"] <= 0.01 and e["med_rgb"] < 1e-4 and e["med_surf"] < 1e-4, e
    # render_visdata with vis_geo (configs/default.yaml:106): returns the shaded view and writes %04d_geo.png
    (tmp_path / "ours").mkdir()
    img = trainer.render_visdata(data, (H, W), 0, str(tmp_path / "ours"))
    far = (np.abs(img.astype(np.int32) - gold["img"].astype(np.int32)).max(-1) > 2).mean()
    assert img.shape == gold["img"].shape and far <= 0.01, far
    assert os.path.exists(str(tmp_path / "ours" / ("%04d_geo.png" % view)))


def test_invariant_depth_loss_vs_live_reference(monkeypatch):
    """training.depth_loss_type = 'invariant' (losses.py:34-57): one Trainer.train_step against the reference, small scene"""
    from nope_nerf_b200 import ops
    ops.set_default_engine("tc")
    H, W, V, N, S = 48, 64, 4, 256, 64
    cfg = FC.default_cfg()
    FC.set_cfg(cfg, {"training.depth_loss_type": "invariant", "training.pc_weight": [0.0, 0.0], "training.rgb_s_weight": [0.0, 0.0],
                     "training.n_training_points": N, "rendering.num_points": S, "training.vis_reprojection_every": 10 ** 9})
    state = FC.start_state(cfg, V, 77, 94)
    gold = _golden("invariant_depth", state)
    data = FC.small_scene(H, W, V=V)
    g = torch.Generator().manual_seed(78)
    ray_idx = torch.randperm(H * W, generator=g)[:N].cuda(); noise = torch.rand(1, N, S, generator=g).cuda()
    _patch_draws(monkeypatch, H * W, N, S, ray_idx, noise)
    trainer, net, pose, dist, _ = _ours(cfg, V, state)
    ld = trainer.train_step(data, it=1, epoch=0, scheduling_start=10000, render_path="/tmp")
    e = dict(loss=abs(float(ld["loss"]) - float(gold["loss"])) / abs(float(gold["loss"])),
             loss_depth=abs(float(ld["loss_depth"]) - float(gold["loss_depth"])) / abs(float(gold["loss_depth"])),
             g_r=rel(pose.r.grad, gold["g_r"]), g_t=rel(pose.t.grad, gold["g_t"]), g_shifts=rel(dist.global_shifts.grad, gold["g_shifts"]))
    _report("invariant_depth", **e)
    assert e["loss"] < 1e-5 and e["loss_depth"] < 1e-5 and e["g_r"] < 2e-3 and e["g_t"] < 2e-3 and e["g_shifts"] < 2e-3, e

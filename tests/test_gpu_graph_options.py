"""Learned focal, scale-invariant depth and pose smoothness on the whole-step CUDA graph (run with -m gpu on an H100).

  * kernel-local checks of nnb_depth_invariant, nnb_pose_smooth and nnb_focal_fwd / nnb_focal_bwd against float64 torch autograd on
    planted inputs;
  * the captured graph step against the general path (Trainer.compute_loss, torch autograd / median / Adam) on identical pixel and
    jitter draws, 8 steps with the loss weights annealing, one capture serving every step;
  * two graph runs from the same seed give the same bits;
  * with 2 GPUs, the ranks of a peer-exchange graph step keep bit-identical parameters (this file is also the 2-rank worker:
    python -m torch.distributed.run --nproc-per-node 2 tests/test_gpu_graph_options.py OUT CASE DP_MODE).
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu
_RAND, _RANDPERM = torch.rand, torch.randperm          # the step tests patch torch.rand / torch.randperm to inject their draws


def _relmax(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


# ---- nnb_depth_invariant ----------------------------------------------------------------------------------------------------
def _invariant_ref64(dp, dg, mask, w, gs):
    """Loss.depth_loss_dpt on the masked rays in float64 (CPU autograd): loss, dense seeds grad_scale * w * dL/d{pred, gt}"""
    from nope_nerf_b200.model.losses import Loss
    m = torch.from_numpy(mask.astype(bool))
    p = torch.from_numpy(dp.astype(np.float64))[m].requires_grad_(True)
    g = torch.from_numpy(dg.astype(np.float64))[m].requires_grad_(True)
    loss = Loss({"depth_loss_type": "invariant"}).depth_loss_dpt(p, g)
    gp, gg = torch.autograd.grad(loss * (w * gs), [p, g])
    sp = np.zeros(dp.shape, np.float64); sg = np.zeros(dp.shape, np.float64)
    sp[mask.astype(bool)] = gp.numpy(); sg[mask.astype(bool)] = gg.numpy()
    return float(loss.detach()), sp, sg


def _planted_depths(case, N=8192):
    rng = np.random.default_rng({"odd": 1, "even": 2, "ties": 3, "one": 4, "small": 5}[case])
    dp = (rng.random(N) * 4 + 1).astype(np.float32)
    dg = (dp * 0.7 + 0.3 + rng.normal(0, 0.2, N)).astype(np.float32)
    mask = (rng.random(N) < 0.7).astype(np.uint8)                    # masked-out rays everywhere
    if case == "odd" and mask.sum() % 2 == 0:
        mask[np.flatnonzero(mask)[0]] = 0
    if case == "even" and mask.sum() % 2 == 1:
        mask[np.flatnonzero(mask)[0]] = 0
    if case == "ties":                                                # many rays share the median value (and others)
        dp = (np.round(dp * 4) / 4).astype(np.float32); dg = (np.round(dg * 8) / 8).astype(np.float32)
    if case == "one":                                                 # all rays masked out but one: s = 0, NaN as in torch
        mask[:] = 0; mask[17] = 1
    if case == "small":
        dp, dg, mask = dp[:7], dg[:7], np.array([1, 0, 1, 1, 0, 1, 1], np.uint8)
    return dp, dg, mask


@pytest.mark.parametrize("case", ["odd", "even", "ties", "one", "small"])
@pytest.mark.parametrize("detach_gt", [False, True])
def test_depth_invariant_kernel_vs_float64(case, detach_gt):
    from nope_nerf_b200 import ops
    dp, dg, mask = _planted_depths(case)
    N = dp.shape[0]; w, gs = 0.37, 0.5
    if case == "ties":
        m = mask.astype(bool); t = np.sort(dp[m])[(m.sum() - 1) // 2]
        assert (dp[m] == t).sum() > 10                               # the median is tied
    rng = np.random.default_rng(9)
    base_p = rng.normal(0, 1e-3, N).astype(np.float32); base_g = rng.normal(0, 1e-3, N).astype(np.float32)
    out = torch.tensor([1.5, 2.0, 3.0, 4.0], device="cuda")
    g_dp = torch.from_numpy(base_p).cuda(); g_dg = torch.from_numpy(base_g).cuda()
    ops.depth_invariant(torch.from_numpy(dp).cuda(), torch.from_numpy(dg).cuda(), torch.from_numpy(mask).cuda(), torch.tensor([w], device="cuda"),
                        out, g_dp, None if detach_gt else g_dg, grad_scale=gs)
    torch.cuda.synchronize()
    loss, sp, sg = _invariant_ref64(dp, dg, mask, w, gs)
    o = out.cpu().numpy().astype(np.float64)
    gp = g_dp.cpu().numpy().astype(np.float64) - base_p; gg = g_dg.cpu().numpy().astype(np.float64) - base_g
    if case == "one":
        assert np.isnan(loss) and np.isnan(o[2]) and np.isnan(o[0])
        assert np.isnan(gp[17]) and np.isnan(sp[17])
        assert np.all(gp[np.arange(N) != 17] == 0)
        return
    assert abs(o[2] - loss) <= 1e-5 * abs(loss), (o[2], loss)
    assert abs(o[0] - (1.5 + w * loss)) <= 1e-5 * abs(1.5 + w * loss) and o[1] == 2.0 and o[3] == 4.0
    assert np.all(gp[mask == 0] == 0) and np.all(gg[mask == 0] == 0)
    assert _relmax(gp, sp) < 1e-4, _relmax(gp, sp)
    if detach_gt:
        assert np.all(gg == 0)
    else:
        assert _relmax(gg, sg) < 1e-4, _relmax(gg, sg)


def test_depth_invariant_zero_weight_writes_nothing():
    from nope_nerf_b200 import ops
    dp, dg, mask = _planted_depths("odd", 1024)
    out = torch.tensor([1.5, 2.0, 3.0, 4.0], device="cuda"); g = torch.zeros(1024, device="cuda")
    ops.depth_invariant(torch.from_numpy(dp).cuda(), torch.from_numpy(dg).cuda(), torch.from_numpy(mask).cuda(), torch.zeros(1, device="cuda"),
                        out, g, g.clone())
    assert out.tolist() == [1.5, 2.0, 3.0, 4.0] and g.abs().max().item() == 0.0


# ---- nnb_pose_smooth --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [2, 3, 200])
def test_pose_smooth_kernel_vs_float64(V):
    from nope_nerf_b200 import ops
    from nope_nerf_b200.model.losses import Loss
    rng = np.random.default_rng(V)
    t = (rng.normal(0, 0.3, (V, 3)) + np.arange(V)[:, None] * 0.05).astype(np.float32)
    if V == 200:
        t[50] = t[49]                                                  # a zero-length step: the norm's sub-gradient is 0
    w1, w2, gs = 0.7, 1.3, 0.5
    base = rng.normal(0, 1e-3, (V, 3)).astype(np.float32)
    g_t = torch.from_numpy(base).cuda(); out2 = torch.zeros(2, device="cuda"); tot = torch.tensor([2.0], device="cuda")
    ops.pose_smooth(torch.from_numpy(t).cuda(), torch.tensor([w1, w2], device="cuda"), out2, loss_total=tot, g_t=g_t, grad_scale=gs)
    torch.cuda.synchronize()
    t64 = torch.from_numpy(t.astype(np.float64)).requires_grad_(True)
    d1, d2 = Loss({"depth_loss_type": "l1"}).get_weight_dist_loss(t64)
    (gs * (w1 * d1 + w2 * d2)).backward()
    o = out2.cpu().numpy()
    assert abs(o[0] - d1.item()) <= 1e-5 * abs(d1.item())
    if V == 2:
        assert np.isnan(o[1]) and np.isnan(d2.item()) and np.isnan(tot.item())   # mean over no difference
    else:
        assert abs(o[1] - d2.item()) <= 1e-5 * abs(d2.item())
        assert abs(tot.item() - (2.0 + gs * (w1 * d1.item() + w2 * d2.item()))) <= 1e-5 * abs(tot.item())
    gk = g_t.cpu().numpy().astype(np.float64) - base
    assert np.all(np.isfinite(gk)) and _relmax(gk, t64.grad.numpy()) < 1e-4, _relmax(gk, t64.grad.numpy())


def test_pose_smooth_zero_weights_write_nothing():
    from nope_nerf_b200 import ops
    out2 = torch.full((2,), 5.0, device="cuda"); g = torch.zeros(6, 3, device="cuda"); tot = torch.ones(1, device="cuda")
    ops.pose_smooth(torch.randn(6, 3, device="cuda"), torch.zeros(2, device="cuda"), out2, loss_total=tot, g_t=g)
    assert out2.tolist() == [5.0, 5.0] and tot.item() == 1.0 and g.abs().max().item() == 0.0


# ---- nnb_focal_fwd / nnb_focal_bwd -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("fx_only", [False, True])
@pytest.mark.parametrize("with_kxy", [False, True])
def test_focal_kernels_vs_float64(order, fx_only, with_kxy):
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    focal = mdl.LearnFocal(True, fx_only, order=order, init_focal=[1.3, 1.7]).cuda()
    fy = None if fx_only else focal.fy
    # forward: the camera matrix the general path builds from LearnFocal (training.py:247-252), bit for bit
    cam = torch.zeros(4, 4, device="cuda")
    ops.focal_fwd(focal.fx.detach(), None if fy is None else fy.detach(), order, cam)
    fxfy = focal(0).detach()
    z4 = torch.zeros(4, device="cuda"); one = torch.ones(1, device="cuda")
    want = torch.cat([fxfy[0:1], z4, -fxfy[1:2], z4, -one, z4, one]).view(4, 4)
    assert torch.equal(cam, want)
    # adjoint against float64 autograd of <g_cam, cam> + g_kxy . (cam[0], cam[5])
    rng = np.random.default_rng(order * 4 + 2 * fx_only + with_kxy)
    g_cam = rng.normal(0, 1, 16).astype(np.float32); g_kxy = rng.normal(0, 1, 2).astype(np.float32)
    fx64 = torch.tensor(float(focal.fx.detach()), dtype=torch.float64, requires_grad=True)
    fy64 = fx64 if fx_only else torch.tensor(float(focal.fy.detach()), dtype=torch.float64, requires_grad=True)
    a, b = (fx64 ** 2, fy64 ** 2) if order == 2 else (fx64, fy64)
    obj = float(g_cam[0]) * a - float(g_cam[5]) * b
    if with_kxy:
        obj = obj + float(g_kxy[0]) * a - float(g_kxy[1]) * b
    obj.backward()
    gf = torch.tensor([0.25, -0.5], device="cuda")                  # the kernel adds into the slot
    ops.focal_bwd(focal.fx.detach(), None if fy is None else fy.detach(), order, torch.from_numpy(g_cam).cuda().view(4, 4),
                  torch.from_numpy(g_kxy).cuda() if with_kxy else None, gf[0], None if fx_only else gf[1])
    got = gf.cpu().numpy().astype(np.float64) - np.array([0.25, -0.5])
    assert abs(got[0] - fx64.grad.item()) <= 1e-6 * max(abs(fx64.grad.item()), 1.0), (got, fx64.grad)
    if fx_only:
        assert got[1] == 0.0
    else:
        assert abs(got[1] - fy64.grad.item()) <= 1e-6 * max(abs(fy64.grad.item()), 1.0), (got, fy64.grad)


# ---- whole training steps ----------------------------------------------------------------------------------------------------
CASES = {
    "focal2": dict(focal=(2, False)),
    "focal2_fx_only": dict(focal=(2, True)),
    "focal1": dict(focal=(1, False)),
    "invariant": dict(inv=True),
    "invariant_detach_gt": dict(inv=True, detach_gt=True),
    "smoothness": dict(smooth=True),
    "all_full_loss": dict(focal=(2, False), inv=True, smooth=True, full=True),
}
H, W, V, N, S, HD, WD = 96, 128, 6, 256, 64, 24, 32
LOSS_KEYS = ("loss", "loss_rgb", "loss_depth", "l2_mean", "loss_pc", "loss_rgb_s", "loss_dist_1st", "loss_dist_2nd")


def _frames_and_draws(steps):
    g = torch.Generator().manual_seed(3)
    up = lambda t, size: torch.nn.functional.interpolate(t, size, mode="bilinear", align_corners=False)
    frames = [dict(img=up(_RAND(1, 3, 12, 16, generator=g), (H, W)), dpt=up(_RAND(1, 1, 6, 8, generator=g), (HD, WD))[0] * 3 + 2)
              for _ in range(V)]
    draws = [(_RANDPERM(H * W, generator=g)[:N], _RAND(N, S, generator=g)) for _ in range(steps)]
    return frames, draws


def _case_cfg(opts):
    from _cfg import default_cfg
    cfg = default_cfg()
    t = cfg["training"]
    if not opts.get("full"):
        t["pc_weight"] = [0.0, 0.0]; t["rgb_s_weight"] = [0.0, 0.0]
    t["n_training_points"] = N; cfg["rendering"]["num_points"] = S
    t["annealing_epochs"] = 10
    if opts.get("inv"):
        t["depth_loss_type"] = "invariant"; t["depth_weight"] = [0.5, 0.1]
    t["detach_gt_depth"] = bool(opts.get("detach_gt", False))
    if opts.get("smooth"):
        t["weight_dist_1st_loss"] = [0.5, 0.1]; t["weight_dist_2nd_loss"] = [2.0, 0.5]
    return cfg


def _build(opts, dev, graph, **kw):
    import nope_nerf_b200.model as mdl
    from oracle import nerf_oracle as O
    cfg = _case_cfg(opts)
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=9, hf_damp=True).items()})
    model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
    pose = mdl.LearnPose(V, True, True, cfg).to(dev); dist = mdl.Learn_Distortion(V, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.copy_(torch.randn(V, 3, generator=torch.Generator().manual_seed(5)) * 0.03)
        pose.t.copy_(torch.randn(V, 3, generator=torch.Generator().manual_seed(6)) * 0.03)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3); opt_p = torch.optim.Adam(pose.parameters(), lr=5e-4)
    opt_d = torch.optim.Adam(dist.parameters(), lr=5e-4)
    focal = opt_f = None
    if opts.get("focal"):
        order, fx_only = opts["focal"]
        # (fx', fy') starts at 1.1 x the dataset's (1.2, 1.6) (LearnFocal stores the root at order 2)
        focal = mdl.LearnFocal(True, fx_only, order=order, init_focal=[1.32, 1.32] if fx_only else [1.32, 1.76]).to(dev)
        opt_f = torch.optim.Adam(focal.parameters(), lr=1e-3)
    tr = mdl.Trainer(model, opt, cfg["training"], device=dev, optimizer_pose=opt_p, pose_param_net=pose, optimizer_distortion=opt_d,
                     distortion_net=dist, optimizer_focal=opt_f, focal_net=focal, use_cuda_graph=graph, pixel_sampler="randperm", **kw)
    return tr, net, pose, dist, focal


def _run(opts, mode, monkeypatch, steps=8, dev=None, view_of=None, **kw):
    """`steps` train steps on injected draws (epochs 0..steps-1, weights anneal from step 4 on); returns losses, parameters and the
    first step's gradients.  mode: 'graph' (captured step), 'eager' (the same kernel sequence launched eagerly every step) or
    'general' (Trainer.compute_loss + torch autograd / Adam: what an eager trainer runs for these options)"""
    dev = dev or torch.device("cuda")
    graph = mode == "graph"
    frames, draws = _frames_and_draws(steps)
    ray_buf = torch.zeros(N, dtype=torch.int64, device=dev); noise_buf = torch.zeros(1, N, S, device=dev)
    monkeypatch.setattr(torch, "randperm", lambda n, device=None: ray_buf)
    monkeypatch.setattr(torch, "rand", lambda *a, **k: noise_buf)
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
    tr, net, pose, dist, focal = _build(opts, dev, graph, **kw)
    if mode == "eager":                                       # route to the graph step, but never capture
        pick = tr._graph_step_or_none

        def eager_graph_step(*a):
            tr.use_cuda_graph = True
            try:
                return pick(*a)
            finally:
                tr.use_cuda_graph = False
        monkeypatch.setattr(tr, "_graph_step_or_none", eager_graph_step)
    losses = []; g_first = None
    for it in range(steps):
        ray_buf.copy_(draws[it][0]); noise_buf[0].copy_(draws[it][1])
        i = view_of(it) if view_of else (it * 2 + 1) % (V - 1)
        data = {"img": frames[i]["img"].to(dev), "img.idx": torch.tensor([i]), "img.dpt": frames[i]["dpt"].to(dev), "img.camera_mat": cam,
                "img.scale_mat": torch.eye(4)[None], "img.ref_imgs": frames[i + 1]["img"].to(dev), "img.ref_dpts": frames[i + 1]["dpt"].to(dev),
                "img.ref_idxs": torch.tensor([i + 1])}
        ld = tr.train_step(data, it=it, epoch=it, scheduling_start=3, render_path=None)
        row = [float(ld[k]) for k in LOSS_KEYS]
        if focal is not None:
            row += [float(ld["focalx"]), float(ld["focaly"])]
        losses.append(row)
        if it == 0:                                           # [MLP | r | t | scales | shifts | fx, fy] of the first step
            buf = tr._gbuf if mode == "general" else tr._peer.reduced
            fg = [] if focal is None else [p.grad.reshape(1) for p in ([focal.fx] if focal.fx_only else [focal.fx, focal.fy])]
            g_first = torch.cat([buf[:net.num_params + 8 * V]] + fg).cpu().numpy().astype(np.float64)
    torch.cuda.synchronize()
    gsteps = [v for v in tr._gsteps.values() if v]
    out = dict(losses=np.array(losses, np.float64), w=net.flat_weights().detach().cpu().numpy().copy(), r=pose.r.detach().cpu().numpy().copy(),
               t=pose.t.detach().cpu().numpy().copy(), scales=dist.global_scales.detach().cpu().numpy().copy(),
               shifts=dist.global_shifts.detach().cpu().numpy().copy(), gsteps=gsteps, steps=steps, tr=tr, g_first=g_first)
    if focal is not None:
        out["focal"] = torch.stack([focal.fx.detach()] + ([] if focal.fx_only else [focal.fy.detach()])).cpu().numpy().copy()
        out["focal_sd_step"] = int(next(iter(tr.optimizer_focal.state_dict()["state"].values()))["step"])
    return out


@pytest.mark.parametrize("case", list(CASES))
def test_graph_replay_equals_eager_on_injected_draws(case, monkeypatch):
    """Mirror of test_gpu_parity.py::test_graph_replay_equals_eager_on_injected_draws for each option: the captured step against the
    same kernel sequence launched eagerly, 8 steps on identical draws with the loss weights annealing (one capture), with the same
    tolerances, plus focal parameters <= 1e-5 relative.  And the new kernels against the general path (torch autograd / median):
    the first step's gradients of every parameter agree to fp32 round-off."""
    from oracle import nerf_oracle as O
    opts = CASES[case]
    ge = _run(opts, "eager", monkeypatch)
    gg = _run(opts, "graph", monkeypatch)
    gp = _run(opts, "general", monkeypatch, steps=1)
    assert len(ge["gsteps"]) == 1 and ge["gsteps"][0].graph is None and ge["gsteps"][0].calls == 8
    assert len(gg["gsteps"]) == 1 and gg["gsteps"][0].graph is not None and gg["gsteps"][0].calls == 8   # ONE capture served every step
    assert not gp["gsteps"]                                                      # eager trainers keep these options on the general path
    le, lg = ge["losses"], gg["losses"]
    if opts.get("full"):
        assert le[:, 4].min() > 0 and le[:, 5].min() > 0
    if opts.get("smooth"):
        assert le[:, 6].min() > 0 and le[:, 7].min() > 0
    n_mlp = ge["tr"].model.renderer.model.num_params
    w0 = O.flatten_params(O.init_params(seed=9, hf_damp=True)).astype(np.float64)
    r0 = (torch.randn(V, 3, generator=torch.Generator().manual_seed(5)) * 0.03).numpy().astype(np.float64)
    t0 = (torch.randn(V, 3, generator=torch.Generator().manual_seed(6)) * 0.03).numpy().astype(np.float64)
    ug, ue = gg["w"] - w0, ge["w"] - w0
    upd = lambda k, p0: np.linalg.norm((gg[k] - p0) - (ge[k] - p0)) / max(np.linalg.norm(ge[k] - p0), 1e-30)
    e = dict(loss=np.abs(le - lg).max() / np.abs(le).max(), w=np.linalg.norm(ug - ue) / np.linalg.norm(ue), r=upd("r", r0), t=upd("t", t0),
             r_abs=np.abs(gg["r"] - ge["r"]).max(), t_abs=np.abs(gg["t"] - ge["t"]).max(), shifts=_relmax(gg["shifts"], ge["shifts"]),
             g1_mlp=_relmax(gg["g_first"][:n_mlp], gp["g_first"][:n_mlp]), g1_pose=_relmax(gg["g_first"][n_mlp:], gp["g_first"][n_mlp:]),
             loss1=np.abs(gg["losses"][0] - gp["losses"][0]).max() / np.abs(gp["losses"][0]).max())
    if "focal" in ge:
        e["focal"] = np.abs(gg["focal"] - ge["focal"]).max() / np.abs(ge["focal"]).max()
        e["g1_focal"] = _relmax(gg["g_first"][n_mlp + 8 * V:], gp["g_first"][n_mlp + 8 * V:])
        assert gg["focal_sd_step"] == ge["focal_sd_step"] == 8                   # focal optimizer state stays torch-compatible
    print(case, e)
    assert e.get("focal", 0.0) <= 1e-5, e
    assert e["loss"] < 1e-5, (e, le, lg)
    assert e["w"] < 2e-2 and e["r"] < 0.1 and e["t"] < 0.1 and e["r_abs"] < 5e-4 and e["t_abs"] < 5e-4 and e["shifts"] < 1e-3, e
    assert e["loss1"] < 1e-5 and e["g1_mlp"] < 1e-4 and e["g1_pose"] < 1e-4 and e.get("g1_focal", 0.0) < 1e-4, e


@pytest.mark.parametrize("case", list(CASES))
def test_graph_step_same_bits_twice(case, monkeypatch):
    a = _run(CASES[case], "graph", monkeypatch, steps=5)
    b = _run(CASES[case], "graph", monkeypatch, steps=5)
    for k in ("losses", "w", "r", "t", "scales", "shifts", "focal"):
        if k in a:
            assert a[k].tobytes() == b[k].tobytes(), (k, np.abs(a[k] - b[k]).max())


def test_default_configuration_layout_unchanged(monkeypatch):
    """without the options the flat gradient buffer, the optimizer state vectors and the graph's node count stay those of the
    default step"""
    from nope_nerf_b200.model.training import Trainer
    r = _run({}, "graph", monkeypatch, steps=3, keep_graph=True)
    tr = r["tr"]; gs = r["gsteps"][0]
    assert tr._gbuf.numel() == tr.model.renderer.model.num_params + 8 * V + 4
    assert gs.steps.numel() == 3 and gs.lrs.numel() == 3 and not (gs.focal or gs.inv or gs.smooth)
    o = _run(CASES["all_full_loss"], "graph", monkeypatch, steps=3, keep_graph=True)
    assert o["tr"]._gbuf.numel() == o["tr"].model.renderer.model.num_params + 8 * V + 8
    nodes = Trainer.graph_kernel_nodes(tr)
    if nodes is not None:
        assert Trainer.graph_kernel_nodes(o["tr"])["kernels"] > nodes["kernels"]


def test_invariant_depth_rays_sharding_keeps_general_path():
    """dp_mode='rays' over several ranks: the reference's median is over the whole batch, so invariant depth stays on the general path"""
    tr, *_ = _build(dict(inv=True), torch.device("cuda"), True)
    tr.world, tr.dp_mode = 2, "rays"
    assert tr._graph_step_or_none({}, 0, 3) is None


# ---- two GPUs ------------------------------------------------------------------------------------------------------------------
def _dp_worker(out, case, dp_mode):
    world = int(os.environ["WORLD_SIZE"]); rank = int(os.environ["RANK"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local); dev = torch.device("cuda", local)
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=dev)
    from nope_nerf_b200 import ops
    ops.set_default_engine("tc")

    class _MP:                                              # pytest's monkeypatch, for the worker process
        def setattr(self, obj, name, val): setattr(obj, name, val)
    view_of = (lambda it: 2 * rank + 1) if dp_mode == "views" else None
    r = _run(CASES[case], "graph", _MP(), steps=4, dev=dev, view_of=view_of, dp_mode=dp_mode, peer_exchange=True)
    assert r["tr"]._peer is not None and r["tr"]._peer.error_flag() == 0 and len(r["gsteps"]) == 1
    chk = torch.from_numpy(np.concatenate([r[k].reshape(-1).astype(np.float64) for k in ("w", "r", "t", "scales", "shifts", "focal") if k in r])).to(dev)
    lst = [torch.zeros_like(chk) for _ in range(world)]
    dist.all_gather(lst, chk)
    assert all(torch.equal(lst[0], x) for x in lst), "ranks diverged"
    if rank == 0:
        np.savez(out, ok=1, finite=int(bool(torch.isfinite(chk).all())))
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("case,dp_mode", [("focal2", "rays"), ("smoothness", "rays"), ("all_full_loss", "views")])
def test_dp_peer_exchange_ranks_bit_identical(case, dp_mode, tmp_path):
    out = str(tmp_path / "dp.npz")
    env = dict(os.environ); env.pop("RANK", None); env.pop("WORLD_SIZE", None); env.pop("LOCAL_RANK", None)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(29500 + (os.getpid() % 500)), os.path.abspath(__file__), out, case, dp_mode]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    z = np.load(out)
    assert int(z["ok"]) == 1 and int(z["finite"]) == 1


if __name__ == "__main__":
    _dp_worker(sys.argv[1], sys.argv[2], sys.argv[3])

"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the C ABI,
against (a) fixtures produced by the unmodified reference (tests/golden, tools/make_golden.py)
and (b) the numpy oracle on the same seeded inputs.

Tolerances (north_star: 1e-4 relative on rendered RGB / depth and on pose gradients):
  outputs   : max-norm error relative to tensor max <= 1e-4
  gradients : <= max(1e-4, 3 x |reference_fp32 - oracle_fp64|).  Gradients flow through
              sin/cos(2^9 p); a 1-ulp difference in p moves them by ~1e-3 on adversarial
              cotangents, so the reference's own fp32 autograd sits that far from the fp64
              truth.  The envelope term is the reference's own rounding, measured per case.
  relu-density configs: the gradient is discontinuous at s = 0, floor 2e-2 (see test_oracle_golden).
"""
import json
import os
import numpy as np
import pytest
import torch

from _util import load_golden, relmax, cfg_from_golden, check_param_digest, ROOT
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu

RENDER_CASES = ["render_tanks_noise", "render_tanks_r0", "render_eval_ones", "render_ndc_distalpha", "render_oddflags",
                "render_tanks_noise_damped", "render_ndc_distalpha_damped", "render_oddflags_damped", "render_eval_ones_damped"]
REPORT = {}


def _report(key, **vals):
    REPORT[key] = {k: float(v) for k, v in vals.items()}
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "parity_report.json"), "w") as f:
        json.dump(REPORT, f, indent=1, sort_keys=True)


def engines():
    from nope_nerf_b200 import _lib as L
    out = [("simt", L.ENGINE_SIMT)]
    if os.environ.get("NNB_SKIP_TC", "0") != "1":
        out.append(("tc", L.ENGINE_TC))
    return out


def cuda(x, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(x))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


def run_case_cuda(g, engine):
    from nope_nerf_b200 import ops, _lib as L
    cfg = cfg_from_golden(g)
    P = O.init_params(seed=int(g["seed"]), white_bkgd=cfg["white_background"], hf_damp=bool(g.get("hf_damp", False)))
    flat = cuda(O.flatten_params(P))
    cam_id = int(g["cam_id"]); N, S, H, W = int(g["N"]), int(g["S"]), int(g["H"]), int(g["W"])
    r, t = cuda(g["r"]), cuda(g["t"])
    init = cuda(g["init_c2w"]) if "init_c2w" in g else None
    c2w = torch.empty(4, 4, device="cuda")
    ops.pose_fwd_raw(r, t, init, cam_id, c2w)
    cam = torch.diag(torch.tensor([float(g["kx"]), float(g["ky"]), -1.0, 1.0])).cuda()
    ndc = cfg["sample_option"] == "ndc"
    flags = ops.flags_from_cfg(cfg, cfg["occ_activation"], eval_=bool(g["eval_mode"]))
    noise = cuda(g["noise"]) if "noise" in g else None
    call = ops.RenderCall(flat, c2w, cam, N=N, S=S, flags=flags, engine=engine, near=0.0 if ndc else cfg["depth_range"][0],
                          far=1.0 if ndc else cfg["depth_range"][1], ray_idx=cuda(g["ray_idx"]), depth_map=cuda(g["dpt"]),
                          scale=torch.tensor([float(g["scale"])]).cuda(), shift=torch.tensor([float(g["shift"])]).cuda(),
                          noise=noise, H=H, W=W, want_z_alpha=True, stash=True)
    mask = call.mask.bool().cpu().numpy()
    out = dict(rgb=call.rgb.cpu().numpy(), depth_pred=call.depth_pred.cpu().numpy()[mask],
               depth_gt=call.depth_gt.cpu().numpy()[mask], z_vals=call.z_vals.cpu().numpy(), alpha=call.alpha.cpu().numpy(),
               c2w=c2w.cpu().numpy())
    gdp = np.zeros(N, np.float32); gdg = np.zeros(N, np.float32)
    gdp[mask] = g["g_dp"]; gdg[mask] = g["g_dg"]
    g_w = torch.zeros(L.NUM_PARAMS, device="cuda"); g_c2w = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
    g_cam = torch.zeros(4, 4, device="cuda")
    call.backward(cuda(g["g_rgb"]), cuda(gdp), cuda(gdg), g_w, g_c2w, g_cam, None, g_ss)
    g_r = torch.zeros_like(r); g_t = torch.zeros_like(t)
    ops.pose_bwd_raw(r, t, init, cam_id, g_c2w, g_r, g_t)
    torch.cuda.synchronize()
    grads = dict(c2w=g_c2w.cpu().numpy(), r=g_r.cpu().numpy()[cam_id], t=g_t.cpu().numpy()[cam_id], ss=g_ss.cpu().numpy(),
                 params=O.unflatten_params(g_w.cpu().numpy()), kxy=np.array([g_cam[0, 0].item(), g_cam[1, 1].item()]))
    return out, grads


def oracle64(g):
    import test_oracle_golden as T
    return T.run_render(g, np.float64)


def oracle32(g):
    import test_oracle_golden as T
    return T.run_render(g, np.float32)


# "-exact": both engines compute MLP weight gradients to fp32 round-off and are held to the same gates
ENGINE_IDS = ["simt-exact", "tc-exact"]


@pytest.mark.parametrize("name", RENDER_CASES)
@pytest.mark.parametrize("eng", ["simt", "tc"], ids=ENGINE_IDS)
def test_render_vs_reference_golden(name, eng):
    """Outputs: <= 1e-4 of the reference.  Gradients, two kinds of case:
      * `*_damped` (oracle.init_params(hf_damp=True): no ReLU-gate switches between fp32 evaluation orders): every gradient
        <= 1e-4 of the fp64 truth (MLP parameter digests 5e-4) and <= max(1e-4, 3 x the reference's own distance from it);
      * default-initialised cases: gradients carry gate-switch noise (tests/test_oracle_golden.py::test_render_gate_matched_and_kxy):
        <= max(1e-4, 3 x envelope), envelope = max(|reference - fp64|, |numpy fp32 - fp64|) = the spread of independent fp32
        evaluations of the same step around the truth."""
    engine = dict(engines()).get(eng)
    if engine is None:
        pytest.skip("engine disabled")
    g = load_golden(name)
    damped = bool(g.get("hf_damp", False))
    out, grads = run_case_cuda(g, engine)
    cam = int(g["cam_id"])
    o64, gr64, g_r64, g_t64, raw, _ = oracle64(g)
    o32, gr32, g_r32, g_t32, _, _ = oracle32(g)
    ss_ref = np.array([g["grad_scale"], g["grad_shift"]])
    ss = lambda gr: np.array([(gr["depth"] * raw).sum(), gr["depth"].sum()])
    # term -> (ours, reference, fp64 oracle, fp32 oracle)
    terms = dict(c2w=(grads["c2w"], g["grad_c2w"], gr64["c2w"], gr32["c2w"]), r=(grads["r"], g["grad_r"][cam], g_r64, g_r32),
                 t=(grads["t"], g["grad_t"][cam], g_t64, g_t32), ss=(grads["ss"], ss_ref, ss(gr64), ss(gr32)),
                 kxy=(grads["kxy"], g["grad_kxy"], gr64["kxy"], gr32["kxy"]))
    e = dict(rgb=relmax(out["rgb"], g["rgb"]), depth_pred=relmax(out["depth_pred"], g["depth_pred"]),
             depth_gt=relmax(out["depth_gt"], g["depth_gt"]), alpha=relmax(out["alpha"], g["alpha"]),
             z=relmax(out["z_vals"], g["z_vals"]), c2w=relmax(out["c2w"], g["c2w"]),
             g_params=check_param_digest(g, grads["params"]), env_params=max(check_param_digest(g, gr64["params"]),
                                                                             check_param_digest(g, gr32["params"])))
    for k, (ours, ref, t64, t32) in terms.items():
        e["g_" + k] = relmax(ours, ref); e["g_%s_vs64" % k] = relmax(ours, t64); e["g_%s_vs32" % k] = relmax(ours, t32)
        e["env_" + k] = max(relmax(t64, ref), relmax(t32, t64)); e["ref64_" + k] = relmax(t64, ref)
    _report("%s/%s" % (name, eng), **e)
    tol = 1e-4
    for k in ("rgb", "depth_pred", "depth_gt", "z", "c2w"):
        assert e[k] < tol, (k, e[k])
    assert e["alpha"] < 2e-4, e["alpha"]
    # render_oddflags (N = 32 rays, un-normalised rays, |p| up to 15): ONE gate switch on a heavy sample moves d t by 2 %; each fp32
    # implementation has its own switches (the exact-fp32 engine shares the numpy oracle's: g_*_vs32 ~ 1e-4), so the envelope of other
    # realisations does not bound the tensor-core engine's -- its `_damped` twin carries the strict gate
    flip_floor = 3e-2 if (name == "render_oddflags") else 1e-4
    for k in terms:
        if damped:
            assert e["g_%s_vs64" % k] < 1e-4, (k, e)
            assert e["g_" + k] < max(1e-4, 3 * e["ref64_" + k]), (k, e)
        else:
            assert e["g_" + k] < max(flip_floor, 3 * e["env_" + k]), (k, e)
    assert e["g_params"] < max(5e-4, 3 * e["env_params"], flip_floor if not damped else 0.0), e


def test_pose_expmap_kernels():
    from nope_nerf_b200 import ops
    g = load_golden("pose_expmap")
    V = g["r"].shape[0]
    r, t = cuda(g["r"]), cuda(g["t"])
    for use_init in (0, 1):
        init = cuda(g["init"]) if use_init else None
        g_r = torch.zeros_like(r); g_t = torch.zeros_like(t)
        for v in range(V):
            c = torch.empty(4, 4, device="cuda")
            ops.pose_fwd_raw(r, t, init, v, c)
            assert relmax(c.cpu().numpy(), g["c2w_%d" % use_init][v]) < 1e-6
            ops.pose_bwd_raw(r, t, init, v, cuda(g["G"][v]), g_r, g_t)
        assert relmax(g_r.cpu().numpy(), g["gr_%d" % use_init]) < 1e-5
        assert relmax(g_t.cpu().numpy(), g["gt_%d" % use_init]) < 1e-5


def _build_trainer(g, engine_name, with_ref):
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    ops.set_default_engine(engine_name)
    cfg = default_cfg()
    S, N, V = int(g["S"]), int(g["N"]), int(g["V"])
    cfg["rendering"]["num_points"] = S; cfg["training"]["n_training_points"] = N
    if not with_ref:
        cfg["training"]["pc_weight"] = [0.0, 0.0]; cfg["training"]["rgb_s_weight"] = [0.0, 0.0]
    cfg["training"]["vis_reprojection_every"] = 10 ** 9
    dev = torch.device("cuda")
    net = mdl.OfficialStaticNerf(cfg)
    P = O.init_params(seed=int(g["seed"]))
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in P.items()})
    rend = mdl.Renderer(net, cfg["rendering"], device=dev)
    model = mdl.get_model(rend, cfg, device=dev)
    pose = mdl.LearnPose(V, True, True, cfg).to(dev)
    dist = mdl.Learn_Distortion(V, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.copy_(cuda(g["r0"])); pose.t.copy_(cuda(g["t0"]))
        dist.global_scales.copy_(cuda(g["scales0"])); dist.global_shifts.copy_(cuda(g["shifts0"]))
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    opt_p = torch.optim.Adam(pose.parameters(), lr=5e-4)
    opt_d = torch.optim.Adam(dist.parameters(), lr=5e-4)
    focal = opt_f = None
    if "focal0" in g:                                   # train.py:140-147
        focal = mdl.LearnFocal(True, False, order=2, init_focal=[1.0, 1.0]).to(dev)
        with torch.no_grad():
            focal.fx.copy_(torch.tensor(float(g["focal0"][0]))); focal.fy.copy_(torch.tensor(float(g["focal0"][1])))
        opt_f = torch.optim.Adam(focal.parameters(), lr=1e-3)
    # use_cuda_graph=False: the golden comparison injects the reference's pixel / jitter draws by patching torch.randperm /
    # torch.rand, which must run eagerly (the same kernel sequence is what the graph path captures)
    trainer = mdl.Trainer(model, opt, cfg["training"], device=dev, optimizer_pose=opt_p, pose_param_net=pose,
                          optimizer_distortion=opt_d, distortion_net=dist, optimizer_focal=opt_f, focal_net=focal, use_cuda_graph=False)
    trainer._test_focal = focal
    return trainer, net, pose, dist


@pytest.mark.parametrize("name,with_ref", [("train_render_only", False), ("train_full_losses", True), ("train_full_lastview", True),
                                           ("train_learn_focal", True)])
@pytest.mark.parametrize("eng", ["simt", "tc"], ids=ENGINE_IDS)
def test_trainer_step_vs_reference_golden(name, with_ref, eng, monkeypatch):
    """Two consecutive reference Trainer.train_step calls."""
    if dict(engines()).get(eng) is None:
        pytest.skip("engine disabled")
    g = load_golden(name)
    trainer, net, pose, dist = _build_trainer(g, eng, with_ref)
    kx, ky = float(g["kx"]), float(g["ky"])
    cam = np.array([[kx, 0, 0, 0], [0, ky, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], np.float32)
    data = {"img": torch.from_numpy(g["img"])[None], "img.idx": torch.tensor([int(g["idx"])]),
            "img.dpt": torch.from_numpy(g["dpt"])[None], "img.camera_mat": torch.from_numpy(cam)[None],
            "img.scale_mat": torch.eye(4)[None], "img.ref_imgs": torch.from_numpy(g["ref"])[None],
            "img.ref_dpts": torch.from_numpy(g["rdpt"])[None], "img.ref_idxs": torch.tensor([int(g["ref_idx"])])}
    state = {"it": 0}
    monkeypatch.setattr(torch, "randperm", lambda n, device=None: cuda(g["ray_idx_%d" % state["it"]]))
    monkeypatch.setattr(torch, "rand", lambda *a, **k: cuda(g["noise_%d" % state["it"]])[None])
    worst = {}
    for it in range(int(g["steps"])):
        state["it"] = it
        ld = trainer.train_step(data, it=it + 1, epoch=0, scheduling_start=10000, render_path="/tmp")
        torch.cuda.synchronize()
        for k in ("loss", "loss_rgb", "loss_depth", "l2_mean", "loss_pc", "loss_rgb_s"):
            ref = float(g["loss_%d.%s" % (it, k)].reshape(-1)[0]); got = float(ld[k].reshape(-1)[0])
            worst["loss_%d_%s" % (it, k)] = abs(got - ref) / max(abs(ref), 1e-3)
        worst["g_r_%d" % it] = relmax(pose.r.grad.cpu().numpy(), g["grad_r_%d" % it])
        worst["g_t_%d" % it] = relmax(pose.t.grad.cpu().numpy(), g["grad_t_%d" % it])
        worst["g_scales_%d" % it] = relmax(dist.global_scales.grad.cpu().numpy(), g["grad_scales_%d" % it])
        worst["g_shifts_%d" % it] = relmax(dist.global_shifts.grad.cpu().numpy(), g["grad_shifts_%d" % it])
        grads = {n: p.grad.cpu().numpy() for n, p in net.named_parameters()}
        worst["g_params_%d" % it] = check_param_digest(g, grads, prefix="pg_%d." % it)
        if "focal0" in g:
            fo = trainer._test_focal
            worst["g_focal_%d" % it] = relmax(np.array([fo.fx.grad.item(), fo.fy.grad.item()]), g["grad_focal_%d" % it])
            for k in ("focalx", "focaly"):
                ref = float(g["loss_%d.%s" % (it, k)].reshape(-1)[0])
                worst["loss_%d_%s" % (it, k)] = abs(float(ld[k]) - ref) / abs(ref)
    worst["r_end"] = relmax(pose.r.detach().cpu().numpy() - g["r0"], g["r_end"] - g["r0"])
    worst["t_end"] = relmax(pose.t.detach().cpu().numpy() - g["t0"], g["t_end"] - g["t0"])
    worst["params_end"] = check_param_digest(g, {n: p.detach().cpu().numpy() for n, p in net.named_parameters()}, prefix="pend.")
    if "focal0" in g:
        fo = trainer._test_focal
        worst["focal_end"] = relmax(np.array([fo.fx.item(), fo.fy.item()]) - g["focal0"], g["focal_end"] - g["focal0"])
    _report("%s/%s" % (name, eng), **worst)
    for k, v in worst.items():
        if k.startswith("loss"):
            assert v < 2e-4, (k, v)        # loss scalars (L1 sums of N*3 terms, fp32)
        elif k.startswith("g_params"):
            assert v < 5e-3, (k, v)        # digests of 24 tensors incl. near-zero ones; second step: parameters already differ by Adam noise
        elif k.startswith("g_"):
            assert v < 2e-3, (k, v)        # first-step gradients incl. the chamfer / warp terms (see module docstring)
        elif k in ("r_end", "t_end", "focal_end"):
            assert v < 5e-2, (k, v)        # Adam's first steps are ~ lr * sign(g): tiny gradients flip easily
        else:
            assert v < 1e-3, (k, v)        # params_end digest


@pytest.mark.parametrize("name", ["render_tanks_noise", "render_ndc_distalpha"])
def test_dropin_autograd_modules(name, monkeypatch):
    """nope_nerf.forward -> Renderer.forward through torch autograd (the drop-in path of network.py / rendering.py)."""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    ops.set_default_engine("simt")
    g = load_golden(name)
    ocfg = cfg_from_golden(g)
    cfg = default_cfg()
    for k in ("dist_alpha", "sample_option", "use_ray_dir", "normalise_ray", "white_background"):
        cfg["rendering"][k] = ocfg[k]
    cfg["rendering"]["depth_range"] = list(ocfg["depth_range"]); cfg["rendering"]["num_points"] = int(g["S"])
    cfg["model"]["occ_activation"] = ocfg["occ_activation"]
    dev = torch.device("cuda")
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=int(g["seed"])).items()})
    model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
    V = g["r"].shape[0]
    pose = mdl.LearnPose(V, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.copy_(cuda(g["r"])); pose.t.copy_(cuda(g["t"]))
    cam_id = int(g["cam_id"]); H, W, N = int(g["H"]), int(g["W"]), int(g["N"])
    scale = torch.tensor(float(g["scale"]), device=dev, requires_grad=True)
    shift = torch.tensor(float(g["shift"]), device=dev, requires_grad=True)
    depth_img = cuda(g["dpt"])[None, None] * scale + shift
    c2w = pose(cam_id)
    world_mat = torch.linalg.inv(c2w).unsqueeze(0)
    cam = torch.diag(torch.tensor([float(g["kx"]), float(g["ky"]), -1.0, 1.0]))[None].to(dev)
    if "noise" in g:
        monkeypatch.setattr(torch, "rand", lambda *a, **k: cuda(g["noise"])[None])
    out = model(cuda(g["pixels"])[None], cuda(g["ray_idx"]), cam, world_mat, torch.eye(4)[None], "nope_nerf", it=0,
                eval_mode=bool(g["eval_mode"]), depth_img=depth_img, add_noise=bool(g["add_noise"]), img_size=(H, W))
    assert set(out.keys()) == {"rgb", "z_vals", "normal", "depth_pred", "depth_gt", "alpha"}
    scalar = (out["rgb"] * cuda(g["g_rgb"])[None]).sum() + (out["depth_pred"] * cuda(g["g_dp"])).sum() + \
        (out["depth_gt"] * cuda(g["g_dg"])).sum()
    scalar.backward()
    e = dict(rgb=relmax(out["rgb"][0].detach().cpu().numpy(), g["rgb"]),
             dp=relmax(out["depth_pred"].detach().cpu().numpy(), g["depth_pred"]),
             g_r=relmax(pose.r.grad.cpu().numpy(), g["grad_r"]), g_t=relmax(pose.t.grad.cpu().numpy(), g["grad_t"]),
             g_scale=abs(scale.grad.item() - float(g["grad_scale"])) / max(abs(float(g["grad_scale"])), 1e-3),
             g_shift=abs(shift.grad.item() - float(g["grad_shift"])) / max(abs(float(g["grad_shift"])), 1e-3),
             g_params=check_param_digest(g, {n: p.grad.cpu().numpy() for n, p in net.named_parameters()}))
    o64, gr64, g_r64, g_t64, raw, _ = oracle64(g)
    env = max(relmax(g_r64, g["grad_r"][cam_id]), relmax(g_t64, g["grad_t"][cam_id]), check_param_digest(g, gr64["params"]))
    e["env"] = env
    _report("dropin/%s" % name, **e)
    assert e["rgb"] < 1e-4 and e["dp"] < 1e-4
    for k in ("g_r", "g_t", "g_scale", "g_shift", "g_params"):
        assert e[k] < max(2e-4, 5 * env), (k, e)      # envelope gate, see module docstring (max over 3 noisy stats -> 5x)


def test_chamfer_vs_oracle():
    from nope_nerf_b200 import ops
    rng = np.random.default_rng(3)
    X = rng.normal(0, 1, (1500, 3)).astype(np.float32); Y = rng.normal(0.1, 1, (1300, 3)).astype(np.float32)
    Y[7] = Y[3]          # exact duplicate: argmin tie -> first index (torch.argmin)
    loss, gX, gY, ixy, iyx = O.chamfer(X.astype(np.float64), Y.astype(np.float64))
    tx = cuda(X).requires_grad_(True); ty = cuda(Y).requires_grad_(True)
    l = ops.chamfer(tx, ty)
    l.backward()
    assert abs(l.item() - loss) < 1e-5 * loss
    assert relmax(tx.grad.cpu().numpy(), gX) < 1e-5 and relmax(ty.grad.cpu().numpy(), gY) < 1e-5


def test_full_size_properties():
    """BASELINE configs[1] size (1024 rays x 128 samples): size-independent properties instead of the
    (too slow) oracle: compositing weights sum <= 1, rgb in [0,1], depth in [near,far], linearity of the
    backward in the cotangent, and SIMT-vs-TC agreement when both engines are present."""
    from nope_nerf_b200 import ops, _lib as L
    N, S, H, W = 1024, 128, 1080, 1920
    gen = torch.Generator(device="cuda").manual_seed(0)
    flat = cuda(O.flatten_params(O.init_params(seed=42)))
    r = torch.randn(4, 3, device="cuda", generator=gen) * 0.05; t = torch.randn(4, 3, device="cuda", generator=gen) * 0.05
    c2w = torch.empty(4, 4, device="cuda"); ops.pose_fwd_raw(r, t, None, 1, c2w)
    cam = torch.diag(torch.tensor([1.2, -1.2 * W / H, -1.0, 1.0])).cuda()
    ray_idx = torch.randperm(H * W, device="cuda", generator=gen)[:N]
    dpt = torch.rand(384, 672, device="cuda", generator=gen) * 6.6 + 0.6
    noise = torch.rand(N, S, device="cuda", generator=gen)
    cfg = dict(O.DEFAULT_CFG)
    flags = ops.flags_from_cfg(cfg, "softplus")
    res = {}
    ga = torch.randn(N, 3, device="cuda", generator=gen) / N; gb = torch.randn(N, 3, device="cuda", generator=gen) / N
    gd = torch.randn(N, device="cuda", generator=gen) / N
    for name, engine in engines():
        def fwd_bwd(g_rgb, g_dp):
            call = ops.RenderCall(flat, c2w, cam, N=N, S=S, flags=flags, engine=engine, near=0.01, far=10.0, ray_idx=ray_idx,
                                  depth_map=dpt, noise=noise, H=H, W=W, want_z_alpha=True, stash=True)
            g_w = torch.zeros(L.NUM_PARAMS, device="cuda"); g_c = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
            outs = (call.rgb.clone(), call.depth_pred.clone(), call.alpha.clone(), call.z_vals.clone())
            call.backward(g_rgb, g_dp, None, g_w, g_c, None, None, g_ss)
            return outs, g_w, g_c
        (rgb, dp, alpha, z), gw_a, gc_a = fwd_bwd(ga, gd)
        _, gw_b, gc_b = fwd_bwd(gb, torch.zeros_like(gd))
        _, gw_ab, gc_ab = fwd_bwd(ga + 2 * gb, gd)
        assert rgb.min() >= 0 and rgb.max() <= 1 + 1e-5
        assert dp.min() >= 0.0 and dp.max() <= 10.0 + 1e-3
        assert (z[:, 1:] >= z[:, :-1]).all()                     # stratified samples stay sorted
        assert alpha.min() >= 0 and alpha.max() <= 1
        lin_w = ((gw_a + 2 * gw_b - gw_ab).abs().max() / gw_ab.abs().max()).item()
        lin_c = ((gc_a + 2 * gc_b - gc_ab).abs().max() / gc_ab.abs().max()).item()
        assert lin_w < 1e-3 and lin_c < 1e-3, (lin_w, lin_c)      # atomics reorder fp32 sums run to run
        res[name] = (rgb, dp, gw_a, gc_a)
        _report("fullsize/%s" % name, lin_w=lin_w, lin_c=lin_c)
    if len(res) == 2:
        a, b = res["simt"], res["tc"]
        e = dict(rgb=((a[0] - b[0]).abs().max() / a[0].abs().max()).item(), dp=((a[1] - b[1]).abs().max() / a[1].abs().max()).item(),
                 gw=((a[2] - b[2]).abs().max() / a[2].abs().max()).item(), gc=((a[3] - b[3]).abs().max() / a[3].abs().max()).item())
        _report("fullsize/simt_vs_tc", **e)
        assert e["rgb"] < 1e-4 and e["dp"] < 1e-4, e
        assert e["gw"] < 2e-3 and e["gc"] < 2e-3, e


def test_cuda_graph_step_matches_eager_sequence():
    """Whole-step CUDA graph vs the same kernel sequence run eagerly: same seed, same frames, 6 steps.  The pixel / jitter
    draws come from torch's CUDA generator in both modes; parameters after the run must agree to fp32 round-off if the
    streams coincide, and the loss trajectories must agree statistically otherwise."""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    ops.set_default_engine("tc")
    H, W, V = 96, 128, 6
    res = {}
    for mode in (False, True):
        cfg = default_cfg()
        cfg["training"]["pc_weight"] = [0.0, 0.0]; cfg["training"]["rgb_s_weight"] = [0.0, 0.0]
        cfg["training"]["n_training_points"] = 256; cfg["rendering"]["num_points"] = 64
        dev = torch.device("cuda")
        torch.manual_seed(7)
        net = mdl.OfficialStaticNerf(cfg)
        net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=9).items()})
        model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
        pose = mdl.LearnPose(V, True, True, cfg).to(dev); dist = mdl.Learn_Distortion(V, True, True, cfg).to(dev)
        opt = torch.optim.Adam(model.parameters(), lr=1e-3); opt_p = torch.optim.Adam(pose.parameters(), lr=5e-4)
        opt_d = torch.optim.Adam(dist.parameters(), lr=5e-4)
        tr = mdl.Trainer(model, opt, cfg["training"], device=dev, optimizer_pose=opt_p, pose_param_net=pose, optimizer_distortion=opt_d,
                         distortion_net=dist, use_cuda_graph=mode, pixel_sampler="hash")
        g = torch.Generator().manual_seed(3)
        frames = [dict(img=torch.rand(1, 3, H, W, generator=g).cuda(), dpt=(torch.rand(1, 24, 32, generator=g) * 6 + 0.6).cuda()) for _ in range(3)]
        cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
        torch.manual_seed(11)
        losses = []
        for it in range(6):
            f = frames[it % 3]
            data = {"img": f["img"], "img.idx": torch.tensor([it % V]), "img.dpt": f["dpt"], "img.camera_mat": cam, "img.scale_mat": torch.eye(4)[None]}
            ld = tr.train_step(data, it=it, epoch=0, scheduling_start=10000, render_path=None)
            losses.append(ld["loss"].item())
        sd = opt.state_dict()
        assert int(next(iter(sd["state"].values()))["step"]) == 6      # optimizer state stays torch-compatible
        res[mode] = (np.array(losses), net.flat_weights().detach().cpu().numpy().copy(), pose.r.detach().cpu().numpy().copy())
    le, lg = res[False][0], res[True][0]
    assert np.all(np.isfinite(lg)) and np.all(np.isfinite(res[True][1]))
    _report("cuda_graph", loss_eager_last=le[-1], loss_graph_last=lg[-1], dparam=np.abs(res[False][1] - res[True][1]).max())
    assert abs(le[0] - lg[0]) < 1e-5 * abs(le[0])                      # first call is eager in both modes
    assert np.abs(lg - le).max() < 0.15 * np.abs(le).max(), (le, lg)   # later draws may differ (graph-safe philox offsets)


@pytest.mark.parametrize("full", [False, True])
def test_graph_replay_equals_eager_on_injected_draws(full, monkeypatch):
    """The captured whole-step graph (render-only, and the FULL loss set with the reference-image stage on its forked stream) against
    the same kernel sequence launched eagerly, on IDENTICAL pixel / jitter draws: torch.randperm / torch.rand are patched to hand out
    persistent device buffers that the test refills before every step, so the replayed graph reads the new draws.  Loss weights
    change during the run (annealing: epoch moves past scheduling_start) without re-capturing.  After 8 steps every parameter must
    agree to the noise of fp32 atomics."""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    ops.set_default_engine("tc")
    H, W, V, N, S, hd, wd = 96, 128, 6, 256, 64, 24, 32
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(3)
    up = lambda t, size: torch.nn.functional.interpolate(t, size, mode="bilinear", align_corners=False)
    frames = [dict(img=up(torch.rand(1, 3, 12, 16, generator=g), (H, W)).cuda(), dpt=(up(torch.rand(1, 1, 6, 8, generator=g), (hd, wd))[0] * 3 + 2).cuda())
              for _ in range(V)]
    draws = [(torch.randperm(H * W, generator=g)[:N].cuda(), torch.rand(N, S, generator=g).cuda()) for _ in range(8)]
    ray_buf = torch.zeros(N, dtype=torch.int64, device=dev); noise_buf = torch.zeros(1, N, S, device=dev)
    monkeypatch.setattr(torch, "randperm", lambda n, device=None: ray_buf)
    monkeypatch.setattr(torch, "rand", lambda *a, **k: noise_buf)
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
    res = {}
    for mode in (False, True):
        cfg = default_cfg()
        if not full:
            cfg["training"]["pc_weight"] = [0.0, 0.0]; cfg["training"]["rgb_s_weight"] = [0.0, 0.0]
        cfg["training"]["n_training_points"] = N; cfg["rendering"]["num_points"] = S
        cfg["training"]["annealing_epochs"] = 10
        net = mdl.OfficialStaticNerf(cfg)
        net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=9, hf_damp=True).items()})
        model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
        pose = mdl.LearnPose(V, True, True, cfg).to(dev); dist = mdl.Learn_Distortion(V, True, True, cfg).to(dev)
        with torch.no_grad():
            pose.r.copy_(torch.randn(V, 3, generator=torch.Generator().manual_seed(5)) * 0.03); pose.t.copy_(torch.randn(V, 3, generator=torch.Generator().manual_seed(6)) * 0.03)
        opt = torch.optim.Adam(model.parameters(), lr=1e-3); opt_p = torch.optim.Adam(pose.parameters(), lr=5e-4)
        opt_d = torch.optim.Adam(dist.parameters(), lr=5e-4)
        tr = mdl.Trainer(model, opt, cfg["training"], device=dev, optimizer_pose=opt_p, pose_param_net=pose, optimizer_distortion=opt_d,
                         distortion_net=dist, use_cuda_graph=mode, pixel_sampler="randperm")
        losses = []
        for it in range(8):
            ray_buf.copy_(draws[it][0]); noise_buf[0].copy_(draws[it][1])
            i = (it * 2 + 1) % (V - 1)          # view pairs (i, i+1); the last view's role swap is covered by the golden tests
            data = {"img": frames[i]["img"], "img.idx": torch.tensor([i]), "img.dpt": frames[i]["dpt"], "img.camera_mat": cam,
                    "img.scale_mat": torch.eye(4)[None], "img.ref_imgs": frames[i + 1]["img"], "img.ref_dpts": frames[i + 1]["dpt"],
                    "img.ref_idxs": torch.tensor([i + 1])}
            ld = tr.train_step(data, it=it, epoch=it, scheduling_start=3, render_path=None)      # weights anneal from step 4 on
            losses.append([ld[k].item() for k in ("loss", "loss_rgb", "loss_depth", "loss_pc", "loss_rgb_s")])
        if mode:
            gsteps = [v for v in tr._gsteps.values() if v]
            assert len(gsteps) == 1 and gsteps[0].graph is not None and gsteps[0].calls == 8      # ONE capture served all weight values
        res[mode] = (np.array(losses), net.flat_weights().detach().cpu().numpy().copy(), pose.r.detach().cpu().numpy().copy(),
                     pose.t.detach().cpu().numpy().copy(), dist.global_shifts.detach().cpu().numpy().copy())
    le, lg = res[False][0], res[True][0]
    w0 = O.flatten_params(O.init_params(seed=9, hf_damp=True)).astype(np.float64)
    ug, ue = res[True][1] - w0, res[False][1] - w0                        # the 8 Adam updates of every MLP weight
    r0 = (torch.randn(V, 3, generator=torch.Generator().manual_seed(5)) * 0.03).numpy().astype(np.float64)
    t0 = (torch.randn(V, 3, generator=torch.Generator().manual_seed(6)) * 0.03).numpy().astype(np.float64)
    upd = lambda k, p0: np.linalg.norm((res[True][k] - p0) - (res[False][k] - p0)) / max(np.linalg.norm(res[False][k] - p0), 1e-30)
    e = dict(loss=np.abs(le - lg).max() / np.abs(le).max(), w=np.linalg.norm(ug - ue) / np.linalg.norm(ue), w_max=relmax(ug, ue),
             r=upd(2, r0), t=upd(3, t0), r_abs=np.abs(res[True][2] - res[False][2]).max(), t_abs=np.abs(res[True][3] - res[False][3]).max(),
             shifts=relmax(res[True][4], res[False][4]))
    _report("graph_vs_eager/%s" % ("full" if full else "render"), **e)
    if full:
        assert le[:, 3].min() > 0 and le[:, 4].min() > 0, le             # the reference-image terms were live
    assert e["loss"] < 1e-5, (e, le, lg)
    # Adam turns a gradient into ~lr * sign(g) while |g| is tiny: weights whose gradient sits at the noise of the fp32 atomics can end up
    # a few lr apart (w_max), the update as a whole agrees (L2).  Pose: same metric on the 8 accumulated updates (a component whose
    # gradient cancels to the atomics' noise may differ by a fraction of one lr = 5e-4 step: measured 1.8e-4 on one t component, i.e.
    # 2 % of the L2 norm of the 18 accumulated t updates; the MLP statistic averages over 6e5 weights and is stable at 5.6e-3)
    assert e["w"] < 2e-2 and e["r"] < 0.1 and e["t"] < 0.1 and e["r_abs"] < 5e-4 and e["t_abs"] < 5e-4 and e["shifts"] < 1e-3, e


def test_adam_resume_from_checkpoint_matches_torch():
    """optimizer.state_dict() / load_state_dict() round trip (the reference's CheckpointIO, train.py:60-67, 249-271): after loading
    a checkpoint taken at step 5 into a NEW Trainer, both the eager fused Adam and the graph path continue bias correction from the
    loaded step, like torch.optim.Adam does."""
    from nope_nerf_b200.model.training import _FlatAdam
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(0)
    p0 = torch.randn(1000, generator=gen).cuda()
    grads = [torch.randn(1000, generator=gen).cuda() * 0.1 for _ in range(8)]
    # torch reference: 8 uninterrupted steps
    pr = torch.nn.Parameter(p0.clone()); opt_r = torch.optim.Adam([pr], lr=1e-2)
    for g_ in grads:
        pr.grad = g_.clone(); opt_r.step()
    # ours: 5 steps, checkpoint, new optimizer + _FlatAdam, load, 3 more steps
    pa = torch.nn.Parameter(p0.clone()); opt_a = torch.optim.Adam([pa], lr=1e-2); fa = _FlatAdam(opt_a)
    for g_ in grads[:5]:
        pa.grad = g_.clone(); fa.step()
    sd = opt_a.state_dict()
    assert int(sd["state"][0]["step"]) == 5
    pb = torch.nn.Parameter(pa.detach().clone()); opt_b = torch.optim.Adam([pb], lr=1e-2); fb = _FlatAdam(opt_b)
    opt_b.load_state_dict(sd)
    for g_ in grads[5:]:
        pb.grad = g_.clone(); fb.step()
    assert fb.nsteps == 8 and int(opt_b.state_dict()["state"][0]["step"]) == 8
    assert relmax(pb.detach().cpu().numpy(), pr.detach().cpu().numpy()) < 1e-6


def test_full_frame_renderer_vs_reference_golden():
    """Extract_Images.render_frame (config 4 caller, model/extracting_images.py:52-77): the whole 27x48 frame in one call;
    the golden's 32 rays (eval mode, ones prior, init_c2w pose) must come out identical."""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    g = load_golden("render_eval_ones")
    cfg = default_cfg(); cfg["rendering"]["num_points"] = int(g["S"]); cfg["extract_images"] = {"resolution": (int(g["H"]), int(g["W"]))}
    dev = torch.device("cuda")
    for eng in ("simt", "tc"):
        ops.set_default_engine(eng)
        net = mdl.OfficialStaticNerf(cfg)
        net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=int(g["seed"])).items()})
        rend = mdl.Renderer(net, cfg["rendering"], device=dev)
        ex = mdl.Extract_Images(rend, cfg, device=dev, render_type="nope_nerf")
        cam = torch.diag(torch.tensor([float(g["kx"]), float(g["ky"]), -1.0, 1.0])).to(dev)
        rgb, depth = ex.render_frame(cuda(g["c2w"]), cam, int(g["H"]), int(g["W"]))
        idx = g["ray_idx"]
        e_rgb = relmax(rgb.reshape(-1, 3).cpu().numpy()[idx], g["rgb"]); e_d = relmax(depth.reshape(-1).cpu().numpy()[idx], g["depth_pred"])
        _report("full_frame/%s" % eng, rgb=e_rgb, depth=e_d)
        assert e_rgb < 1e-4 and e_d < 1e-4, (eng, e_rgb, e_d)
        # row-block sharding (multi-GPU frame rendering) reproduces the same pixels
        top, _ = ex.render_frame(cuda(g["c2w"]), cam, int(g["H"]), int(g["W"]), rows=(0, 13))
        bot, _ = ex.render_frame(cuda(g["c2w"]), cam, int(g["H"]), int(g["W"]), rows=(13, int(g["H"])))
        assert torch.equal(torch.cat([top, bot], 0), rgb)


def test_trainer_pose_vs_oracle(monkeypatch):
    """Trainer_pose (model/eval_pose_one_epoch.py:62-98): frozen field, eval mode, ones prior, F.mse_loss; pose gradients only."""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    H, W, V, N, S = 30, 40, 4, 64, 64
    rng = np.random.default_rng(5)
    cfg = default_cfg(); cfg["rendering"]["num_points"] = S; cfg["eval_pose"]["n_points"] = N
    dev = torch.device("cuda")
    P = O.init_params(seed=13)
    r0 = rng.normal(0, .05, (V, 3)).astype(np.float32); t0 = rng.normal(0, .05, (V, 3)).astype(np.float32)
    img = rng.uniform(0, 1, (3, H, W)).astype(np.float32)
    ray_idx = rng.permutation(H * W)[:N]
    kx, ky = 1.2, -1.6
    # oracle
    ocfg = dict(O.DEFAULT_CFG); ocfg["num_points"] = S
    c2w = O.make_c2w(r0[2].astype(np.float64), t0[2].astype(np.float64))
    P64 = {k: v.astype(np.float64) for k, v in P.items()}
    pix = O.pixels_from_idx(ray_idx, H, W, np.float64)
    out, cache = O.render_forward(P64, pix, np.ones(N), c2w, kx, ky, ocfg, noise=None, eval_=True)
    gt = img.reshape(3, -1)[:, ray_idx].T.astype(np.float64)
    loss = ((out["rgb"] - gt) ** 2).mean()
    gr = O.render_backward(P64, cache, 2 * (out["rgb"] - gt) / (3 * N), np.zeros(N), np.zeros(N))
    g_r, g_t = O.make_c2w_bwd(r0[2].astype(np.float64), t0[2].astype(np.float64), None, gr["c2w"])
    for eng in ("simt", "tc"):
        ops.set_default_engine(eng)
        net = mdl.OfficialStaticNerf(cfg)
        net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in P.items()})
        model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
        pose = mdl.LearnPose(V, True, True, cfg).to(dev)
        with torch.no_grad():
            pose.r.copy_(cuda(r0)); pose.t.copy_(cuda(t0))
        opt = torch.optim.Adam(pose.parameters(), lr=1e-3)
        tp = mdl.Trainer_pose(model, cfg["eval_pose"], device=dev, optimizer_pose=opt, pose_param_net=pose)
        monkeypatch.setattr(torch, "randperm", lambda n, device=None: cuda(ray_idx))
        cam = torch.tensor([[kx, 0, 0, 0], [0, ky, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
        data = {"img": torch.from_numpy(img)[None], "img.idx": torch.tensor([2]), "img.camera_mat": cam, "img.scale_mat": torch.eye(4)[None]}
        w_before = net.flat_weights().clone()
        ld = tp.train_step(data)
        e = dict(loss=abs(ld["loss"].item() - loss) / loss, g_r=relmax(pose.r.grad.cpu().numpy()[2], g_r), g_t=relmax(pose.t.grad.cpu().numpy()[2], g_t))
        _report("trainer_pose/%s" % eng, **e)
        assert e["loss"] < 1e-5 and e["g_r"] < 2e-4 and e["g_t"] < 2e-4, (eng, e)
        assert torch.equal(net.flat_weights(), w_before)               # the field stays frozen
        assert float(pose.r.grad.abs().sum() - pose.r.grad[2].abs().sum()) == 0.0


@pytest.mark.parametrize("name", ["mlp_alpha_softplus", "mlp_sigma_relu"])
def test_field_forward_on_points_vs_reference_golden(name):
    """OfficialStaticNerf.forward(p, ray_d, return_addocc=True) + autograd (model/official_nerf.py:69-96)."""
    import nope_nerf_b200.model as mdl
    from _cfg import default_cfg
    g = load_golden(name)
    cfg = default_cfg(); cfg["rendering"]["dist_alpha"] = bool(g["dist_alpha"]); cfg["model"]["occ_activation"] = str(g["occ"])
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=int(g["seed"])).items()})
    net = net.cuda()
    tp = cuda(g["pts"]).requires_grad_(True); td = cuda(g["dirs"]).requires_grad_(True)
    rgb, a = net(tp, td, return_addocc=True)
    assert rgb.shape == (tp.shape[0], 3) and a.shape == (tp.shape[0], 1)
    ((rgb * cuda(g["g_rgb"])).sum() + (a[:, 0] * cuda(g["g_a"])).sum()).backward()
    floor = 2e-2 if str(g["occ"]) == "relu" else 1e-4
    e = dict(rgb=relmax(rgb.detach().cpu().numpy(), g["rgb"]), a=relmax(a.detach().cpu().numpy()[:, 0], g["a"]),
             g_pts=relmax(tp.grad.cpu().numpy(), g["g_pts"]), g_dirs=relmax(td.grad.cpu().numpy(), g["g_dirs"]),
             g_params=check_param_digest(g, {n: p.grad.cpu().numpy() for n, p in net.named_parameters()}))
    _report("field/%s" % name, **e)
    assert e["rgb"] < 1e-4 and e["a"] < 1e-4
    assert e["g_pts"] < max(floor, 2e-4) and e["g_dirs"] < max(floor, 2e-4) and e["g_params"] < max(floor, 5e-4), e
    assert net(tp.detach(), only_occupancy=True).shape == (tp.shape[0], 1)


def test_pixel_sampler_distinct_and_uniform():
    from nope_nerf_b200 import ops
    torch.manual_seed(0)
    HW, N = 1080 * 1920, 1024
    counts = torch.zeros(16, device="cuda")
    for _ in range(50):
        idx = ops.sample_pixels(HW, N, "cuda")
        assert idx.min() >= 0 and idx.max() < HW and torch.unique(idx).numel() == N
        counts += torch.bincount((idx * 16 // HW), minlength=16).float()
    frac = (counts / counts.sum()).cpu().numpy()
    assert np.abs(frac - 1 / 16).max() < 0.01            # 51 200 draws over 16 bins: sigma ~ 0.001
    small = ops.sample_pixels(4096, 2048, "cuda")        # dense case exercises the duplicate / probing paths
    assert torch.unique(small).numel() == 2048
    big = ops.sample_pixels(HW, 8192, "cuda")            # largest batch the in-graph sampler serves (8 GPUs x 1024 rays)
    assert big.min() >= 0 and big.max() < HW and torch.unique(big).numel() == 8192


@pytest.mark.parametrize("name", ["train_full_losses", "train_full_lastview"])
def test_native_ref_stage_vs_oracle(name):
    """nnb_refstage (fused kernels of the reference-image stage) vs oracle.ref_stage on the full-loss goldens' inputs.
    (First green on hardware in round 2: losses 1e-7, gradients 1e-6.)"""
    from nope_nerf_b200 import ops
    from test_host import _ref_stage_case
    c = _ref_stage_case(name)
    g = c["g"]
    l, gr = O.ref_stage(g["img"].astype(np.float64), g["ref"].astype(np.float64), g["dpt"].astype(np.float64), g["rdpt"].astype(np.float64),
                        c["c2w"].astype(np.float64), c["c2wr"].astype(np.float64), c["dist"][0], c["dist"][1], c["distr"][0], c["distr"][1],
                        c["is_last"], c["kx"], c["ky"], cfg=c["cfg"])
    c2w = cuda(c["c2w"]).requires_grad_(True); dist = torch.tensor(c["dist"], device="cuda", requires_grad=True)
    kx = torch.tensor(c["kx"], device="cuda", requires_grad=True); ky = torch.tensor(c["ky"], device="cuda", requires_grad=True)
    total, losses = ops.refstage(c2w, dist, cuda(c["c2wr"]), torch.tensor(c["distr"], device="cuda"), cuda(g["img"]), cuda(g["ref"]), cuda(g["dpt"]),
                                 cuda(g["rdpt"]), c["is_last"], kx, ky)
    total.backward()
    e = dict(loss_pc=abs(losses[0].item() - l["loss_pc"]) / l["loss_pc"], loss_rgb_s=abs(losses[1].item() - l["loss_rgb_s"]) / l["loss_rgb_s"],
             g_c2w=relmax(c2w.grad.cpu().numpy()[:3], gr["c2w"][:3]),
             g_dist=relmax(dist.grad.cpu().numpy(), np.array([gr["scale"], gr["shift"]])),
             g_kxy=relmax(np.array([kx.grad.item(), ky.grad.item()]), gr["kxy"]))
    _report("native_ref_stage/%s" % name, **e)
    assert e["loss_pc"] < 1e-5 and e["loss_rgb_s"] < 1e-5 and e["g_c2w"] < 1e-4 and e["g_dist"] < 1e-4 and e["g_kxy"] < 1e-4, e


@pytest.mark.parametrize("N,S", [(5, 32), (3, 64), (7, 32), (130, 32), (33, 64), (999, 128), (9, 256)])
def test_ragged_last_tile_tc_vs_simt(N, S):
    """N*S not a multiple of the 128-sample tile: the tensor-core engine pads the last tile with clamped rows whose cotangents are
    zero; outputs and gradients must agree with the exact-fp32 engine (weights from init_params(hf_damp=True), so that the
    comparison of the two engines' GRADIENTS is not dominated by single ReLU-gate switches on a handful of rays)."""
    from nope_nerf_b200 import ops, _lib as L
    if len(engines()) < 2:
        pytest.skip("needs both engines")
    H, W = 40, 56
    gen = torch.Generator(device="cuda").manual_seed(N * 1000 + S)
    flat = cuda(O.flatten_params(O.init_params(seed=5, hf_damp=True)))
    r = torch.randn(3, 3, device="cuda", generator=gen) * 0.05; t = torch.randn(3, 3, device="cuda", generator=gen) * 0.05
    c2w = torch.empty(4, 4, device="cuda"); ops.pose_fwd_raw(r, t, None, 1, c2w)
    cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0])).cuda()
    ray_idx = torch.randperm(H * W, device="cuda", generator=gen)[:N]
    dpt = torch.rand(20, 28, device="cuda", generator=gen) * 6.6 + 0.6
    noise = torch.rand(N, S, device="cuda", generator=gen)
    flags = ops.flags_from_cfg(dict(O.DEFAULT_CFG), "softplus")
    g_rgb = torch.randn(N, 3, device="cuda", generator=gen) / N; g_dp = torch.randn(N, device="cuda", generator=gen) / N
    res = {}
    for name, engine in engines():
        call = ops.RenderCall(flat, c2w, cam, N=N, S=S, flags=flags, engine=engine, near=0.01, far=10.0, ray_idx=ray_idx, depth_map=dpt,
                              noise=noise, H=H, W=W, stash=True)
        g_w = torch.zeros(L.NUM_PARAMS, device="cuda"); g_c = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
        rgb, dp = call.rgb.clone(), call.depth_pred.clone()
        call.backward(g_rgb, g_dp, None, g_w, g_c, None, None, g_ss)
        torch.cuda.synchronize()
        res[name] = (rgb, dp, g_w, g_c, g_ss)
    a, b = res["simt"], res["tc"]
    rel = lambda x, y: ((x - y).abs().max() / x.abs().max().clamp_min(1e-30)).item()
    e = dict(rgb=rel(a[0], b[0]), dp=rel(a[1], b[1]), gw=rel(a[2], b[2]), gc=rel(a[3], b[3]), gss=rel(a[4], b[4]))
    _report("ragged/%dx%d" % (N, S), **e)
    assert e["rgb"] < 1e-4 and e["dp"] < 1e-4 and e["gw"] < 5e-4 and e["gc"] < 1e-4 and e["gss"] < 1e-4, e

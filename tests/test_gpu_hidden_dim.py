"""GPU: the field at model.hidden_dim 128 and 64 on both engines.
(1) render forward + backward against the reference (tests/golden/*_d{128,64}*.npz, tools/make_golden.py hidden) with the gates of
test_gpu_parity.test_render_vs_reference_golden; (2) OfficialStaticNerf.forward / infer_occ / gradient on explicit points; (3) two
Trainer steps, eager and CUDA-graph, against the reference Trainer, and graph replay against eager; (4) the tensor-core engine against
the exact-fp32 engine at C2 size (1024 rays x 128 samples); (5) an unsupported width is rejected by the module and by the C ABI."""
import ctypes as C
import numpy as np
import pytest
import torch

from _util import load_golden, relmax, cfg_from_golden, check_param_digest
from oracle import nerf_oracle as O
from test_gpu_parity import engines, cuda, _report
import test_hidden_dim_golden as HG

pytestmark = pytest.mark.gpu
DIMS = (128, 64)


def run_render_cuda(g, engine):
    from nope_nerf_b200 import ops, _lib as L
    cfg = cfg_from_golden(g)
    D = int(g["hidden_dim"])
    P = O.init_params(seed=int(g["seed"]), D=D, white_bkgd=cfg["white_background"], hf_damp=bool(g["hf_damp"]))
    flat = cuda(O.flatten_params(P))
    cam_id = int(g["cam_id"]); N, S, H, W = int(g["N"]), int(g["S"]), int(g["H"]), int(g["W"])
    r, t = cuda(g["r"]), cuda(g["t"])
    c2w = torch.empty(4, 4, device="cuda")
    ops.pose_fwd_raw(r, t, None, cam_id, c2w)
    cam = torch.diag(torch.tensor([float(g["kx"]), float(g["ky"]), -1.0, 1.0])).cuda()
    ndc = cfg["sample_option"] == "ndc"
    call = ops.RenderCall(flat, c2w, cam, N=N, S=S, flags=ops.flags_from_cfg(cfg, cfg["occ_activation"], eval_=bool(g["eval_mode"])),
                          engine=engine, near=0.0 if ndc else cfg["depth_range"][0], far=1.0 if ndc else cfg["depth_range"][1],
                          ray_idx=cuda(g["ray_idx"]), depth_map=cuda(g["dpt"]), scale=torch.tensor([float(g["scale"])]).cuda(),
                          shift=torch.tensor([float(g["shift"])]).cuda(), noise=cuda(g["noise"]), H=H, W=W, want_z_alpha=True, stash=True,
                          hidden_dim=D)
    mask = call.mask.bool().cpu().numpy()
    out = dict(rgb=call.rgb.cpu().numpy(), depth_pred=call.depth_pred.cpu().numpy()[mask], depth_gt=call.depth_gt.cpu().numpy()[mask],
               z_vals=call.z_vals.cpu().numpy(), alpha=call.alpha.cpu().numpy())
    gdp = np.zeros(N, np.float32); gdg = np.zeros(N, np.float32)
    gdp[mask] = g["g_dp"]; gdg[mask] = g["g_dg"]
    g_w = torch.zeros(L.num_params(D), device="cuda"); g_c2w = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
    call.backward(cuda(g["g_rgb"]), cuda(gdp), cuda(gdg), g_w, g_c2w, torch.zeros(4, 4, device="cuda"), None, g_ss)
    g_r = torch.zeros_like(r); g_t = torch.zeros_like(t)
    ops.pose_bwd_raw(r, t, None, cam_id, g_c2w, g_r, g_t)
    torch.cuda.synchronize()
    return out, dict(c2w=g_c2w.cpu().numpy(), r=g_r.cpu().numpy()[cam_id], t=g_t.cpu().numpy()[cam_id], ss=g_ss.cpu().numpy(),
                     params=O.unflatten_params(g_w.cpu().numpy(), D=D))


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("base", HG.RENDER)
@pytest.mark.parametrize("eng", ["simt", "tc"])
def test_render_vs_reference_golden(base, D, eng):
    """outputs <= 1e-4 of the reference; `_damped` cases: every gradient <= 1e-4 of the fp64 oracle and <= max(1e-4, 3 x the
    reference's own distance from it); default-initialised cases: <= max(1e-4, 3 x envelope) (see test_gpu_parity)"""
    engine = dict(engines()).get(eng)
    if engine is None:
        pytest.skip("engine disabled")
    g = load_golden(HG.golden_name(base, D))
    damped = bool(g["hf_damp"])
    cam = int(g["cam_id"])
    out, grads = run_render_cuda(g, engine)
    o64, gr64, g_r64, g_t64, raw = HG.oracle_render(g, np.float64)
    o32, gr32, g_r32, g_t32, _ = HG.oracle_render(g, np.float32)
    ss = lambda gr: np.array([(gr["depth"] * raw).sum(), gr["depth"].sum()])
    terms = dict(c2w=(grads["c2w"], g["grad_c2w"], gr64["c2w"], gr32["c2w"]), r=(grads["r"], g["grad_r"][cam], g_r64, g_r32),
                 t=(grads["t"], g["grad_t"][cam], g_t64, g_t32), ss=(grads["ss"], np.array([g["grad_scale"], g["grad_shift"]]), ss(gr64), ss(gr32)))
    e = dict(rgb=relmax(out["rgb"], g["rgb"]), depth_pred=relmax(out["depth_pred"], g["depth_pred"]), depth_gt=relmax(out["depth_gt"], g["depth_gt"]),
             alpha=relmax(out["alpha"], g["alpha"]), z=relmax(out["z_vals"], g["z_vals"]), g_params=check_param_digest(g, grads["params"]),
             env_params=max(check_param_digest(g, gr64["params"]), check_param_digest(g, gr32["params"])))
    for k, (ours, ref, t64, t32) in terms.items():
        e["g_" + k] = relmax(ours, ref); e["g_%s_vs64" % k] = relmax(ours, t64)
        e["env_" + k] = max(relmax(t64, ref), relmax(t32, t64)); e["ref64_" + k] = relmax(t64, ref)
    _report("hidden/%s_d%d/%s" % (base, D, eng), **e)
    for k in ("rgb", "depth_pred", "depth_gt", "z"):
        assert e[k] < 1e-4, (k, e[k])
    assert e["alpha"] < 2e-4, e["alpha"]
    for k in terms:
        if damped:
            assert e["g_%s_vs64" % k] < 1e-4, (k, e)
            assert e["g_" + k] < max(1e-4, 3 * e["ref64_" + k]), (k, e)
        else:
            assert e["g_" + k] < max(1e-4, 3 * e["env_" + k]), (k, e)
    assert e["g_params"] < max(5e-4, 3 * e["env_params"]), e


def _module(D, dist_alpha=False, occ="softplus"):
    import nope_nerf_b200.model as mdl
    from _cfg import default_cfg
    cfg = default_cfg(); cfg["model"]["hidden_dim"] = D; cfg["rendering"]["dist_alpha"] = dist_alpha; cfg["model"]["occ_activation"] = occ
    return mdl.OfficialStaticNerf(cfg), cfg


def test_field_explicit_points_d128():
    """OfficialStaticNerf.forward (outputs + autograd to points, directions and parameters), infer_occ and gradient() at D = 128"""
    g = load_golden("mlp_alpha_softplus_d128")
    net, _ = _module(128)
    P = O.init_params(seed=int(g["seed"]), D=128)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in P.items()})
    net = net.cuda()
    p = cuda(g["pts"]).requires_grad_(True); d = cuda(g["dirs"]).requires_grad_(True)
    rgb, a = net(p, d, return_addocc=True)
    ((rgb * cuda(g["g_rgb"])).sum() + (a[:, 0] * cuda(g["g_a"])).sum()).backward()
    e = dict(rgb=relmax(rgb.detach().cpu().numpy(), g["rgb"]), a=relmax(a.detach().cpu().numpy()[:, 0], g["a"]),
             g_pts=relmax(p.grad.cpu().numpy(), g["g_pts"]), g_dirs=relmax(d.grad.cpu().numpy(), g["g_dirs"]),
             g_params=check_param_digest(g, {n: q.grad.cpu().numpy() for n, q in net.named_parameters()}))
    # infer_occ / gradient(): the density logit and -d logit / d p against the fp64 oracle
    P64 = {k: v.astype(np.float64) for k, v in P.items()}
    pts64 = g["pts"].astype(np.float64)
    h = O.encode_position(pts64, 10)
    x = h
    for li, name in enumerate(["layers0.0", "layers0.2", "layers0.4", "layers0.6", "layers1.0", "layers1.2", "layers1.4", "layers1.6"]):
        if li == 4:
            x = np.concatenate([x, h], -1)
        x = np.maximum(x @ P64[name + ".weight"].T + P64[name + ".bias"], 0.0)
    logit = x @ P64["fc_density.weight"].T + P64["fc_density.bias"]
    _, s = net.infer_occ(cuda(g["pts"]))
    e["logit"] = relmax(s.detach().cpu().numpy(), logit)
    gn = net.gradient(cuda(g["pts"]), 0)
    assert tuple(gn.shape) == (g["pts"].shape[0], 1, 3)
    q = torch.from_numpy(pts64).requires_grad_(True)
    hq = torch.cat([q] + [f(q * 2.0 ** l) for l in range(10) for f in (torch.sin, torch.cos)], -1)
    assert np.allclose(hq.detach().numpy(), h)
    xq = hq
    for li, name in enumerate(["layers0.0", "layers0.2", "layers0.4", "layers0.6", "layers1.0", "layers1.2", "layers1.4", "layers1.6"]):
        if li == 4:
            xq = torch.cat([xq, hq], -1)
        xq = torch.relu(xq @ torch.from_numpy(P64[name + ".weight"]).T + torch.from_numpy(P64[name + ".bias"]))
    (xq @ torch.from_numpy(P64["fc_density.weight"]).T).sum().backward()
    e["normal"] = relmax(gn[:, 0].cpu().numpy(), -q.grad.numpy())
    _report("hidden/field_d128", **e)
    assert e["rgb"] < 1e-5 and e["a"] < 1e-4 and e["logit"] < 1e-4, e
    assert e["g_pts"] < 1e-3 and e["g_dirs"] < 1e-3 and e["g_params"] < 1e-3 and e["normal"] < 1e-3, e


def _trainer(g, eng, D, use_cuda_graph):
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    ops.set_default_engine(eng)
    cfg = default_cfg()
    S, N, V = int(g["S"]), int(g["N"]), int(g["V"])
    cfg["model"]["hidden_dim"] = D
    cfg["rendering"]["num_points"] = S; cfg["training"]["n_training_points"] = N
    cfg["training"]["vis_reprojection_every"] = 10 ** 9
    dev = torch.device("cuda")
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=int(g["seed"]), D=D).items()})
    model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
    pose = mdl.LearnPose(V, True, True, cfg).to(dev); dist = mdl.Learn_Distortion(V, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.copy_(cuda(g["r0"])); pose.t.copy_(cuda(g["t0"]))
        dist.global_scales.copy_(cuda(g["scales0"])); dist.global_shifts.copy_(cuda(g["shifts0"]))
    opt = torch.optim.Adam(model.parameters(), lr=1e-3); opt_p = torch.optim.Adam(pose.parameters(), lr=5e-4)
    opt_d = torch.optim.Adam(dist.parameters(), lr=5e-4)
    tr = mdl.Trainer(model, opt, cfg["training"], device=dev, optimizer_pose=opt_p, pose_param_net=pose, optimizer_distortion=opt_d,
                     distortion_net=dist, use_cuda_graph=use_cuda_graph, pixel_sampler="randperm")
    return tr, net, pose, dist


def _run_golden_steps(g, eng, D, graph, monkeypatch):
    """the reference's pixel / jitter draws go through fixed device buffers, which a captured graph reads on every replay"""
    N, S = int(g["N"]), int(g["S"])
    ray_buf = torch.zeros(N, dtype=torch.int64, device="cuda"); noise_buf = torch.zeros(1, N, S, device="cuda")
    monkeypatch.setattr(torch, "randperm", lambda n, device=None: ray_buf)
    monkeypatch.setattr(torch, "rand", lambda *a, **k: noise_buf)
    tr, net, pose, dist = _trainer(g, eng, D, graph)
    kx, ky = float(g["kx"]), float(g["ky"])
    cam = np.array([[kx, 0, 0, 0], [0, ky, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], np.float32)
    data = {"img": torch.from_numpy(g["img"])[None], "img.idx": torch.tensor([int(g["idx"])]), "img.dpt": torch.from_numpy(g["dpt"])[None],
            "img.camera_mat": torch.from_numpy(cam)[None], "img.scale_mat": torch.eye(4)[None], "img.ref_imgs": torch.from_numpy(g["ref"])[None],
            "img.ref_dpts": torch.from_numpy(g["rdpt"])[None], "img.ref_idxs": torch.tensor([int(g["ref_idx"])])}
    steps = []
    for it in range(int(g["steps"])):
        ray_buf.copy_(cuda(g["ray_idx_%d" % it])); noise_buf[0].copy_(cuda(g["noise_%d" % it]))
        ld = tr.train_step(data, it=it + 1, epoch=0, scheduling_start=10000, render_path="/tmp")
        torch.cuda.synchronize()
        steps.append(dict(ld={k: float(ld[k].reshape(-1)[0]) for k in ("loss", "loss_rgb", "loss_depth", "loss_pc", "loss_rgb_s")},
                          r=pose.r.grad.cpu().numpy().copy(), t=pose.t.grad.cpu().numpy().copy(),
                          scales=dist.global_scales.grad.cpu().numpy().copy(), shifts=dist.global_shifts.grad.cpu().numpy().copy(),
                          params={n: p.grad.cpu().numpy().copy() for n, p in net.named_parameters()}))
    if graph:
        gsteps = [v for v in tr._gsteps.values() if v]
        assert len(gsteps) == 1 and gsteps[0].graph is not None, "the CUDA-graph step did not run"
    end = dict(r=pose.r.detach().cpu().numpy(), t=pose.t.detach().cpu().numpy(), flat=net.flat_weights().detach().cpu().numpy().copy(),
               params={n: p.detach().cpu().numpy() for n, p in net.named_parameters()})
    return steps, end


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("eng", ["simt", "tc"])
@pytest.mark.parametrize("graph", [False, True])
def test_trainer_steps_vs_reference_golden(D, eng, graph, monkeypatch):
    """gates of test_gpu_parity.test_trainer_step_vs_reference_golden ('exact' weight gradients)"""
    if dict(engines()).get(eng) is None:
        pytest.skip("engine disabled")
    g = load_golden("train_full_losses_d%d" % D)
    steps, end = _run_golden_steps(g, eng, D, graph, monkeypatch)
    worst = {}
    for it, st in enumerate(steps):
        for k, v in st["ld"].items():
            ref = float(np.ravel(g["loss_%d.%s" % (it, k)])[0])
            worst["loss_%d_%s" % (it, k)] = abs(v - ref) / max(abs(ref), 1e-3)
        for k in ("r", "t", "scales", "shifts"):
            worst["g_%s_%d" % (k, it)] = relmax(st[k], g["grad_%s_%d" % (k, it)])
        worst["g_params_%d" % it] = check_param_digest(g, st["params"], prefix="pg_%d." % it)
    worst["r_end"] = relmax(end["r"] - g["r0"], g["r_end"] - g["r0"])
    worst["t_end"] = relmax(end["t"] - g["t0"], g["t_end"] - g["t0"])
    worst["params_end"] = check_param_digest(g, end["params"], prefix="pend.")
    _report("hidden/train_d%d/%s%s" % (D, eng, "-graph" if graph else ""), **worst)
    for k, v in worst.items():
        if k.startswith("loss"):
            assert v < 2e-4, (k, v)
        elif k.startswith("g_params"):
            assert v < 5e-3, (k, v)
        elif k.startswith("g_"):
            assert v < 2e-3, (k, v)
        elif k in ("r_end", "t_end"):
            assert v < 5e-2, (k, v)
        else:
            assert v < 1e-3, (k, v)


@pytest.mark.parametrize("D", DIMS)
def test_graph_replay_equals_eager(D, monkeypatch):
    """the captured graph step runs the kernels of the eager step on the same inputs; the reference-image stage accumulates with
    float atomics, so the gates are those of test_gpu_refopts.test_graph_replay_equals_eager_refopts"""
    g = load_golden("train_full_losses_d%d" % D)
    se, ee = _run_golden_steps(g, "tc", D, False, monkeypatch)
    sg, eg = _run_golden_steps(g, "tc", D, True, monkeypatch)
    w0 = O.flatten_params(O.init_params(seed=int(g["seed"]), D=D)).astype(np.float64)
    e = dict(loss=max(abs(a["ld"][k] - b["ld"][k]) / abs(a["ld"][k]) for a, b in zip(se, sg) for k in a["ld"]),
             g_r=max(relmax(b["r"], a["r"]) for a, b in zip(se, sg)), g_t=max(relmax(b["t"], a["t"]) for a, b in zip(se, sg)),
             w=np.linalg.norm(eg["flat"] - ee["flat"]) / np.linalg.norm(ee["flat"] - w0))
    _report("hidden/graph_vs_eager_d%d" % D, **e)
    assert e["loss"] < 1e-5 and e["g_r"] < 1e-3 and e["g_t"] < 1e-3 and e["w"] < 2e-2, e


def test_c2_size_tc_vs_simt_d128():
    """1024 rays x 128 samples (the C2 batch) at D = 128: the tensor-core engine against the exact-fp32 engine, forward and backward;
    gates of test_gpu_fullsize_ref (outputs 1e-4; gradients of the pose 2e-3, MLP gradient 5e-3 of its max)"""
    from nope_nerf_b200 import ops, _lib as L
    D, N, S, H, W = 128, 1024, 128, 1080, 1920
    rng = np.random.default_rng(7)
    flat = cuda(O.flatten_params(O.init_params(seed=5, D=D, hf_damp=True)))
    c2w = cuda(O.make_c2w(rng.normal(0, 0.05, 3).astype(np.float32), rng.normal(0, 0.05, 3).astype(np.float32)))
    cam = torch.diag(torch.tensor([1.2, -2.1, -1.0, 1.0])).cuda()
    ray_idx = cuda(rng.permutation(H * W)[:N].astype(np.int64)); noise = cuda(rng.uniform(0, 1, (N, S)).astype(np.float32))
    dpt = cuda(rng.uniform(0.6, 7.2, (384, 672)).astype(np.float32))
    g_rgb = cuda(rng.normal(0, 1, (N, 3)).astype(np.float32)); g_dp = cuda(rng.normal(0, 1, N).astype(np.float32))
    flags = ops.flags_from_cfg(dict(O.DEFAULT_CFG), "softplus")
    res = {}
    for name, engine in (("simt", L.ENGINE_SIMT), ("tc", L.ENGINE_TC)):
        call = ops.RenderCall(flat, c2w, cam, N=N, S=S, flags=flags, engine=engine, near=0.01, far=10.0, ray_idx=ray_idx, depth_map=dpt,
                              scale=torch.tensor([1.05]).cuda(), shift=torch.tensor([0.02]).cuda(), noise=noise, H=H, W=W, stash=True, hidden_dim=D)
        g_w = torch.zeros(L.num_params(D), device="cuda"); g_c = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
        out = (call.rgb.clone(), call.depth_pred.clone())
        call.backward(g_rgb, g_dp, None, g_w, g_c, None, None, g_ss)
        torch.cuda.synchronize()
        res[name] = [x.cpu().numpy() for x in out + (g_c, g_ss, g_w)]
    s, t = res["simt"], res["tc"]
    e = dict(rgb=relmax(t[0], s[0]), depth=relmax(t[1], s[1]), g_c2w=relmax(t[2], s[2]), g_ss=relmax(t[3], s[3]), g_w=relmax(t[4], s[4]))
    _report("hidden/c2_tc_vs_simt_d128", **e)
    assert e["rgb"] < 1e-4 and e["depth"] < 1e-4, e
    assert e["g_c2w"] < 2e-3 and e["g_ss"] < 2e-3 and e["g_w"] < 5e-3, e


def test_unsupported_width_c_abi_error():
    """hidden_dim 96: the module raises NotImplementedError, the workspace query returns 0 and nnb_render_fwd returns an error"""
    from nope_nerf_b200 import ops, _lib as L
    with pytest.raises(NotImplementedError):
        _module(96)
    with pytest.raises(ValueError, match="hidden_dim 96"):
        ops.RenderCall(torch.zeros(L.NUM_PARAMS, device="cuda"), torch.eye(4, device="cuda"), torch.eye(4, device="cuda"), N=8, S=32,
                       flags=0, engine=L.ENGINE_SIMT, near=0.1, far=1.0, pixels=torch.zeros(8, 2, device="cuda"),
                       depth=torch.ones(8, device="cuda"), hidden_dim=96)
    N, S = 8, 32
    w = torch.zeros(L.NUM_PARAMS, device="cuda"); eye = torch.eye(4, device="cuda")
    pix = torch.zeros(N, 2, device="cuda"); dep = torch.ones(N, device="cuda")
    outs = [torch.empty(N, 3, device="cuda"), torch.empty(N, device="cuda"), torch.empty(N, device="cuda"), torch.empty(N, dtype=torch.uint8, device="cuda")]
    ws = torch.empty(L.lib.nnb_workspace_bytes(N, S, 0, L.ENGINE_SIMT), dtype=torch.uint8, device="cuda")
    a = L.RenderArgs()
    a.weights, a.c2w, a.cam, a.pixels, a.depth = w.data_ptr(), eye.data_ptr(), eye.data_ptr(), pix.data_ptr(), dep.data_ptr()
    a.N, a.S, a.near_, a.far_, a.engine = N, S, 0.1, 1.0, L.ENGINE_SIMT
    a.rgb, a.depth_pred, a.depth_gt, a.mask = (o.data_ptr() for o in outs)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    a.hidden_dim = 96
    rc = L.lib.nnb_render_fwd(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc < 0 and b"hidden_dim 96" in L.lib.nnb_last_error()
    a.pts = pix.data_ptr()
    out = torch.empty(N, 4, device="cuda")
    assert L.lib.nnb_field_fwd(C.byref(a), out.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)) < 0
    a.hidden_dim = 0          # 0 means 256: the same call succeeds
    assert L.lib.nnb_render_fwd(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    torch.cuda.synchronize()

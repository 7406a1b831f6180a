"""GPU: rendering.num_points outside {32, 64, 128, 256} on both engines (the tensor-core engine serves 16..1024 samples per ray, the
exact-fp32 engine 2..1024).
(1) render forward + backward against the reference (tests/golden/render_*_s{48,96,200,300}*.npz, tools/make_golden.py samples) with the
gates of test_gpu_parity.test_render_vs_reference_golden; (2) Trainer steps, eager and CUDA-graph, against the reference Trainer at
S = 48 (full losses) and S = 300 (render only), and graph replay against eager; (3) the tensor-core engine against the exact-fp32 engine
at C2 size (1024 rays x 96 | 200 samples, 512 rays x 512 samples); (4) Extract_Images.render_frame and Trainer_pose off the old sample
counts; (5) the engine rule of ops.pick_engine and the C ABI's sample-count errors."""
import ctypes as C
import numpy as np
import pytest
import torch

from _util import load_golden, relmax, check_param_digest
from oracle import nerf_oracle as O
from test_gpu_parity import engines, cuda, _report
import test_gpu_parity as GP
import test_sample_count_golden as SG

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _keep_default_engine(monkeypatch):
    """tests below switch the process-wide default engine; it is restored after each test"""
    from nope_nerf_b200 import ops
    monkeypatch.setattr(ops, "_DEFAULT_ENGINE", list(ops._DEFAULT_ENGINE))


@pytest.mark.parametrize("name", SG.RENDER_ALL)
@pytest.mark.parametrize("eng", ["simt", "tc"])
def test_render_vs_reference_golden(name, eng):
    """outputs <= 1e-4 of the reference; `_damped` cases: every gradient <= 1e-4 of the fp64 oracle and <= max(1e-4, 3 x the
    reference's own distance from it); default-initialised cases: <= max(1e-4, 3 x envelope)"""
    GP.test_render_vs_reference_golden(name, eng)


def _trainer(g, eng, with_ref, use_cuda_graph):
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    ops.set_default_engine(eng)
    cfg = default_cfg()
    S, N, V = int(g["S"]), int(g["N"]), int(g["V"])
    cfg["rendering"]["num_points"] = S; cfg["training"]["n_training_points"] = N
    if not with_ref:
        cfg["training"]["pc_weight"] = [0.0, 0.0]; cfg["training"]["rgb_s_weight"] = [0.0, 0.0]
    cfg["training"]["vis_reprojection_every"] = 10 ** 9
    dev = torch.device("cuda")
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=int(g["seed"])).items()})
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


TRAIN = [("train_full_losses_s48", True), ("train_render_only_s300", False)]


def _run_golden_steps(name, with_ref, eng, graph, monkeypatch):
    """the reference's pixel / jitter draws go through fixed device buffers, which a captured graph reads on every replay"""
    g = load_golden(name)
    N, S = int(g["N"]), int(g["S"])
    ray_buf = torch.zeros(N, dtype=torch.int64, device="cuda"); noise_buf = torch.zeros(1, N, S, device="cuda")
    monkeypatch.setattr(torch, "randperm", lambda n, device=None: ray_buf)
    monkeypatch.setattr(torch, "rand", lambda *a, **k: noise_buf)
    tr, net, pose, dist = _trainer(g, eng, with_ref, graph)
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
    return g, steps, end


@pytest.mark.parametrize("name,with_ref", TRAIN)
@pytest.mark.parametrize("eng", ["simt", "tc"])
@pytest.mark.parametrize("graph", [False, True])
def test_trainer_steps_vs_reference_golden(name, with_ref, eng, graph, monkeypatch):
    """gates of test_gpu_parity.test_trainer_step_vs_reference_golden ('exact' weight gradients)"""
    if dict(engines()).get(eng) is None:
        pytest.skip("engine disabled")
    g, steps, end = _run_golden_steps(name, with_ref, eng, graph, monkeypatch)
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
    _report("samples/%s/%s%s" % (name, eng, "-graph" if graph else ""), **worst)
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


@pytest.mark.parametrize("name,with_ref", TRAIN)
def test_graph_replay_equals_eager(name, with_ref, monkeypatch):
    """the captured graph step runs the kernels of the eager step on the same inputs.  Render only (S = 300): every reduction runs in
    a fixed order, so the two agree bit for bit.  With the reference-image stage (S = 48), whose float atomics run on a forked stream,
    the gates are those of test_gpu_refopts.test_graph_replay_equals_eager_refopts."""
    g, se, ee = _run_golden_steps(name, with_ref, "tc", False, monkeypatch)
    _, sg, eg = _run_golden_steps(name, with_ref, "tc", True, monkeypatch)
    w0 = O.flatten_params(O.init_params(seed=int(g["seed"]))).astype(np.float64)
    e = dict(loss=max(abs(a["ld"][k] - b["ld"][k]) / abs(a["ld"][k]) for a, b in zip(se, sg) for k in a["ld"] if a["ld"][k] != 0.0),
             g_r=max(relmax(b["r"], a["r"]) for a, b in zip(se, sg)), g_t=max(relmax(b["t"], a["t"]) for a, b in zip(se, sg)),
             w=np.linalg.norm(eg["flat"] - ee["flat"]) / np.linalg.norm(ee["flat"] - w0))
    _report("samples/graph_vs_eager/%s" % name, **e)
    if with_ref:
        assert e["loss"] < 1e-5 and e["g_r"] < 1e-3 and e["g_t"] < 1e-3 and e["w"] < 2e-2, e
    else:
        for a, b in zip(se, sg):
            assert a["ld"] == b["ld"]
            for k in ("r", "t", "scales", "shifts"):
                assert np.array_equal(a[k], b[k]), k
            for n in a["params"]:
                assert np.array_equal(a["params"][n], b["params"][n]), n
        assert np.array_equal(eg["flat"], ee["flat"]) and np.array_equal(eg["r"], ee["r"]) and np.array_equal(eg["t"], ee["t"])


@pytest.mark.parametrize("N,S", [(1024, 96), (1024, 200), (512, 512)])
def test_c2_size_tc_vs_simt(N, S):
    """C2-size batches at sample counts the tensor-core engine did not serve before: TC against the exact-fp32 engine, forward and
    backward, with the gates of test_gpu_hidden_dim.test_c2_size_tc_vs_simt_d128 (outputs 1e-4; pose / scale-shift gradients 2e-3, MLP
    gradient 5e-3 of its max)"""
    from nope_nerf_b200 import ops, _lib as L
    H, W = 1080, 1920
    rng = np.random.default_rng(S)
    flat = cuda(O.flatten_params(O.init_params(seed=5, hf_damp=True)))
    c2w = cuda(O.make_c2w(rng.normal(0, 0.05, 3).astype(np.float32), rng.normal(0, 0.05, 3).astype(np.float32)))
    cam = torch.diag(torch.tensor([1.2, -2.1, -1.0, 1.0])).cuda()
    ray_idx = cuda(rng.permutation(H * W)[:N].astype(np.int64)); noise = cuda(rng.uniform(0, 1, (N, S)).astype(np.float32))
    dpt = cuda(rng.uniform(0.6, 7.2, (384, 672)).astype(np.float32))
    g_rgb = cuda(rng.normal(0, 1, (N, 3)).astype(np.float32)); g_dp = cuda(rng.normal(0, 1, N).astype(np.float32))
    flags = ops.flags_from_cfg(dict(O.DEFAULT_CFG), "softplus")
    res = {}
    for name, engine in (("simt", L.ENGINE_SIMT), ("tc", L.ENGINE_TC)):
        call = ops.RenderCall(flat, c2w, cam, N=N, S=S, flags=flags, engine=engine, near=0.01, far=10.0, ray_idx=ray_idx, depth_map=dpt,
                              scale=torch.tensor([1.05]).cuda(), shift=torch.tensor([0.02]).cuda(), noise=noise, H=H, W=W, stash=True)
        assert call.args.engine == engine
        g_w = torch.zeros(L.NUM_PARAMS, device="cuda"); g_c = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
        out = (call.rgb.clone(), call.depth_pred.clone())
        call.backward(g_rgb, g_dp, None, g_w, g_c, None, None, g_ss)
        torch.cuda.synchronize()
        call.release()
        res[name] = [x.cpu().numpy() for x in out + (g_c, g_ss, g_w)]
    s, t = res["simt"], res["tc"]
    e = dict(rgb=relmax(t[0], s[0]), depth=relmax(t[1], s[1]), g_c2w=relmax(t[2], s[2]), g_ss=relmax(t[3], s[3]), g_w=relmax(t[4], s[4]))
    _report("samples/c2_tc_vs_simt_%dx%d" % (N, S), **e)
    assert e["rgb"] < 1e-4 and e["depth"] < 1e-4, e
    assert e["g_c2w"] < 2e-3 and e["g_ss"] < 2e-3 and e["g_w"] < 5e-3, e


@pytest.mark.parametrize("N,S", [(333, 16), (301, 17), (97, 21), (130, 40), (77, 100)])
def test_ragged_small_s_tc_vs_simt(N, S):
    """the tensor-core engine against the exact-fp32 engine at small S, where one 64-row block overlaps up to 5 rays (S = 17, 21: the
    size of the per-ray bias buffer), with N*S not a multiple of the 128-sample tile (gates of test_gpu_parity's ragged-tile test)"""
    GP.test_ragged_last_tile_tc_vs_simt(N, S)


def test_render_frame_s512_tc_vs_simt():
    """Extract_Images.render_frame (the frame renderer of Extract_Images and Eval_Images) at 512 samples per ray on a row block of a
    1080 x 1920 frame: the tensor-core engine against the exact-fp32 engine"""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    H, W, S = 1080, 1920, 512
    cfg = default_cfg(); cfg["rendering"]["num_points"] = S; cfg["extract_images"] = {"resolution": (H, W)}
    dev = torch.device("cuda")
    c2w = cuda(O.make_c2w(np.array([0.02, -0.03, 0.01], np.float32), np.array([0.05, 0.0, -0.04], np.float32)))
    cam = torch.diag(torch.tensor([1.2, -2.1, -1.0, 1.0])).to(dev)
    res = {}
    for eng in ("simt", "tc"):
        ops.set_default_engine(eng)
        net = mdl.OfficialStaticNerf(cfg)
        net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=7, hf_damp=True).items()})
        ex = mdl.Extract_Images(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev, render_type="nope_nerf")
        rgb, depth = ex.render_frame(c2w, cam, H, W, rows=(531, 549))
        torch.cuda.synchronize()
        assert rgb.shape[:2] == (18, W)
        res[eng] = (rgb.cpu().numpy(), depth.cpu().numpy())
    e = dict(rgb=relmax(res["tc"][0], res["simt"][0]), depth=relmax(res["tc"][1], res["simt"][1]))
    _report("samples/render_frame_s512", **e)
    assert e["rgb"] < 1e-4 and e["depth"] < 1e-4, e


def test_trainer_pose_s100_vs_oracle(monkeypatch):
    """Trainer_pose at 100 samples per ray on both engines against the fp64 oracle (gates of test_gpu_parity.test_trainer_pose_vs_oracle).
    Weights from init_params(hf_damp=True), as in the `_damped` goldens: with the default initialisation a few hidden-unit ReLU gates sit
    within fp32 rounding of zero, and the pose gradient then depends on which side each evaluation order puts them."""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    H, W, V, N, S = 30, 40, 4, 64, 100
    rng = np.random.default_rng(6)
    cfg = default_cfg(); cfg["rendering"]["num_points"] = S; cfg["eval_pose"]["n_points"] = N
    dev = torch.device("cuda")
    P = O.init_params(seed=13, hf_damp=True)
    r0 = rng.normal(0, .05, (V, 3)).astype(np.float32); t0 = rng.normal(0, .05, (V, 3)).astype(np.float32)
    img = rng.uniform(0, 1, (3, H, W)).astype(np.float32)
    ray_idx = rng.permutation(H * W)[:N]
    kx, ky = 1.2, -1.6
    ocfg = dict(O.DEFAULT_CFG); ocfg["num_points"] = S
    c2w = O.make_c2w(r0[2].astype(np.float64), t0[2].astype(np.float64))
    P64 = {k: v.astype(np.float64) for k, v in P.items()}
    out, cache = O.render_forward(P64, O.pixels_from_idx(ray_idx, H, W, np.float64), np.ones(N), c2w, kx, ky, ocfg, noise=None, eval_=True)
    gt = img.reshape(3, -1)[:, ray_idx].T.astype(np.float64)
    loss = ((out["rgb"] - gt) ** 2).mean()
    gr = O.render_backward(P64, cache, 2 * (out["rgb"] - gt) / (3 * N), np.zeros(N), np.zeros(N))
    g_r, g_t = O.make_c2w_bwd(r0[2].astype(np.float64), t0[2].astype(np.float64), None, gr["c2w"])
    monkeypatch.setattr(torch, "randperm", lambda n, device=None: cuda(ray_idx))
    for eng in ("simt", "tc"):
        ops.set_default_engine(eng)
        net = mdl.OfficialStaticNerf(cfg)
        net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in P.items()})
        model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
        pose = mdl.LearnPose(V, True, True, cfg).to(dev)
        with torch.no_grad():
            pose.r.copy_(cuda(r0)); pose.t.copy_(cuda(t0))
        tp = mdl.Trainer_pose(model, cfg["eval_pose"], device=dev, optimizer_pose=torch.optim.Adam(pose.parameters(), lr=1e-3),
                              pose_param_net=pose)
        cam = torch.tensor([[kx, 0, 0, 0], [0, ky, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
        data = {"img": torch.from_numpy(img)[None], "img.idx": torch.tensor([2]), "img.camera_mat": cam, "img.scale_mat": torch.eye(4)[None]}
        ld = tp.train_step(data)
        e = dict(loss=abs(ld["loss"].item() - loss) / loss, g_r=relmax(pose.r.grad.cpu().numpy()[2], g_r), g_t=relmax(pose.t.grad.cpu().numpy()[2], g_t))
        _report("samples/trainer_pose_s100/%s" % eng, **e)
        assert e["loss"] < 1e-5 and e["g_r"] < 2e-4 and e["g_t"] < 2e-4, (eng, e)


def test_pick_engine():
    """the tensor-core engine by default for 16 <= S <= 1024, the exact-fp32 engine below; an explicit SIMT choice is kept"""
    from nope_nerf_b200 import ops, _lib as L
    ops.set_default_engine("tc")
    for S in (16, 48, 100, 200, 256, 300, 1024):
        assert ops.pick_engine(None, S) == L.ENGINE_TC, S
        assert ops.pick_engine(L.ENGINE_TC, S) == L.ENGINE_TC, S
        assert ops.pick_engine(L.ENGINE_SIMT, S) == L.ENGINE_SIMT, S
    for S in (2, 8, 15):
        assert ops.pick_engine(None, S) == L.ENGINE_SIMT, S
    ops.set_default_engine("simt")
    assert ops.pick_engine(None, 100) == L.ENGINE_SIMT


def test_sample_count_c_abi_errors():
    """nnb_render_fwd rejects S = 1 and S = 1025 on both engines and S = 8 on the tensor-core engine, and runs S = 8 (SIMT), 16 (TC) and
    1024 (both)"""
    from nope_nerf_b200 import _lib as L
    N = 8
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    w = cuda(O.flatten_params(O.init_params(seed=1))); eye = torch.eye(4, device="cuda")
    pix = torch.full((N, 2), 0.1, device="cuda"); dep = torch.ones(N, device="cuda")
    outs = [torch.empty(N, 3, device="cuda"), torch.empty(N, device="cuda"), torch.empty(N, device="cuda"), torch.empty(N, dtype=torch.uint8, device="cuda")]
    ws = torch.empty(max(L.lib.nnb_workspace_bytes(N, 1024, 0, e) for e in (L.ENGINE_SIMT, L.ENGINE_TC)), dtype=torch.uint8, device="cuda")

    def call(S, engine):
        a = L.RenderArgs()
        a.weights, a.c2w, a.cam, a.pixels, a.depth = w.data_ptr(), eye.data_ptr(), eye.data_ptr(), pix.data_ptr(), dep.data_ptr()
        a.N, a.S, a.near_, a.far_, a.engine = N, S, 0.1, 1.0, engine
        a.rgb, a.depth_pred, a.depth_gt, a.mask = (o.data_ptr() for o in outs)
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        return L.lib.nnb_render_fwd(C.byref(a), st), L.lib.nnb_last_error()
    for engine in (L.ENGINE_SIMT, L.ENGINE_TC):
        for S in (1, 1025):
            rc, msg = call(S, engine)
            assert rc < 0 and b"S must be in [2,1024]" in msg, (S, engine, rc, msg)
    rc, msg = call(8, L.ENGINE_TC)
    assert rc < 0 and b"tensor-core engine needs S in [16,1024]" in msg, (rc, msg)
    for S, engine in ((8, L.ENGINE_SIMT), (16, L.ENGINE_TC), (1024, L.ENGINE_SIMT), (1024, L.ENGINE_TC)):
        rc, msg = call(S, engine)
        assert rc == 0, (S, engine, msg)
        torch.cuda.synchronize()
        assert torch.isfinite(outs[0]).all(), (S, engine)

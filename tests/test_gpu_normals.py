"""GPU: rendering.normal_loss and the differentiable OfficialStaticNerf.gradient.
(1) Renderer.nope_nerf's out['normal'] (diff_norm) and the gradients of a fixed weighting of it with respect to the MLP, r, t, kx / ky,
scale and shift against the unmodified reference (tools/make_golden.py normals; the stored neighbour offsets replace the draw), within
max(1e-4 max|fp64|, 3 max|fp32 - fp64|) of the reference's own runs (the distortion gradients also within the envelope of d/d t
that they are sums of, see the test); (2) gradient() values are the bits of the first-order path
(nnb_field_bwd with cotangent 1 on the logit), with a grad_fn when p requires grad, and a third derivative raises; (3) the CUDA-graph training step with normal_loss gives the
bits of normal_loss False, and the eager step leaves the CUDA generator where the reference's draws leave it; (4) no valid prior / no
points: empty results without a library call."""
import numpy as np
import pytest
import torch

from _util import load_golden
from oracle import nerf_oracle as O
import _normals_ref as NR

pytestmark = pytest.mark.gpu


def _net(D, seed=61, hf_damp=True, normal_loss=True, sample_option="uniform"):
    import nope_nerf_b200.model as mdl
    from _cfg import default_cfg
    cfg = default_cfg()
    cfg["model"]["hidden_dim"] = D
    cfg["rendering"]["normal_loss"] = normal_loss
    cfg["rendering"]["sample_option"] = sample_option
    if sample_option == "ndc":
        cfg["rendering"]["dist_alpha"] = True; cfg["rendering"]["depth_range"] = [0.0, 1.0]
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=seed, D=D, hf_damp=hf_damp).items()})
    net = net.cuda()
    return cfg, net, mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"))


def _golden_run(g, name, grad_inputs=True):
    """Renderer.nope_nerf on a fixture's inputs with its neighbour offsets, backward of the fixed weighting of out['normal'];
    grad_inputs=False: pose, camera matrix and depth are plain tensors (only the MLP can receive gradients)"""
    from nope_nerf_b200 import ops
    D, N, S, cam = int(g["hidden_dim"]), int(g["N"]), int(g["S"]), int(g["cam_id"])
    cfg, net, rend = _net(D, seed=int(g["seed"]), sample_option="ndc" if "ndc" in name else "uniform")
    cfg["rendering"]["num_points"] = S
    cu = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    r = cu(g["r"]).requires_grad_(grad_inputs); t = cu(g["t"]).requires_grad_(grad_inputs)
    c2w = ops.pose_c2w(r, t, None, cam)
    kxy = torch.tensor([float(g["kx"]), float(g["ky"])], device="cuda", requires_grad=grad_inputs)
    z4 = torch.zeros(4, device="cuda"); one = torch.ones(1, device="cuda")
    camera_mat = torch.cat([kxy[0:1], z4, kxy[1:2], z4, -one, z4, one]).view(1, 4, 4)
    scale = torch.tensor(float(g["scale"]), device="cuda", requires_grad=grad_inputs)
    shift = torch.tensor(float(g["shift"]), device="cuda", requires_grad=grad_inputs)
    _, raw = NR.inputs(g)
    depth = cu(raw) * scale + shift
    out = rend.nope_nerf(cu(g["pixels"])[None], depth, camera_mat, None, None, add_noise=False, it=0, c2w=c2w,
                         normal_noise=cu(g["nbr"]))
    dn = out["normal"]
    assert dn.shape == (N,)
    (dn * cu(g["wts"])).sum().backward()
    got = {"diff_norm": dn.detach().cpu().numpy()}
    if grad_inputs:
        got.update(grad_r=r.grad[cam].cpu().numpy(), grad_t=t.grad[cam].cpu().numpy(), grad_kxy=kxy.grad.cpu().numpy(),
                   grad_scale=scale.grad.cpu().numpy(), grad_shift=shift.grad.cpu().numpy())
    for n_, prm in net.named_parameters():
        got["pg." + n_] = np.zeros(prm.numel()) if prm.grad is None else prm.grad.reshape(-1).cpu().numpy()
    return got, raw


@pytest.mark.parametrize("name", NR.NAMES)
def test_normal_loss_vs_reference_golden(name):
    g = load_golden(name)
    got, raw = _golden_run(g, name)
    report = {}
    # d/d scale and d/d shift are one sum over the rays of (d L / d x) . (d x / d depth), |d x / d depth| = |ray_vector| <= 1.5 here
    # (|x / kx|, |y / ky| <= 0.84): besides their own rule they get the envelope of d/d t, the sum of the same d L / d x, times that bound
    # (and the largest raw depth for the scale).  One scalar's fp32-vs-fp64 difference alone is a noisy estimate of the rounding level.
    # Measured on NVIDIA H100 80GB HBM3 (700 W power limit), error over the plain rule max(1e-4 |fp64|, 3 |fp32 - fp64|): grad_shift
    # 1.45x (normals_ndc_d64: 0.171 against 0.118, value 387.4) and 2.01x (normals_uniform_d256: 1.12 against 0.559, value -51.1),
    # grad_scale 1.73x (normals_uniform_d256: 7.09 against 4.10, value -2525); every other quantity within the plain rule (at most
    # 0.85 of it).  With the envelope the largest ratio is 0.85.
    t_env = 3 * float(np.abs(g["grad_t.f32"].astype(np.float64) - g["grad_t.f64"]).max()) * 1.5
    extra = {"grad_shift": t_env, "grad_scale": t_env * float(raw.max())}
    for key in [k[:-4] for k in g if k.endswith(".f64")]:
        err, tol = NR.gate(g, key, NR.sel(g, key, got[key]))
        report[key] = (err, max(tol, extra.get(key, 0.0)))
    bad = {k: v for k, v in report.items() if not v[0] <= v[1]}
    print(name, "worst err/tol", max(v[0] / max(v[1], 1e-30) for v in report.values()))
    assert not bad, bad


@pytest.mark.parametrize("name", ["normals_uniform_d64", "normals_ndc_d256"])
def test_normal_loss_trains_mlp_with_fixed_inputs(name):
    """with pose, camera matrix and depth that carry no gradient, out['normal'] still reaches the MLP, as in the reference (whose
    gradient() sets requires_grad on the points itself): the MLP gradients are the bits of the run with gradient-carrying inputs,
    which the golden test gates against the reference, and they are non-zero"""
    g = load_golden(name)
    a, _ = _golden_run(g, name, grad_inputs=True)
    b, _ = _golden_run(g, name, grad_inputs=False)
    assert a["diff_norm"].tobytes() == b["diff_norm"].tobytes()
    for k in a:
        if k.startswith("pg."):
            assert a[k].tobytes() == b[k].tobytes(), k
    assert np.abs(b["pg.layers0.0.weight"]).max() > 0 and np.abs(b["pg.fc_density.weight"]).max() > 0


@pytest.mark.parametrize("D", [64, 256])
def test_gradient_autograd_is_field_hvp(D):
    """the autograd glue of gradient(): an eikonal-style loss on gradient(p) gives p and the MLP the bits of one nnb_field_hvp call
    with the cotangent that reaches n (tests/test_gpu_field_hvp.py checks that call against float64 double backward)"""
    from test_gpu_field_hvp import hvp_call
    P = O.init_params(seed=4, D=D)
    _, net, _ = _net(D, seed=4, hf_damp=False)
    rng = np.random.default_rng(D)
    p_np = rng.uniform(-1, 1, (777, 3)).astype(np.float32)
    p = torch.from_numpy(p_np).cuda().requires_grad_(True)
    out = net.gradient(p, 0)
    seen = []
    out.register_hook(lambda gr: seen.append(gr.detach().clone()))
    out.norm(dim=-1).mean().backward()
    u = (-seen[0][:, 0, :]).cpu().numpy()              # cotangent on n (gradient() returns -n)
    g_p, g_w, _ = hvp_call(P, D, p_np, u)
    assert p.grad.cpu().numpy().tobytes() == g_p.cpu().numpy().tobytes()
    flat_grad = torch.cat([q.grad.reshape(-1) if q.grad is not None else torch.zeros(q.numel(), device="cuda") for q in net.parameters()])
    assert flat_grad.cpu().numpy().tobytes() == g_w.cpu().numpy().tobytes()
    assert float(flat_grad.abs().max()) > 0


def test_gradient_bits_and_third_derivative():
    """gradient() equals the first-order path's bits (field_query + autograd.grad, the earlier implementation) with and without a
    graph; its result is differentiable once and a third derivative raises"""
    from nope_nerf_b200.field import field_query
    for D in (64, 256):
        _, net, _ = _net(D, seed=5, hf_damp=False)
        p = (torch.rand(3001, 3, generator=torch.Generator().manual_seed(D)) * 2 - 1).cuda()
        with torch.enable_grad():
            q = p.detach().clone().requires_grad_(True)
            _, s = field_query(net, q, None, raw_density=True)
            old, = torch.autograd.grad(s, q, torch.ones_like(s))
        old = -old.unsqueeze(1)
        new = net.gradient(p.clone().requires_grad_(True), 0)
        assert new.grad_fn is not None and new.shape == (3001, 1, 3)
        new_ng = net.gradient(p, 0)              # p without requires_grad: plain values, as before
        assert new_ng.grad_fn is None and not new_ng.requires_grad
        with torch.no_grad():
            new_nm = net.gradient(p.clone().requires_grad_(True), 0)
        assert new_nm.grad_fn is None
        for x in (new, new_ng, new_nm):
            assert x.detach().cpu().numpy().tobytes() == old.cpu().numpy().tobytes()
        pr = p.clone().requires_grad_(True)
        gn = net.gradient(pr, 0).norm(dim=-1).mean()
        g1, = torch.autograd.grad(gn, pr, create_graph=True)
        assert torch.isfinite(g1).all()
        with pytest.raises(RuntimeError):
            g1.sum().backward()


def test_no_surface_points_no_library_call(monkeypatch):
    import nope_nerf_b200.field as F
    cfg, net, rend = _net(64)
    cfg["rendering"]["num_points"] = 16

    def boom(*a, **k):
        raise AssertionError("library called")
    monkeypatch.setattr(F._GradFn, "apply", boom)
    assert net.gradient(torch.zeros(0, 3, device="cuda"), 0).shape == (0, 1, 3)
    pe = torch.zeros(0, 3, device="cuda", requires_grad=True)
    ge = net.gradient(pe, 0)
    assert ge.shape == (0, 1, 3) and ge.grad_fn is not None
    ge.norm(dim=-1).sum().backward()                   # an empty batch gives zero gradients instead of raising
    assert pe.grad is not None and pe.grad.shape == (0, 3)
    N = 32
    pix = (torch.rand(1, N, 2, generator=torch.Generator().manual_seed(1)) * 2 - 1).cuda()
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], device="cuda")[None]
    out = rend.nope_nerf(pix, torch.zeros(N, device="cuda"), cam, None, None, add_noise=False, it=0, c2w=torch.eye(4, device="cuda"))
    assert out["normal"] is not None and out["normal"].shape == (0,)
    out = rend.nope_nerf(pix, torch.ones(N, device="cuda"), cam, None, None, add_noise=False, it=0, eval_=True, c2w=torch.eye(4, device="cuda"))
    assert out["normal"] is None


def _trainer(normal_loss, use_cuda_graph, depth_loss_type="l1"):
    import nope_nerf_b200.model as mdl
    from _cfg import default_cfg
    from nope_nerf_b200 import ops
    ops.set_default_engine("tc")
    cfg = default_cfg()
    N, S, V = 256, 32, 4
    cfg["training"]["n_training_points"] = N; cfg["rendering"]["num_points"] = S
    cfg["training"]["pc_weight"] = [0.0, 0.0]; cfg["training"]["rgb_s_weight"] = [0.0, 0.0]
    cfg["training"]["depth_loss_type"] = depth_loss_type
    cfg["rendering"]["normal_loss"] = normal_loss
    dev = torch.device("cuda")
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=9, hf_damp=True).items()})
    model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
    pose = mdl.LearnPose(V, True, True, cfg).to(dev); dist = mdl.Learn_Distortion(V, True, True, cfg).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3); opt_p = torch.optim.Adam(pose.parameters(), lr=5e-4)
    opt_d = torch.optim.Adam(dist.parameters(), lr=5e-4)
    tr = mdl.Trainer(model, opt, cfg["training"], device=dev, optimizer_pose=opt_p, pose_param_net=pose, optimizer_distortion=opt_d,
                     distortion_net=dist, use_cuda_graph=use_cuda_graph)
    return tr, net, pose, dist, N, S


def _frames(V=4, H=48, W=64):
    g = torch.Generator().manual_seed(3)
    return [dict(img=torch.rand(1, 3, H, W, generator=g).cuda(), dpt=(torch.rand(1, 12, 16, generator=g) * 3 + 2).cuda()) for _ in range(V)]


def _data(fr, i):
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
    return {"img": fr["img"], "img.idx": torch.tensor([i]), "img.dpt": fr["dpt"], "img.camera_mat": cam, "img.scale_mat": torch.eye(4)[None]}


def test_graph_step_normal_loss_same_bits():
    frames = _frames()
    res = {}
    for nl in (False, True):
        torch.manual_seed(0)
        tr, net, pose, dist, _, _ = _trainer(nl, True)
        losses = []
        for it in range(4):
            ld = tr.train_step(_data(frames[it % 4], it % 4), it=it, epoch=0, scheduling_start=10000, render_path=None)
            losses.append(torch.stack([ld[k].detach().reshape(()) for k in ("loss", "loss_rgb", "loss_depth")]))
        torch.cuda.synchronize()
        res[nl] = [torch.stack(losses).cpu().numpy().tobytes(), net.flat_weights().cpu().numpy().tobytes(), pose.r.detach().cpu().numpy().tobytes(),
                   pose.t.detach().cpu().numpy().tobytes(), dist.global_scales.detach().cpu().numpy().tobytes()]
    assert res[False] == res[True]


@pytest.mark.parametrize("path", ["fixed", "general"])
def test_eager_step_keeps_reference_random_stream(path):
    """one eager step with normal_loss: randperm, the sample jitter rand(1, N, S) and the neighbours' rand(n_valid, 3), in that order"""
    frames = _frames()
    torch.manual_seed(1)
    tr, net, pose, dist, N, S = _trainer(True, False, depth_loss_type="invariant" if path == "general" else "l1")
    h, w = frames[0]["img"].shape[-2:]
    s0 = torch.cuda.get_rng_state()
    tr.train_step(_data(frames[1], 1), it=0, epoch=0, scheduling_start=10000, render_path=None)
    torch.cuda.synchronize()
    s1 = torch.cuda.get_rng_state()
    torch.cuda.set_rng_state(s0)
    torch.randperm(h * w, device="cuda")
    torch.rand(1, N, S, device="cuda")
    torch.rand(N, 3, device="cuda")          # every prior depth is positive: all N rays are valid
    assert torch.equal(torch.cuda.get_rng_state(), s1)
    torch.cuda.set_rng_state(s0)
    torch.randperm(h * w, device="cuda")
    torch.rand(1, N, S, device="cuda")
    assert not torch.equal(torch.cuda.get_rng_state(), s1)

"""GPU: full-loss training steps are reproducible bit for bit.
(1) the dense chamfer equals float64 numpy exactly on planted inputs whose every term and partial sum is exact, so the group sums
count every contribution once, and a non-finite term still shows; (2) the chamfer and the reference-image stage give the same bytes twice on identical inputs,
and the stage keeps its fp64 oracle gates; (3) the CUDA-graph step equals the eager run of the same step body bit for bit with the
full losses on; (4) the general path (Trainer.compute_loss, torch.optim.Adam, learned focal) run twice gives identical bits; (5) with two GPUs, a
dp_mode='views' full-loss run twice gives identical parameters (skipped on one GPU)."""
import numpy as np
import pytest
import torch

from _util import load_golden, relmax
from oracle import nerf_oracle as O
import _refopts_oracle as RO
from test_gpu_parity import _build_trainer, _report, cuda

pytestmark = pytest.mark.gpu

AXES = np.eye(3)


def _cluster_case(rng, P, Q, spacing=64.0, max_pow=3, zero=False):
    """Q centres far apart on the x axis; every X point sits at a centre plus (+-2^k) along one axis (k <= max_pow), or on the centre
    itself when zero=True and the draw says so.  Every nearest-neighbour vector is then axis-aligned with a power-of-two length (or 0)."""
    Y = np.stack([np.arange(Q) * spacing, np.zeros(Q), np.zeros(Q)], -1)
    owner = np.concatenate([np.arange(Q), rng.integers(0, Q, P - Q)]) if P >= Q else rng.integers(0, Q, P)
    off = AXES[rng.integers(0, 3, P)] * (rng.choice([-1.0, 1.0], P) * 2.0 ** rng.integers(0, max_pow + 1, P))[:, None]
    if zero:
        off[rng.random(P) < 0.25] = 0.0
    return Y[owner] + off, Y


def _planted(name):
    rng = np.random.default_rng(11)
    if name == "one_nn":        # every X point's nearest neighbour is Y[0] (4096 pairs in one group); Y[1] ties between X[-1] and Y[0]
        X, _ = _cluster_case(rng, 4095, 1)
        X = np.concatenate([X, [[512.0, 0.0, 0.0]]])
        Y = np.array([[0.0, 0.0, 0.0], [1024.0, 0.0, 0.0]])
    elif name == "ties":        # X halfway between consecutive Y (first index wins), Y halfway between consecutive X
        Y = np.stack([np.arange(8) * 4.0, np.zeros(8), np.zeros(8)], -1)
        X = Y + np.array([2.0, 0.0, 0.0])
    elif name == "p_ne_q":
        X, Y = _cluster_case(rng, 256, 16)
    elif name == "p1":
        Y = np.array([[1.0, 0, 0], [0, -2.0, 0], [0, 0, 4.0], [-1.0, 0, 0]]) + np.array([3.0, 5.0, -7.0])
        X = np.array([[3.0, 5.0, -7.0]])
    elif name == "zero_dist":
        X, Y = _cluster_case(rng, 128, 32, zero=True)
    return X.astype(np.float32), Y.astype(np.float32)


def _native_chamfer(X, Y):
    from nope_nerf_b200 import ops
    tx = cuda(X).requires_grad_(True); ty = cuda(Y).requires_grad_(True)
    l = ops.chamfer(tx, ty)
    l.backward()
    torch.cuda.synchronize()
    return l.detach().cpu().numpy().reshape(1), tx.grad.cpu().numpy(), ty.grad.cpu().numpy()


@pytest.mark.parametrize("name", ["one_nn", "ties", "p_ne_q", "p1", "zero_dist"])
def test_chamfer_exact_on_planted_inputs(name):
    X, Y = _planted(name)
    l, gX, gY, ixy, iyx = O.chamfer(X.astype(np.float64), Y.astype(np.float64))
    for A, B, idx in ((X, Y, ixy), (Y, X, iyx)):        # the planting holds: axis-aligned, power-of-two (or zero) pair vectors
        v = np.abs(A.astype(np.float64) - B[idx])
        assert ((v > 0).sum(-1) <= 1).all()
        n = v.sum(-1)
        assert ((n == 0) | (n == 2.0 ** np.round(np.log2(np.where(n > 0, n, 1))))).all()
    assert len(X) & (len(X) - 1) == 0 and len(Y) & (len(Y) - 1) == 0
    if name == "one_nn":
        assert (ixy == 0).all()
    if name == "zero_dist":
        assert (np.abs(X.astype(np.float64) - Y[ixy]).sum(-1) == 0).any()
    gl, ggX, ggY = _native_chamfer(X, Y)
    for got, ref in ((gl, np.array([l])), (ggX, gX), (ggY, gY)):
        ref32 = ref.astype(np.float32)
        assert np.array_equal(ref32.astype(np.float64), ref), "planted case is not exact in float32"
        assert got.tobytes() == ref32.tobytes(), (name, np.abs(got - ref32).max())


def test_chamfer_non_finite_term_shows():
    """an infinite coordinate makes its own pair's term NaN; the adjoint of that pair's target comes out NaN, the others stay finite"""
    X, Y = _planted("p_ne_q")
    X[5, 1] = np.inf
    _, ggX, ggY = _native_chamfer(X, Y)
    assert np.isnan(ggX[5]).any() and np.isnan(ggY[0]).any()
    bad_y = np.isnan(ggY).any(-1); bad_x = np.isnan(ggX).any(-1)
    assert bad_y.sum() == 1 and bad_x.sum() == 1, (np.nonzero(bad_x), np.nonzero(bad_y))


@pytest.mark.parametrize("case", ["random", "one_nn"])
def test_chamfer_same_bits_twice(case):
    """C2 size (P = Q = 16 128) twice on identical inputs; a smaller pair against the fp64 oracle"""
    rng = np.random.default_rng(5)
    P = 96 * 168
    X = rng.normal(size=(P, 3)).astype(np.float32)
    Y = (rng.normal(size=(P, 3)) + 0.05).astype(np.float32)
    if case == "one_nn":                                  # every X point's nearest neighbour is the same Y point
        Y[1:] += 100.0
    a, b = _native_chamfer(X, Y), _native_chamfer(X, Y)
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()
    Xs, Ys = X[:2000], Y[:1500]
    l, gX, gY, _, _ = O.chamfer(Xs.astype(np.float64), Ys.astype(np.float64))
    gl, ggX, ggY = _native_chamfer(Xs, Ys)
    e = dict(loss=abs(float(gl[0]) - l) / l, gX=relmax(ggX, gX), gY=relmax(ggY, gY))
    _report("repro/chamfer/%s" % case, **e)
    assert all(v < 1e-4 for v in e.values()), e


def _c2_inputs():
    rng = np.random.default_rng(17)
    H, W, hd, wd = 216, 384, 384, 672
    up = lambda t, size: torch.nn.functional.interpolate(torch.from_numpy(t)[None], size, mode="bilinear", align_corners=False)[0].numpy()
    img = up(rng.uniform(0, 1, (3, 18, 32)).astype(np.float32), (H, W)); ref = up(rng.uniform(0, 1, (3, 18, 32)).astype(np.float32), (H, W))
    dpt = up(rng.uniform(1.5, 6, (1, 12, 21)).astype(np.float32), (hd, wd))[0]; rdpt = up(rng.uniform(1.5, 6, (1, 12, 21)).astype(np.float32), (hd, wd))[0]
    c2w = O.make_c2w(rng.normal(0, 0.03, 3).astype(np.float32), rng.normal(0, 0.05, 3).astype(np.float32)).astype(np.float32)
    c2wr = O.make_c2w(rng.normal(0, 0.03, 3).astype(np.float32), rng.normal(0, 0.05, 3).astype(np.float32)).astype(np.float32)
    return img, ref, dpt, rdpt, c2w, c2wr, (1.03, 0.02), (0.97, -0.04), 1.2, -1.6


@pytest.mark.parametrize("is_last", [False, True])
@pytest.mark.parametrize("with_ssim,grad_ref", [(False, False), (True, True)])
def test_refstage_c2_same_bits_twice(is_last, with_ssim, grad_ref):
    """ops.refstage at C2 size twice: losses and every gradient byte-identical; the fp64 oracle gates of test_gpu_refopts"""
    from nope_nerf_b200 import ops
    img, ref, dpt, rdpt, c2w, c2wr, dc, dr, kx, ky = _c2_inputs()

    def run():
        c2w_t = cuda(c2w).requires_grad_(True); dist = torch.tensor(dc, device="cuda", requires_grad=True)
        c2wr_t = cuda(c2wr).requires_grad_(grad_ref); distr = torch.tensor(dr, device="cuda", requires_grad=grad_ref)
        total, losses = ops.refstage(c2w_t, dist, c2wr_t, distr, cuda(img), cuda(ref), cuda(dpt), cuda(rdpt), is_last, kx, ky,
                                     with_ssim=with_ssim)
        total.backward()
        out = [total.detach(), losses, c2w_t.grad, dist.grad] + ([c2wr_t.grad, distr.grad] if grad_ref else [])
        return [t.cpu().numpy() for t in out]

    a, b = run(), run()
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()
    cfg = dict(O.REF_CFG, with_ssim=with_ssim, detach_ref_img=not grad_ref)
    f64 = lambda x: np.asarray(x, np.float64)
    l, gr = RO.ref_stage(f64(img), f64(ref), f64(dpt), f64(rdpt), f64(c2w), f64(c2wr), dc[0], dc[1], dr[0], dr[1], is_last, kx, ky, cfg=cfg)
    e = dict(loss_pc=abs(a[1][0] - l["loss_pc"]) / l["loss_pc"], loss_rgb_s=abs(a[1][1] - l["loss_rgb_s"]) / l["loss_rgb_s"],
             g_c2w=relmax(a[2][:3], gr["c2w"][:3]), g_dist=relmax(a[3], np.array([gr["scale"], gr["shift"]])))
    if grad_ref:
        e.update(g_c2w_ref=relmax(a[4][:3], gr["c2w_ref"][:3]), g_dist_ref=relmax(a[5], np.array([gr["scale_ref"], gr["shift_ref"]])))
    _report("repro/refstage/last%d_ssim%d_ref%d" % (is_last, with_ssim, grad_ref), **e)
    assert all(v <= 1e-4 for v in e.values()), e


@pytest.mark.parametrize("with_ssim,detach_ref_img", [(False, True), (True, False)])
def test_graph_replay_equals_eager_full_loss_bits(with_ssim, detach_ref_img, monkeypatch):
    """the setup of test_gpu_refopts.test_graph_replay_equals_eager_refopts (tensor-core engine, injected draws, full losses from the
    first step): graph replay and the eager run of the same step body give bit-identical losses, r, t, scales, shifts and weights"""
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
    steps = 5
    draws = [(torch.randperm(H * W, generator=g)[:N].cuda(), torch.rand(N, S, generator=g).cuda()) for _ in range(steps)]
    ray_buf = torch.zeros(N, dtype=torch.int64, device=dev); noise_buf = torch.zeros(1, N, S, device=dev)
    monkeypatch.setattr(torch, "randperm", lambda n, device=None: ray_buf)
    monkeypatch.setattr(torch, "rand", lambda *a, **k: noise_buf)
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
    res = {}
    for mode in (False, True):
        cfg = default_cfg()
        cfg["training"]["n_training_points"] = N; cfg["rendering"]["num_points"] = S
        cfg["training"]["annealing_epochs"] = 10
        cfg["training"]["with_ssim"] = with_ssim; cfg["training"]["detach_ref_img"] = detach_ref_img
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
        for it in range(steps):
            ray_buf.copy_(draws[it][0]); noise_buf[0].copy_(draws[it][1])
            i = (it * 2 + 1) % (V - 1)
            data = {"img": frames[i]["img"], "img.idx": torch.tensor([i]), "img.dpt": frames[i]["dpt"], "img.camera_mat": cam,
                    "img.scale_mat": torch.eye(4)[None], "img.ref_imgs": frames[i + 1]["img"], "img.ref_dpts": frames[i + 1]["dpt"],
                    "img.ref_idxs": torch.tensor([i + 1])}
            ld = tr.train_step(data, it=it, epoch=it, scheduling_start=3, render_path=None)
            losses.append([ld[k].item() for k in ("loss", "loss_rgb", "loss_depth", "loss_pc", "loss_rgb_s")])
        if mode:
            gsteps = [v for v in tr._gsteps.values() if v]
            assert len(gsteps) == 1 and gsteps[0].graph is not None and gsteps[0].calls == steps
        res[mode] = dict(losses=np.array(losses, np.float32), w=net.flat_weights().detach().cpu().numpy().copy(),
                         r=pose.r.detach().cpu().numpy().copy(), t=pose.t.detach().cpu().numpy().copy(),
                         scales=dist.global_scales.detach().cpu().numpy().copy(), shifts=dist.global_shifts.detach().cpu().numpy().copy())
    assert res[False]["losses"][:, 3].min() > 0 and res[False]["losses"][:, 4].min() > 0
    for k in res[False]:
        assert res[False][k].tobytes() == res[True][k].tobytes(), (k, np.abs(res[False][k] - res[True][k]).max())


def _run_general(name, monkeypatch):
    """two reference Trainer.train_step calls of golden `name` through Trainer.compute_loss (fused_adam False, torch.optim.Adam)"""
    g = load_golden(name)
    trainer, net, pose, dist = _build_trainer(g, "tc", True)
    trainer.fused_adam = False
    kx, ky = float(g["kx"]), float(g["ky"])
    cam = np.array([[kx, 0, 0, 0], [0, ky, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], np.float32)
    data = {"img": torch.from_numpy(g["img"])[None], "img.idx": torch.tensor([int(g["idx"])]),
            "img.dpt": torch.from_numpy(g["dpt"])[None], "img.camera_mat": torch.from_numpy(cam)[None],
            "img.scale_mat": torch.eye(4)[None], "img.ref_imgs": torch.from_numpy(g["ref"])[None],
            "img.ref_dpts": torch.from_numpy(g["rdpt"])[None], "img.ref_idxs": torch.tensor([int(g["ref_idx"])])}
    state = {"it": 0}
    monkeypatch.setattr(torch, "randperm", lambda n, device=None: cuda(g["ray_idx_%d" % state["it"]]))
    monkeypatch.setattr(torch, "rand", lambda *a, **k: cuda(g["noise_%d" % state["it"]])[None])
    losses = []
    for it in range(int(g["steps"])):
        state["it"] = it
        ld = trainer.train_step(data, it=it + 1, epoch=0, scheduling_start=10000, render_path="/tmp")
        losses.append([float(ld[k].reshape(-1)[0]) for k in ("loss", "loss_pc", "loss_rgb_s")])
    torch.cuda.synchronize()
    out = dict(losses=np.array(losses, np.float32), w=net.flat_weights().detach().cpu().numpy().copy(),
               r=pose.r.detach().cpu().numpy().copy(), t=pose.t.detach().cpu().numpy().copy(),
               scales=dist.global_scales.detach().cpu().numpy().copy(), shifts=dist.global_shifts.detach().cpu().numpy().copy())
    if trainer._test_focal is not None:
        out["focal"] = torch.stack([trainer._test_focal.fx.detach(), trainer._test_focal.fy.detach()]).reshape(-1).cpu().numpy()
    return out


@pytest.mark.parametrize("name", ["train_full_losses", "train_learn_focal"])
def test_general_path_same_bits_twice(name, monkeypatch):
    a, b = _run_general(name, monkeypatch), _run_general(name, monkeypatch)
    assert a["losses"][:, 1].min() > 0
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), (k, np.abs(a[k] - b[k]).max())


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("peer", [0, 1])
def test_dp_views_full_loss_same_bits_twice(peer, tmp_path):
    """the 2-rank dp_mode='views' worker of test_gpu_multi (CUDA graph, full losses: pc_weight = rgb_s_weight = 1 before annealing)"""
    from test_gpu_multi import _run
    a = _run(str(tmp_path), "a", "views", 1, peer, 2)
    b = _run(str(tmp_path), "b", "views", 1, peer, 2)
    for k in ("g_first", "loss0", "w", "r", "t", "shifts"):
        assert a[k].tobytes() == b[k].tobytes(), k

"""GPU: nnb_render_frame_bwd (ops.render_frame_bwd, ops.render_frame_grad): the gradients of the volumetric
frame at t_min = 0 on the tensor-core engine, from reverse rounds over 32-sample chunks with a chunk-sized stash.
(1) the call's forward outputs equal nnb_render_fwd's bit for bit, and every gradient agrees with nnb_render_fwd (NNB_STASH) +
nnb_render_bwd on the same inputs to 1e-4 of each tensor's maximum (the two differ only in the order of their sums), over both density
heads, NDC and uniform sampling, dist_alpha, white_background, D = 64, 128 and 256, S = 16 ... 1024 and ragged N; (2) repeated calls and
workspaces filled with zeros, NaN bytes and 0x7E give the same bits; (3) the workspace grows with S by one float per ray and chunk, and a
call at N = 4096, S = 1024, D = 256 runs; (4) render_frame_grad under autograd gives render_autograd's outputs and gradients."""
import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
from test_gpu_parity import cuda

pytestmark = pytest.mark.gpu


def _flat(D, seed=7):
    return cuda(O.flatten_params(O.init_params(seed=seed, D=D, hf_damp=True)))


def _case(N, S, D, cfg_over=None, occ="softplus", eval_=False, seed=0):
    from nope_nerf_b200 import ops
    rng = np.random.default_rng(seed)
    cfg = dict(O.DEFAULT_CFG); cfg.update(cfg_over or {})
    ndc = cfg["sample_option"] == "ndc"
    H, W = 240, 320
    c2w = cuda(O.make_c2w(np.array([0.02, -0.03, 0.01], np.float32), np.array([0.05, 0.0, -0.04], np.float32)))
    cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0])).cuda()
    kw = dict(N=N, S=S, flags=ops.flags_from_cfg(cfg, occ, eval_=eval_), near=0.0 if ndc else 0.01, far=1.0 if ndc else 10.0,
              ray_idx=cuda(rng.permutation(H * W)[:N].astype(np.int64)),
              depth_map=cuda(rng.uniform(0.6, 7.2, (48, 64)).astype(np.float32)), scale=torch.tensor([1.05]).cuda(),
              shift=torch.tensor([0.02]).cuda(), H=H, W=W, hidden_dim=D)
    g_rgb = cuda(rng.normal(0, 1, (N, 3)).astype(np.float32))
    g_dp = cuda(rng.normal(0, 0.1, N).astype(np.float32))
    g_dg = cuda(rng.normal(0, 0.1, N).astype(np.float32))
    return _flat(D), c2w, cam, kw, (g_rgb, g_dp, g_dg)


def _frame_bwd(flat, c2w, cam, kw, gs):
    from nope_nerf_b200 import ops, _lib as L
    g_w = torch.zeros(L.num_params(kw["hidden_dim"]), device="cuda")
    g_c, g_k, g_ss = torch.zeros(4, 4, device="cuda"), torch.zeros(4, 4, device="cuda"), torch.zeros(2, device="cuda")
    outs = ops.render_frame_bwd(flat, c2w, cam, *gs, g_w, g_c, g_k, None, g_ss, **kw)
    return outs, (g_w, g_c, g_k, g_ss)


def _stash_bwd(flat, c2w, cam, kw, gs):
    from nope_nerf_b200 import ops, _lib as L
    call = ops.RenderCall(flat, c2w, cam, stash=True, engine=L.ENGINE_TC, **kw)
    outs = (call.rgb.clone(), call.depth_pred.clone(), call.depth_gt.clone(), call.mask.clone())
    g_w = torch.zeros(L.num_params(kw["hidden_dim"]), device="cuda")
    g_c, g_k, g_ss = torch.zeros(4, 4, device="cuda"), torch.zeros(4, 4, device="cuda"), torch.zeros(2, device="cuda")
    call.backward(*gs, g_w, g_c, g_k, None, g_ss)
    return outs, (g_w, g_c, g_k, g_ss)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(b.double().abs().max().item(), 1e-30))


def _check(case):
    from nope_nerf_b200.model.official_nerf import param_slices
    flat, c2w, cam, kw, gs = case
    fo, fg = _frame_bwd(flat, c2w, cam, kw, gs)
    so, sg = _stash_bwd(flat, c2w, cam, kw, gs)
    torch.cuda.synchronize()
    for x, y, name in zip(fo, so, ("rgb", "depth_pred", "depth_gt", "mask")):
        assert torch.equal(x, y), name
    worst = 0.0
    for (o, n, shape) in param_slices(kw["hidden_dim"]):
        ref = sg[0][o:o + n]
        if ref.abs().max() == 0:
            assert fg[0][o:o + n].abs().max() == 0
            continue
        e = _rel(fg[0][o:o + n], ref)
        worst = max(worst, e)
        assert e < 1e-4, (o, shape, e)
    e_pose = [_rel(fg[i], sg[i]) for i in (1, 2, 3)]
    print("frame_bwd vs stash bwd N=%d S=%d D=%d: worst dW %.2e, g_c2w %.2e, g_cam %.2e, g_scale_shift %.2e"
          % (kw["N"], kw["S"], kw["hidden_dim"], worst, *e_pose))
    assert max(e_pose) < 1e-4, e_pose
    return worst, e_pose


OPTS = [dict(), dict(dist_alpha=True), dict(white_background=True), dict(sample_option="ndc"),
        dict(dist_alpha=True, white_background=True, normalise_ray=False, use_ray_dir=False)]


@pytest.mark.parametrize("opt", range(len(OPTS)))
@pytest.mark.parametrize("occ", ["softplus", "relu"])
def test_matches_stash_backward_over_options(opt, occ):
    _check(_case(300, 48, 128, OPTS[opt], occ=occ, seed=opt))


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("N,S", [(257, 16), (1000, 48), (129, 128), (130, 512), (37, 1024)])
def test_matches_stash_backward_over_sizes(D, N, S):
    _check(_case(N, S, D, seed=N + S))


def test_eval_flag():
    _check(_case(200, 64, 256, eval_=True))


def test_deterministic_and_workspace_independent():
    from nope_nerf_b200 import ops, _lib as L
    flat, c2w, cam, kw, gs = _case(500, 80, 256, dict(dist_alpha=True), seed=5)
    ref = _frame_bwd(flat, c2w, cam, kw, gs)
    nbytes = L.lib.nnb_render_frame_bwd_workspace_bytes(kw["N"], kw["S"], 256)
    for fill in (0x00, 0xFF, 0x7E):
        ops._pool.give(torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda"))   # the next call takes this workspace
        got = _frame_bwd(flat, c2w, cam, kw, gs)
        for x, y in zip(got[0] + got[1], ref[0] + ref[1]):
            assert torch.equal(x, y), fill
    ops._pool.free.clear()


def test_workspace_growth_and_a_large_call():
    from nope_nerf_b200 import ops, _lib as L
    N = 4096
    sizes = {S: L.lib.nnb_render_frame_bwd_workspace_bytes(N, S, 256) for S in (128, 512, 1024)}
    print("nnb_render_frame_bwd_workspace_bytes(4096, S, 256):", sizes,
          "nnb_workspace_bytes_dim(4096, 1024, NNB_STASH):", L.lib.nnb_workspace_bytes_dim(N, 1024, L.STASH, L.ENGINE_TC, 256))
    for a, b in ((128, 512), (512, 1024)):
        assert sizes[b] - sizes[a] <= 4 * N * ((b - a) // 32) + 256
    free = torch.cuda.mem_get_info()[0]
    assert L.lib.nnb_workspace_bytes_dim(N, 1024, L.STASH, L.ENGINE_TC, 256) > free   # the stash path cannot be sized here
    flat, c2w, cam, kw, gs = _case(N, 1024, 256, seed=9)
    outs, grads = _frame_bwd(flat, c2w, cam, kw, gs)
    torch.cuda.synchronize()
    assert all(torch.isfinite(g).all() for g in grads) and grads[0].abs().max() > 0
    ref = ops.render_frame(flat, c2w, cam, engine=L.ENGINE_TC, **kw)
    for x, y in zip(outs, ref):
        assert torch.equal(x, y)
    ops._pool.free.clear()


def test_autograd_function():
    from nope_nerf_b200 import ops, _lib as L
    from nope_nerf_b200.model.official_nerf import param_slices
    flat, c2w, cam, kw, gs = _case(400, 64, 128, seed=3)
    params = [torch.nn.Parameter(flat[o:o + n].clone().view(shape)) for (o, n, shape) in param_slices(128)]
    depth = cuda(np.random.default_rng(4).uniform(0.6, 7.2, 400).astype(np.float32))
    res = []
    for fn in (ops.render_autograd, ops.render_frame_grad):
        c = c2w.clone().requires_grad_(True); d = depth.clone().requires_grad_(True)
        for p in params: p.grad = None
        meta = dict(N=400, S=64, flags=kw["flags"], engine=L.ENGINE_TC, near=kw["near"], far=kw["far"], ray_idx=kw["ray_idx"], H=kw["H"],
                    W=kw["W"], hidden_dim=128, param_slices=param_slices(128))
        flatp = torch.cat([p.detach().reshape(-1) for p in params])
        rgb, dp, dg, mask = fn(meta, flatp, c, cam, d, None, None, params)[:4]
        ((rgb * gs[0]).sum() + (dp * gs[1]).sum() + (dg * gs[2]).sum()).backward()
        res.append((rgb.detach(), [p.grad.clone() for p in params], c.grad.clone(), d.grad.clone()))
    assert torch.equal(res[0][0], res[1][0])
    for a, b in zip(res[1][1], res[0][1]):
        if b.abs().max() > 0:
            assert _rel(a, b) < 1e-4
    assert _rel(res[1][2], res[0][2]) < 1e-4 and _rel(res[1][3], res[0][3]) < 1e-4
    with pytest.raises(ValueError):
        ops.render_frame_grad(dict(meta, noise=torch.zeros(400, 64, device="cuda")), flatp, c2w, cam, depth, None, None, params)

"""GPU: nnb_render_frame (ops.render_frame, Renderer(frame_t_min=...)): the volumetric view of a frame with compositing fused into the
tensor-core forward.
(1) bit equality with nnb_render_fwd on the tensor-core engine at t_min = 0 over the rendering options, both density heads, every width,
sample counts with and without a partial last chunk, ragged / row-block / permuted rays and a whole 1080 x 1920 frame; (2) Eval_Images and
Extract_Images with frame_t_min = 0 against the default path and the stored reference results; (3) t_min > 0 on a field with surfaces:
unstopped rays exact, stopped rays within the header's bound; (4) determinism: repeated calls, uneven splits, poisoned workspaces; (5) a
whole 1080 x 1920 frame at S = 512 in one call."""
import os

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
from test_gpu_parity import cuda

pytestmark = pytest.mark.gpu

EPS = 1e-6   # NNB_EPS


@pytest.fixture(autouse=True)
def _keep_default_engine(monkeypatch):
    from nope_nerf_b200 import ops
    monkeypatch.setattr(ops, "_DEFAULT_ENGINE", list(ops._DEFAULT_ENGINE))


def _flat(D, seed=7):
    return cuda(O.flatten_params(O.init_params(seed=seed, D=D, hf_damp=True)))


def _scene(N, H=1080, W=1920, order="random", seed=0):
    """c2w, cam and N ray ids of an H x W frame: 'random' distinct pixels, 'block' a row block, 'perm' a permuted row block"""
    rng = np.random.default_rng(seed)
    c2w = cuda(O.make_c2w(np.array([0.02, -0.03, 0.01], np.float32), np.array([0.05, 0.0, -0.04], np.float32)))
    cam = torch.diag(torch.tensor([1.2, -2.1, -1.0, 1.0])).cuda()
    if order == "random":
        idx = rng.permutation(H * W)[:N]
    else:
        idx = np.arange(531 * W, 531 * W + N)
        if order == "perm":
            idx = rng.permutation(idx)
    return c2w, cam, cuda(idx.astype(np.int64))


def _kw(cfg_over=None, occ="softplus", D=256, S=128, N=1000, H=1080, W=1920, ray_idx=None, eval_=True):
    from nope_nerf_b200 import ops
    cfg = dict(O.DEFAULT_CFG); cfg.update(cfg_over or {})
    ndc = cfg["sample_option"] == "ndc"
    return dict(N=N, S=S, flags=ops.flags_from_cfg(cfg, occ, eval_=eval_), engine=None, near=0.0 if ndc else 0.01, far=1.0 if ndc else 10.0,
                ray_idx=ray_idx, depth_map=cuda(np.random.default_rng(3).uniform(0.6, 7.2, (48, 64)).astype(np.float32)),
                scale=torch.tensor([1.05]).cuda(), shift=torch.tensor([0.02]).cuda(), H=H, W=W, hidden_dim=D)


def _render_fwd(flat, c2w, cam, **kw):
    from nope_nerf_b200 import ops, _lib as L
    call = ops.RenderCall(flat, c2w, cam, stash=False, **dict(kw, engine=L.ENGINE_TC))
    assert call.args.engine == L.ENGINE_TC
    return call.rgb, call.depth_pred, call.depth_gt, call.mask


def _frame(flat, c2w, cam, t_min=0.0, want_stats=False, **kw):
    from nope_nerf_b200 import ops
    return ops.render_frame(flat, c2w, cam, t_min=t_min, want_stats=want_stats, **kw)


def _assert_same(a, b, what):
    for name, x, y in zip(("rgb", "depth_pred", "depth_gt", "mask"), a, b):
        assert x.shape == y.shape and torch.equal(x, y), (what, name, float((x.double() - y.double()).abs().max()))


OPTIONS = {
    "uniform": ({}, "softplus"),
    "ndc": ({"sample_option": "ndc"}, "softplus"),
    "dist_alpha": ({"dist_alpha": True}, "softplus"),
    "white_background": ({"white_background": True}, "softplus"),
    "no_ray_dir": ({"use_ray_dir": False}, "softplus"),
    "no_normalise": ({"normalise_ray": False}, "softplus"),
    "relu": ({}, "relu"),
    "relu_dist_alpha_ndc": ({"dist_alpha": True, "sample_option": "ndc"}, "relu"),
}


@pytest.mark.parametrize("opt", sorted(OPTIONS))
@pytest.mark.parametrize("eval_", [True, False])
def test_bit_equal_options(opt, eval_):
    over, occ = OPTIONS[opt]
    flat = _flat(256)
    c2w, cam, idx = _scene(1001)
    kw = _kw(over, occ, N=1001, ray_idx=idx, eval_=eval_)
    _assert_same(_frame(flat, c2w, cam, **kw), _render_fwd(flat, c2w, cam, **kw), opt)


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("S", [16, 17, 21, 32, 33, 100, 128, 200, 512])
def test_bit_equal_widths_and_sample_counts(D, S):
    flat = _flat(D)
    for N, order in ((1003, "random"), (517, "block"), (998, "perm")):
        c2w, cam, idx = _scene(N, order=order, seed=S)
        kw = _kw({"dist_alpha": S % 2 == 1}, D=D, S=S, N=N, ray_idx=idx)
        _assert_same(_frame(flat, c2w, cam, **kw), _render_fwd(flat, c2w, cam, **kw), (D, S, N, order))


def _extract(D=256, S=128, H=1080, W=1920, t_min=None, seed=7):
    import nope_nerf_b200.model as mdl
    from _cfg import default_cfg
    cfg = default_cfg(); cfg["rendering"]["num_points"] = S; cfg["extract_images"] = {"resolution": (H, W)}; cfg["model"]["hidden_dim"] = D
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=seed, D=D, hf_damp=True).items()})
    dev = torch.device("cuda")
    return mdl.Extract_Images(mdl.Renderer(net, cfg["rendering"], device=dev, frame_t_min=t_min), cfg, device=dev, render_type="nope_nerf")


def _pose():
    c2w = cuda(O.make_c2w(np.array([0.02, -0.03, 0.01], np.float32), np.array([0.05, 0.0, -0.04], np.float32)))
    return c2w, torch.diag(torch.tensor([1.2, -2.1, -1.0, 1.0])).cuda()


def test_whole_1080p_frame_s128_equals_row_blocks():
    """a whole 1080 x 1920 frame at S = 128 in one nnb_render_frame call against Extract_Images.render_frame's nnb_render_fwd in row blocks"""
    H, W = 1080, 1920
    c2w, cam = _pose()
    ex0, ex1 = _extract(), _extract(t_min=0.0)
    rgb1, dep1 = ex1.render_frame(c2w, cam, H, W)
    torch.cuda.synchronize()
    for r0, r1 in ((0, 270), (270, 541), (541, 1000), (1000, 1080)):
        rgb0, dep0 = ex0.render_frame(c2w, cam, H, W, rows=(r0, r1))
        assert torch.equal(rgb0, rgb1[r0:r1]) and torch.equal(dep0, dep1[r0:r1]), (r0, r1)


def test_large_s_whole_frame_in_its_workspace():
    """a whole 1080 x 1920 frame at S = 512 in one call (1.36 GB of workspace; nnb_render_fwd would need 34 GB), rows 531..548 against the
    existing row-block render"""
    from nope_nerf_b200 import _lib as L, ops
    H, W, S = 1080, 1920, 512
    c2w, cam = _pose()
    need = L.lib.nnb_render_frame_workspace_bytes(H * W, S, 256)
    assert need < 1.4e9
    taken = []
    real_take = ops._pool.take
    ops._pool.take = lambda n, dev: taken.append(n) or real_take(n, dev)
    try:
        rgb1, dep1 = _extract(S=S, t_min=0.0).render_frame(c2w, cam, H, W)
    finally:
        ops._pool.take = real_take
    assert taken == [need]
    rgb0, dep0 = _extract(S=S).render_frame(c2w, cam, H, W, rows=(531, 549))
    assert torch.equal(rgb0, rgb1[531:549]) and torch.equal(dep0, dep1[531:549])


def test_eval_images_and_generate_images_at_t0(tmp_path):
    """Eval_Images.eval_images and Extract_Images.generate_images with frame_t_min = 0: the same frame, depth, MSE, PSNR and SSIM as the
    default path, which is checked against the stored reference results (tests/golden/fullsize_eval_images.npz) as in
    test_gpu_fullsize_ref.test_eval_images_vs_live_reference"""
    import nope_nerf_b200.model as mdl
    import _fullsize_cases as FC
    from test_gpu_fullsize_ref import _golden, _ours
    from nope_nerf_b200 import ops
    ops.set_default_engine("tc")
    H, W, V = 48, 64, 4
    cfg = FC.default_cfg()
    cfg["extract_images"] = {"resolution": [H, W]}
    state = FC.start_state(cfg, V, 21, 97)
    gold = _golden("eval_images", state)
    data = FC.small_scene(H, W, V=V)
    lp = lambda a, b, normalize=True: (a - b).abs().mean()
    res = {}
    for name, t_min in (("default", None), ("frame", 0.0)):
        trainer, net, pose, dist, model = _ours(cfg, V, state)
        model.renderer.frame_t_min = t_min
        c2ws = torch.stack([pose(i) for i in range(V)]).detach()
        ev = mdl.Eval_Images(model.renderer, cfg, use_learnt_poses=True, use_learnt_focal=False, device=torch.device("cuda"),
                             render_type="nope_nerf", c2ws=c2ws)
        d = ev.eval_images(data, str(tmp_path / name), None, lp, None)
        ex = mdl.Extract_Images(model.renderer, cfg, use_learnt_poses=True, use_learnt_focal=False, device=torch.device("cuda"))
        g = ex.generate_images(data, str(tmp_path / ("gen_" + name)), c2ws, None, 0, False)
        res[name] = (d, g)
    (d0, g0), (d1, g1) = res["default"], res["frame"]
    for k in ("mse", "psnr", "ssim"):
        assert float(d0[k]) == float(d1[k]), k
    assert np.array_equal(d0["img"], d1["img"]) and np.array_equal(d0["depth"], d1["depth"])
    assert np.array_equal(g0["img"], g1["img"]) and np.array_equal(g0["depth"], g1["depth"])
    assert np.array_equal(np.load(str(tmp_path / "gen_default" / "depth_out" / "1.npy")), np.load(str(tmp_path / "gen_frame" / "depth_out" / "1.npy")))
    assert abs(d1["mse"] - float(gold["mse"])) / float(gold["mse"]) < 1e-4 and abs(d1["psnr"] - float(gold["psnr"])) < 1e-3
    assert abs(d1["ssim"] - float(gold["ssim"])) < 1e-5
    assert float(np.abs(d1["img"].astype(np.int32) - gold["img"].astype(np.int32)).max()) <= 1


def _surface_case(D, white_bg=False):
    """the seeded geometry field of the tests (density logits x 10: opaque surfaces inside the sphere) seen from view 1 of the small scene"""
    import sys
    from _util import ROOT
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from geometry_normals_cost import geometry_net
    import nope_nerf_b200.model as mdl
    net, cfg, state = geometry_net(D)
    pose = mdl.LearnPose(4, True, True, cfg).cuda()
    with torch.no_grad():
        pose.r.copy_(state["r"]); pose.t.copy_(state["t"])
        c2w = pose(1).detach().contiguous()
    H, W = 120, 160
    cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0])).cuda()
    from nope_nerf_b200 import ops
    rc = dict(cfg["rendering"]); rc["white_background"] = white_bg
    kw = dict(N=H * W, S=128, flags=ops.flags_from_cfg(rc, "softplus", eval_=True), engine=None, near=0.01, far=10.0,
              ray_idx=torch.arange(H * W, device="cuda"), depth_map=torch.ones(1, 1, device="cuda"), H=H, W=W, hidden_dim=D)
    return net.flat_weights(), c2w, cam, kw


@pytest.mark.parametrize("D", [64, 256])
@pytest.mark.parametrize("white_bg", [False, True])
def test_early_termination_bound(D, white_bg):
    flat, c2w, cam, kw = _surface_case(D, white_bg)
    S = kw["S"]
    ref = _frame(flat, c2w, cam, t_min=0.0, want_stats=True, **kw)
    assert bool((ref[4] == S).all())
    _assert_same(ref[:4], _render_fwd(flat, c2w, cam, **kw), "t_min = 0")
    shares = {}
    for t_min in (1e-4, 1e-3):
        out = _frame(flat, c2w, cam, t_min=t_min, want_stats=True, **kw)
        n_eval, t_final = out[4], out[5]
        full = n_eval == S
        stopped = ~full
        shares[t_min] = float(stopped.float().mean())
        assert bool(((n_eval % 32 == 0) | full).all()) and bool((n_eval > 0).all())
        assert bool((t_final[stopped] < t_min).all())
        for k in range(4):   # a ray that was not stopped has the bits of the t_min = 0 call
            assert torch.equal(out[k][full], ref[k][full]), (t_min, k)
        assert torch.equal(out[2], ref[2]) and torch.equal(out[3], ref[3])
        bound = t_final[stopped].double() * (1 + EPS * S * (1 + EPS) ** S)
        slack = 1.01 * bound + 4 * np.finfo(np.float32).eps
        d_rgb = (out[0][stopped].double() - ref[0][stopped].double()).abs().max(1).values
        assert bool((d_rgb <= (2 if white_bg else 1) * slack).all()), float((d_rgb / slack).max())
        d_dep = (out[1][stopped].double() - ref[1][stopped].double()).abs()
        assert bool((d_dep <= kw["far"] * slack + 4 * np.finfo(np.float32).eps * kw["far"]).all())
    assert shares[1e-3] > 0 and shares[1e-3] >= shares[1e-4], shares


def test_determinism_splits_and_poisoned_workspaces():
    from nope_nerf_b200 import ops, _lib as L
    flat, c2w, cam, kw = _surface_case(128)
    N = kw["N"]
    for t_min in (0.0, 1e-3):
        a = _frame(flat, c2w, cam, t_min=t_min, want_stats=True, **kw)
        b = _frame(flat, c2w, cam, t_min=t_min, want_stats=True, **kw)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        # uneven blocks of the same rays, and a permutation
        cuts = [0, 1, 5, 4000, 4001, 11111, N]
        parts = [_frame(flat, c2w, cam, t_min=t_min, want_stats=True, **dict(kw, N=e - s, ray_idx=kw["ray_idx"][s:e]))
                 for s, e in zip(cuts[:-1], cuts[1:])]
        for k in range(6):
            assert torch.equal(torch.cat([p[k] for p in parts]), a[k]), k
        perm = torch.randperm(N, generator=torch.Generator().manual_seed(5)).cuda()
        c = _frame(flat, c2w, cam, t_min=t_min, want_stats=True, **dict(kw, ray_idx=kw["ray_idx"][perm]))
        for k in range(6):
            assert torch.equal(c[k], a[k][perm]), k
        # workspaces filled with zeros, NaN bytes and large finite words
        need = L.lib.nnb_render_frame_workspace_bytes(N, kw["S"], kw["hidden_dim"])
        real_take = ops._pool.take
        outs = []
        for fill in (0x00, 0xFF, 0x7E):
            ws = torch.full((need,), fill, dtype=torch.uint8, device="cuda")
            ops._pool.take = lambda n, dev: ws
            try:
                outs.append(_frame(flat, c2w, cam, t_min=t_min, want_stats=True, **kw))
            finally:
                ops._pool.take = real_take
        for o in outs:
            for k in range(6):
                assert torch.equal(o[k], a[k]), k


def test_simt_engine_and_small_s_keep_the_old_path():
    """Renderer(frame_t_min=...) with the SIMT engine (explicit, or S < 16) renders through nnb_render_fwd, as without the option"""
    from nope_nerf_b200 import ops, _lib as L
    H, W = 30, 40
    c2w, cam = _pose()
    for S, eng in ((128, L.ENGINE_SIMT), (8, None)):
        ex0, ex1 = _extract(S=S, H=H, W=W), _extract(S=S, H=H, W=W, t_min=1e-2)
        ex0.renderer.engine = eng; ex1.renderer.engine = eng
        a, b = ex0.render_frame(c2w, cam, H, W), ex1.render_frame(c2w, cam, H, W)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    with pytest.raises(RuntimeError, match="nnb_render_frame"):
        _frame(_flat(256), c2w, cam, **dict(_kw(N=10, ray_idx=torch.arange(10, device="cuda")), engine=L.ENGINE_SIMT))

"""GPU: nnb_render_frame_engine on the exact-fp32 engine (ops.render_frame_engine(engine=ENGINE_SIMT), Renderer(frame_engine='simt')): the
volumetric frame with compositing fused into the exact forward, at any S from 2 to 1024.
(1) bit equality with nnb_render_fwd on the exact engine (RenderCall(engine=ENGINE_SIMT, stash=False)) at t_min = 0 over the rendering
options, every width, sample counts below, at and above one 32-sample chunk, ragged / row-block / permuted rays and a whole 1080 x 1920
frame; (2) t_min > 0 on a field with surfaces: unstopped rays exact, stopped rays within the header's bound; (3) determinism: repeated
calls, uneven splits, a permutation, poisoned workspaces; (4) Eval_Images and Extract_Images against Renderer(engine=ENGINE_SIMT) and the
stored reference results; (5) a workspace that does not grow with S."""
import numpy as np
import pytest
import torch

from test_gpu_render_frame import EPS, OPTIONS, _assert_same, _flat, _kw, _pose, _scene, _surface_case

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _release_workspaces():
    """the library's workspace pool keeps every size it has handed out; drop the ones this module added (a 1080p frame and 3.8 GB row
    blocks among them), so that the memory is free for the modules that run after it"""
    from nope_nerf_b200 import ops
    before = {k: len(v) for k, v in ops._pool.free.items()}
    yield
    for k in list(ops._pool.free):
        del ops._pool.free[k][before.get(k, 0):]
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _keep_default_engine(monkeypatch):
    from nope_nerf_b200 import ops
    monkeypatch.setattr(ops, "_DEFAULT_ENGINE", list(ops._DEFAULT_ENGINE))


def _render_fwd(flat, c2w, cam, **kw):
    from nope_nerf_b200 import ops, _lib as L
    call = ops.RenderCall(flat, c2w, cam, stash=False, **dict(kw, engine=L.ENGINE_SIMT))
    assert call.args.engine == L.ENGINE_SIMT
    return call.rgb, call.depth_pred, call.depth_gt, call.mask


def _frame(flat, c2w, cam, t_min=0.0, want_stats=False, **kw):
    from nope_nerf_b200 import ops, _lib as L
    return ops.render_frame_engine(flat, c2w, cam, t_min=t_min, want_stats=want_stats, **dict(kw, engine=L.ENGINE_SIMT))


@pytest.mark.parametrize("opt", sorted(OPTIONS))
@pytest.mark.parametrize("eval_", [True, False])
def test_bit_equal_options(opt, eval_):
    over, occ = OPTIONS[opt]
    flat = _flat(256)
    c2w, cam, idx = _scene(1001)
    kw = _kw(over, occ, N=1001, ray_idx=idx, eval_=eval_)
    _assert_same(_frame(flat, c2w, cam, **kw), _render_fwd(flat, c2w, cam, **kw), opt)


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("S", [2, 3, 8, 15, 16, 17, 31, 32, 33, 100, 128, 200, 512])
def test_bit_equal_widths_and_sample_counts(D, S):
    flat = _flat(D)
    for N, order in ((1003, "random"), (517, "block"), (998, "perm")):
        c2w, cam, idx = _scene(N, order=order, seed=S)
        kw = _kw({"dist_alpha": S % 2 == 1}, D=D, S=S, N=N, ray_idx=idx)
        out = _frame(flat, c2w, cam, want_stats=True, **kw)
        _assert_same(out[:4], _render_fwd(flat, c2w, cam, **kw), (D, S, N, order))
        assert bool((out[4] == S).all())


@pytest.mark.parametrize("D", [64, 256])
@pytest.mark.parametrize("S", [100, 128])
@pytest.mark.parametrize("white_bg", [False, True])
def test_early_termination_bound(D, S, white_bg):
    flat, c2w, cam, kw = _surface_case(D, white_bg)
    kw = dict(kw, S=S)
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
        assert bool(((n_eval % 32 == 0) | full).all()) and bool((n_eval > 0).all())   # R = 32 at these S
        assert bool((t_final[stopped] < t_min).all())
        for k in range(4):   # a ray that was not stopped has the bits of the t_min = 0 call
            assert torch.equal(out[k][full], ref[k][full]), (t_min, k)
        assert torch.equal(out[2], ref[2]) and torch.equal(out[3], ref[3])
        bound = t_final[stopped].double() * (1 + EPS * S * (1 + EPS) ** S)   # the header's bound, from each ray's own t_final
        slack = 1.01 * bound + 4 * np.finfo(np.float32).eps
        d_rgb = (out[0][stopped].double() - ref[0][stopped].double()).abs().max(1).values
        assert bool((d_rgb <= (2 if white_bg else 1) * slack).all()), float((d_rgb / slack).max())
        d_dep = (out[1][stopped].double() - ref[1][stopped].double()).abs()
        assert bool((d_dep <= kw["far"] * slack + 4 * np.finfo(np.float32).eps * kw["far"]).all())
    assert shares[1e-3] > 0 and shares[1e-3] >= shares[1e-4], shares


def test_small_s_rays_stop_after_their_only_chunk():
    """below 32 samples a ray is one ray-chunk of R = S rows: n_eval == S and the bits of t_min = 0 at any t_min"""
    flat, c2w, cam, kw = _surface_case(128)
    for S in (2, 13, 31):
        kw_s = dict(kw, S=S)
        ref = _frame(flat, c2w, cam, t_min=0.0, want_stats=True, **kw_s)
        _assert_same(ref[:4], _render_fwd(flat, c2w, cam, **kw_s), S)
        out = _frame(flat, c2w, cam, t_min=1e-3, want_stats=True, **kw_s)
        assert bool((out[4] == S).all())
        for k in range(6):
            assert torch.equal(out[k], ref[k]), (S, k)


@pytest.mark.parametrize("S", [13, 128])
def test_determinism_splits_and_poisoned_workspaces(S):
    from nope_nerf_b200 import ops, _lib as L
    flat, c2w, cam, kw = _surface_case(128)
    kw = dict(kw, S=S)
    N = kw["N"]
    for t_min in (0.0, 1e-3):
        a = _frame(flat, c2w, cam, t_min=t_min, want_stats=True, **kw)
        b = _frame(flat, c2w, cam, t_min=t_min, want_stats=True, **kw)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        for cuts in ([0, 1, 5, 4000, 4001, 11111, N], [0, 7, N - 3, N], [0, 9600, N]):   # uneven blocks of the same rays
            parts = [_frame(flat, c2w, cam, t_min=t_min, want_stats=True, **dict(kw, N=e - s, ray_idx=kw["ray_idx"][s:e]))
                     for s, e in zip(cuts[:-1], cuts[1:])]
            for k in range(6):
                assert torch.equal(torch.cat([p[k] for p in parts]), a[k]), (cuts, k)
        perm = torch.randperm(N, generator=torch.Generator().manual_seed(5)).cuda()
        c = _frame(flat, c2w, cam, t_min=t_min, want_stats=True, **dict(kw, ray_idx=kw["ray_idx"][perm]))
        for k in range(6):
            assert torch.equal(c[k], a[k][perm]), k
        # workspaces filled with zeros, NaN bytes and large finite words
        need = L.lib.nnb_render_frame_workspace_bytes_engine(N, S, kw["hidden_dim"], L.ENGINE_SIMT)
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


def _extract(D=256, S=128, H=1080, W=1920, engine=None, t_min=None, frame_engine=None, seed=7):
    import nope_nerf_b200.model as mdl
    from _cfg import default_cfg
    from oracle import nerf_oracle as O
    cfg = default_cfg(); cfg["rendering"]["num_points"] = S; cfg["extract_images"] = {"resolution": (H, W)}; cfg["model"]["hidden_dim"] = D
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=seed, D=D, hf_damp=True).items()})
    dev = torch.device("cuda")
    rend = mdl.Renderer(net, cfg["rendering"], device=dev, engine=engine, frame_t_min=t_min, frame_engine=frame_engine)
    return mdl.Extract_Images(rend, cfg, device=dev, render_type="nope_nerf")


def test_whole_1080p_frame_s512_equals_row_blocks():
    """a whole 1080 x 1920 frame at D = 64, S = 512 in one exact-frame call (1.36 GB of workspace; nnb_render_fwd would need 34 GB) against
    RenderCall on the exact engine in row blocks of 120 rows"""
    from nope_nerf_b200 import _lib as L, ops
    H, W, S, D = 1080, 1920, 512, 64
    c2w, cam = _pose()
    need = L.lib.nnb_render_frame_workspace_bytes_engine(H * W, S, D, L.ENGINE_SIMT)
    assert need < 1.4e9
    taken = []
    real_take = ops._pool.take
    ops._pool.take = lambda n, dev: taken.append(n) or real_take(n, dev)
    try:
        rgb1, dep1 = _extract(D=D, S=S, t_min=0.0, frame_engine="simt").render_frame(c2w, cam, H, W)
    finally:
        ops._pool.take = real_take
    assert taken == [need]
    ex0 = _extract(D=D, S=S, engine=L.ENGINE_SIMT)
    for r0 in range(0, H, 120):
        rgb0, dep0 = ex0.render_frame(c2w, cam, H, W, rows=(r0, r0 + 120))
        assert torch.equal(rgb0, rgb1[r0:r0 + 120]) and torch.equal(dep0, dep1[r0:r0 + 120]), r0


def test_small_s_frame_engine_gives_the_default_bits():
    """at S = 8 the default path already runs on the exact engine (nnb_render_fwd); frame_engine='simt' gives its bits"""
    H, W = 30, 40
    c2w, cam = _pose()
    for D in (64, 256):
        a = _extract(D=D, S=8, H=H, W=W).render_frame(c2w, cam, H, W)
        b = _extract(D=D, S=8, H=H, W=W, t_min=0.0, frame_engine="simt").render_frame(c2w, cam, H, W)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), D


def test_eval_images_and_generate_images_at_t0(tmp_path):
    """Eval_Images.eval_images and Extract_Images.generate_images with Renderer(frame_t_min=0, frame_engine='simt'): the same frame, depth,
    MSE, PSNR and SSIM as Renderer(engine=ENGINE_SIMT) without the option, and the stored reference results
    (tests/golden/fullsize_eval_images.npz) at the tolerance test_gpu_render_frame uses for the tensor-core frame"""
    import nope_nerf_b200.model as mdl
    import _fullsize_cases as FC
    from test_gpu_fullsize_ref import _golden, _ours
    from nope_nerf_b200 import _lib as L
    H, W, V = 48, 64, 4
    cfg = FC.default_cfg()
    cfg["extract_images"] = {"resolution": [H, W]}
    state = FC.start_state(cfg, V, 21, 97)
    gold = _golden("eval_images", state)
    data = FC.small_scene(H, W, V=V)
    lp = lambda a, b, normalize=True: (a - b).abs().mean()
    res = {}
    for name in ("simt", "frame"):
        trainer, net, pose, dist, model = _ours(cfg, V, state)
        if name == "simt":
            model.renderer.engine = L.ENGINE_SIMT
        else:
            model.renderer.frame_t_min = 0.0; model.renderer.frame_engine = "simt"
        c2ws = torch.stack([pose(i) for i in range(V)]).detach()
        ev = mdl.Eval_Images(model.renderer, cfg, use_learnt_poses=True, use_learnt_focal=False, device=torch.device("cuda"),
                             render_type="nope_nerf", c2ws=c2ws)
        d = ev.eval_images(data, str(tmp_path / name), None, lp, None)
        ex = mdl.Extract_Images(model.renderer, cfg, use_learnt_poses=True, use_learnt_focal=False, device=torch.device("cuda"))
        g = ex.generate_images(data, str(tmp_path / ("gen_" + name)), c2ws, None, 0, False)
        res[name] = (d, g)
    (d0, g0), (d1, g1) = res["simt"], res["frame"]
    for k in ("mse", "psnr", "ssim"):
        assert float(d0[k]) == float(d1[k]), k
    assert np.array_equal(d0["img"], d1["img"]) and np.array_equal(d0["depth"], d1["depth"])
    assert np.array_equal(g0["img"], g1["img"]) and np.array_equal(g0["depth"], g1["depth"])
    assert np.array_equal(np.load(str(tmp_path / "gen_simt" / "depth_out" / "1.npy")), np.load(str(tmp_path / "gen_frame" / "depth_out" / "1.npy")))
    assert abs(d1["mse"] - float(gold["mse"])) / float(gold["mse"]) < 1e-4 and abs(d1["psnr"] - float(gold["psnr"])) < 1e-3
    assert abs(d1["ssim"] - float(gold["ssim"])) < 1e-5
    assert float(np.abs(d1["img"].astype(np.int32) - gold["img"].astype(np.int32)).max()) <= 1


def test_workspace_does_not_grow_with_s():
    from nope_nerf_b200 import _lib as L
    for N in (1, 1000, 1080 * 1920):
        for D in L.HIDDEN_DIMS:
            sizes = {L.lib.nnb_render_frame_workspace_bytes_engine(N, S, D, L.ENGINE_SIMT) for S in (2, 8, 31, 32, 33, 128, 512, 1024)}
            assert len(sizes) == 1 and sizes.pop() > 0, (N, D)

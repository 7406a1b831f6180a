"""GPU: the differentiable frame on the exact-fp32 engine (nnb_render_frame_bwd_engine, nnb_render_frame_train_fwd_engine / _bwd_engine
on NNB_ENGINE_SIMT; ops.ExactFrameRenderCall, ops.render_frame_bwd / render_frame_grad with the exact engine, Trainer and Renderer with
frame_grad_engine='simt').
(1) the forward equals nnb_render_fwd on the exact engine bit for bit, with and without noise, over both density heads, NDC and uniform
sampling, dist_alpha, white_background, eval, D = 64, 128 and 256, S = 2 ... 1024 and ragged N; (2) at S <= 32 (one chunk) the gradients
equal nnb_render_fwd (NNB_STASH) + nnb_render_bwd on the exact engine bit for bit; (3) at S > 32 they agree to 1e-4 of each tensor's
maximum; (4) without noise the pair equals the one-call backward bit for bit; (5) repeated pairs, workspaces filled with 0x00, 0xFF and
0x7E, two interleaved pairs and a graph-captured pair give the same bits; (6) the _engine calls on the tensor-core engine equal the calls
without the suffix bit for bit; (7) a call at N = 4096, S = 1024, D = 256 runs in 1/30 of the stash path's workspace; (8) Trainer(frame_grad
=True, frame_grad_engine='simt'): step 1's losses equal the default exact path's, graph replay equals the eager step body bit for bit, a
step at S = 8 runs, and the stored reference Trainer results meet the default path's tolerances; (9) Renderer(frame_grad=True,
frame_grad_engine='simt').nope_nerf against the default exact path."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
from test_gpu_parity import cuda
from test_gpu_render_frame_grad import _case, _rel, OPTS
import test_gpu_graph_options as GO
import test_gpu_parity as GP
import test_gpu_sample_count as SC

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _keep_default_engine(monkeypatch):
    """tests below switch the process-wide default engine; it is restored after each test"""
    from nope_nerf_b200 import ops
    monkeypatch.setattr(ops, "_DEFAULT_ENGINE", list(ops._DEFAULT_ENGINE))


@pytest.fixture(scope="module", autouse=True)
def _release_pool():
    """the workspaces this module adds to the library's pool (up to a few GB each) are dropped when it finishes"""
    yield
    from nope_nerf_b200 import ops
    ops._pool.free.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _noise(kw, seed):
    return cuda(np.random.default_rng(seed).uniform(0, 1, (kw["N"], kw["S"])).astype(np.float32))


def _grads(D):
    from nope_nerf_b200 import _lib as L
    return (torch.zeros(L.num_params(D), device="cuda"), torch.zeros(4, 4, device="cuda"), torch.zeros(4, 4, device="cuda"),
            torch.zeros(2, device="cuda"))


def _with_depth(kw, seed):
    kw = dict(kw); kw.pop("depth_map")
    kw["depth"] = cuda(np.random.default_rng(seed).uniform(0.6, 7.2, kw["N"]).astype(np.float32))
    return kw


def _run(cls, flat, c2w, cam, kw, gs, noise=None, engine=None):
    """cls (a RenderCall class) forward + backward: (rgb, depth_pred, depth_gt, mask), (g_weights, g_c2w, g_cam, g_scale_shift[, g_depth])"""
    from nope_nerf_b200 import ops, _lib as L
    extra = dict(stash=True, engine=L.ENGINE_SIMT if engine is None else engine) if cls is ops.RenderCall else dict(engine=engine)
    call = cls(flat, c2w, cam, noise=noise, **extra, **kw)
    outs = tuple(t.clone() for t in (call.rgb, call.depth_pred, call.depth_gt, call.mask))
    g_w, g_c, g_k, g_ss = _grads(kw["hidden_dim"])
    g_d = torch.empty(kw["N"], device="cuda") if kw.get("depth") is not None else None
    call.backward(*gs, g_w, g_c, g_k, g_d, g_ss)
    return outs, (g_w, g_c, g_k, g_ss) + ((g_d,) if g_d is not None else ())


def _pair(*a, **k):
    from nope_nerf_b200 import ops
    return _run(ops.ExactFrameRenderCall, *a, **k)


def _stash(*a, **k):
    from nope_nerf_b200 import ops
    return _run(ops.RenderCall, *a, **k)


def _one_call(flat, c2w, cam, kw, gs, engine=None):
    from nope_nerf_b200 import ops, _lib as L
    g_w, g_c, g_k, g_ss = _grads(kw["hidden_dim"])
    g_d = torch.empty(kw["N"], device="cuda") if kw.get("depth") is not None else None
    outs = ops.render_frame_bwd(flat, c2w, cam, *gs, g_w, g_c, g_k, g_d, g_ss, engine=L.ENGINE_SIMT if engine is None else engine, **kw)
    return outs, (g_w, g_c, g_k, g_ss) + ((g_d,) if g_d is not None else ())


def _bits(res):
    outs, grads = res
    return [t.clone() for t in tuple(outs) + tuple(grads)]


def _assert_equal(got, ref, what=""):
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(_bits(got), _bits(ref))):
        assert torch.equal(x, y), (what, i, float((x.double() - y.double()).abs().max()))


# ---- (1) forward bits ---------------------------------------------------------------------------------------------------------
def _fwd_bits(flat, c2w, cam, kw, noise):
    from nope_nerf_b200 import ops, _lib as L
    ref = ops.RenderCall(flat, c2w, cam, engine=L.ENGINE_SIMT, stash=False, noise=noise, **kw)
    got = ops.ExactFrameRenderCall(flat, c2w, cam, engine=L.ENGINE_TC, noise=noise, **kw)   # the engine argument is ignored
    got.release()
    torch.cuda.synchronize()
    for name in ("rgb", "depth_pred", "depth_gt", "mask"):
        assert torch.equal(getattr(got, name), getattr(ref, name)), name


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("opt", range(len(OPTS)))
@pytest.mark.parametrize("occ", ["softplus", "relu"])
def test_forward_bits_over_options(opt, occ, noise):
    flat, c2w, cam, kw, _ = _case(301, 48, 128, OPTS[opt], occ=occ, seed=opt)
    _fwd_bits(flat, c2w, cam, kw, _noise(kw, opt) if noise else None)


SIZES = [(257, 2), (100, 8), (301, 15), (257, 16), (129, 31), (130, 32), (77, 33), (1000, 48), (129, 128), (130, 512), (37, 1024)]


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("N,S", SIZES)
def test_forward_bits_over_sizes(N, S, D, noise):
    flat, c2w, cam, kw, _ = _case(N, S, D, seed=N + S)
    _fwd_bits(flat, c2w, cam, kw, _noise(kw, S) if noise else None)


def test_forward_bits_eval():
    flat, c2w, cam, kw, _ = _case(200, 24, 256, eval_=True)
    _fwd_bits(flat, c2w, cam, kw, _noise(kw, 1))
    flat, c2w, cam, kw, _ = _case(200, 64, 64, dict(white_background=True), eval_=True)
    _fwd_bits(flat, c2w, cam, kw, None)


# ---- (2) one chunk: the stash path's bits ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("opt", range(len(OPTS)))
@pytest.mark.parametrize("occ", ["softplus", "relu"])
def test_one_chunk_equals_stash_backward_over_options(opt, occ, noise):
    flat, c2w, cam, kw, gs = _case(301, 32, 128, OPTS[opt], occ=occ, seed=40 + opt)
    nz = _noise(kw, opt) if noise else None
    _assert_equal(_pair(flat, c2w, cam, kw, gs, nz), _stash(flat, c2w, cam, kw, gs, nz), (opt, occ, noise))


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("N,S", [(257, 2), (100, 8), (301, 15), (257, 16), (129, 31), (130, 32)])
def test_one_chunk_equals_stash_backward_over_sizes(N, S, D):
    flat, c2w, cam, kw, gs = _case(N, S, D, seed=N + S)
    nz = _noise(kw, S)
    _assert_equal(_pair(flat, c2w, cam, kw, gs, nz), _stash(flat, c2w, cam, kw, gs, nz), (N, S, D))


def test_one_chunk_eval_and_depth_input():
    flat, c2w, cam, kw, gs = _case(200, 24, 256, dict(dist_alpha=True), eval_=True, seed=3)
    _assert_equal(_pair(flat, c2w, cam, kw, gs), _stash(flat, c2w, cam, kw, gs), "eval")
    kw = _with_depth(kw, 4)
    _assert_equal(_pair(flat, c2w, cam, kw, gs, _noise(kw, 4)), _stash(flat, c2w, cam, kw, gs, _noise(kw, 4)), "depth")


# ---- (3) several chunks: within 1e-4 of the stash path ---------------------------------------------------------------------------
def _check_close(case, noise=True):
    from nope_nerf_b200.model.official_nerf import param_slices
    flat, c2w, cam, kw, gs = case
    nz = _noise(kw, kw["N"]) if noise else None
    po, pg = _pair(flat, c2w, cam, kw, gs, nz)
    so, sg = _stash(flat, c2w, cam, kw, gs, nz)
    torch.cuda.synchronize()
    for x, y in zip(po, so):
        assert torch.equal(x, y)
    worst = 0.0
    for (o, n, shape) in param_slices(kw["hidden_dim"]):
        ref = sg[0][o:o + n]
        if ref.abs().max() == 0:
            assert pg[0][o:o + n].abs().max() == 0
            continue
        e = _rel(pg[0][o:o + n], ref)
        worst = max(worst, e)
        assert e < 1e-4, (o, shape, e)
    e_pose = [_rel(pg[i], sg[i]) for i in range(1, len(sg))]
    print("exact frame pair vs exact stash bwd N=%d S=%d D=%d: worst dW %.2e, g_c2w %.2e, g_cam %.2e, g_scale_shift %.2e"
          % (kw["N"], kw["S"], kw["hidden_dim"], worst, *e_pose[:3]))
    assert max(e_pose) < 1e-4, e_pose


@pytest.mark.parametrize("opt", range(len(OPTS)))
@pytest.mark.parametrize("occ", ["softplus", "relu"])
def test_chunks_match_stash_backward_over_options(opt, occ):
    _check_close(_case(300, 48, 128, OPTS[opt], occ=occ, seed=opt))


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("N,S", [(77, 33), (1000, 48), (129, 128), (130, 512), (37, 1024)])
def test_chunks_match_stash_backward_over_sizes(D, N, S):
    _check_close(_case(N, S, D, seed=N + S))


def test_chunks_eval_and_depth_input():
    case = _case(200, 64, 256, eval_=True, seed=6)
    _check_close(case, noise=False)
    flat, c2w, cam, kw, gs = case
    _check_close((flat, c2w, cam, _with_depth(kw, 7), gs))


# ---- (4) the split equals the one-call backward ----------------------------------------------------------------------------------
SPLIT = [(300, 48, 128, 0, "softplus", False), (300, 48, 64, 1, "relu", False), (300, 8, 256, 3, "relu", False),
         (300, 48, 128, 4, "softplus", True), (129, 2, 128, 2, "softplus", True), (37, 1024, 256, 0, "softplus", False)]


@pytest.mark.parametrize("case", range(len(SPLIT)))
def test_split_equals_one_call_backward(case):
    N, S, D, opt, occ, depth_in = SPLIT[case]
    flat, c2w, cam, kw, gs = _case(N, S, D, OPTS[opt], occ=occ, seed=case)
    if depth_in:
        kw = _with_depth(kw, case)
    got = _pair(flat, c2w, cam, kw, gs)
    _assert_equal(got, _one_call(flat, c2w, cam, kw, gs), case)
    assert got[1][0].abs().max() > 0 and got[1][1].abs().max() > 0


# ---- (5) determinism and isolation ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [8, 80])
def test_repeated_and_workspace_independent(S):
    from nope_nerf_b200 import ops, _lib as L
    flat, c2w, cam, kw, gs = _case(500, S, 256, dict(dist_alpha=True), seed=5)
    noise = _noise(kw, 5)
    ref = _pair(flat, c2w, cam, kw, gs, noise)
    for _ in range(2):
        _assert_equal(_pair(flat, c2w, cam, kw, gs, noise), ref, "repeat")
    nbytes = L.lib.nnb_render_frame_bwd_workspace_bytes_engine(kw["N"], kw["S"], 256, L.ENGINE_SIMT)
    for fill in (0x00, 0xFF, 0x7E):
        ops._pool.free.clear()
        ops._pool.give(torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda"))   # the next call takes this workspace
        _assert_equal(_pair(flat, c2w, cam, kw, gs, noise), ref, fill)
        ops._pool.free.clear()
        ops._pool.give(torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda"))
        _assert_equal(_one_call(flat, c2w, cam, kw, gs), _pair(flat, c2w, cam, kw, gs), ("one call", fill))
    ops._pool.free.clear()


def test_interleaved_pairs_on_separate_workspaces():
    from nope_nerf_b200 import ops
    A = _case(400, 96, 128, seed=21); B = _case(250, 12, 128, dict(white_background=True), seed=22)
    nA, nB = _noise(A[3], 21), _noise(B[3], 22)
    solo = [_bits(_pair(*A, nA)), _bits(_pair(*B, nB))]
    calls, outs = [], []
    for (flat, c2w, cam, kw, gs), noise in ((A, nA), (B, nB)):            # fwd A, fwd B
        calls.append(ops.ExactFrameRenderCall(flat, c2w, cam, engine=None, noise=noise, **kw))
    assert calls[0].ws.data_ptr() != calls[1].ws.data_ptr()
    for call, (flat, c2w, cam, kw, gs) in zip(calls, (A, B)):              # bwd A, bwd B
        grads = _grads(kw["hidden_dim"])
        call.backward(*gs, grads[0], grads[1], grads[2], None, grads[3])
        outs.append([t.clone() for t in (call.rgb, call.depth_pred, call.depth_gt, call.mask) + grads])
    torch.cuda.synchronize()
    for got, ref in zip(outs, solo):
        for x, y in zip(got, ref):
            assert torch.equal(x, y)


def test_pair_replayed_from_a_cuda_graph():
    from nope_nerf_b200 import ops
    flat, c2w, cam, kw, gs = _case(300, 160, 128, seed=31)
    noise = _noise(kw, 31)
    ref = _bits(_pair(flat, c2w, cam, kw, gs, noise))                      # eager: also the one-time set-up
    grads = _grads(kw["hidden_dim"])
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for g in grads:
            g.zero_()
        call = ops.ExactFrameRenderCall(flat, c2w, cam, engine=None, noise=noise, **kw)
        call.pooled = False                                                # memory of a captured graph never returns to the pool
        ws = call.ws
        call.backward(*gs, grads[0], grads[1], grads[2], None, grads[3])
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        got = [call.rgb, call.depth_pred, call.depth_gt, call.mask] + list(grads)
        for x, y in zip(got, ref):
            assert torch.equal(x, y)
    del graph, ws


# ---- (6) the tensor-core path is unchanged ---------------------------------------------------------------------------------------
def _tc_pair_direct(flat, c2w, cam, kw, gs, noise, suffix):
    """FrameRenderCall's pair with the C calls named by suffix ('' or '_engine') on the tensor-core engine"""
    from nope_nerf_b200 import ops, _lib as L
    call = ops.FrameRenderCall(flat, c2w, cam, engine=L.ENGINE_TC, noise=noise, **kw)     # runs nnb_render_frame_train_fwd
    if suffix:
        L.check(L.lib.nnb_render_frame_train_fwd_engine(C.byref(call.args), ops._stream()), "train_fwd_engine")
    outs = tuple(t.clone() for t in (call.rgb, call.depth_pred, call.depth_gt, call.mask))
    g = _grads(kw["hidden_dim"])
    b = L.RenderBwdArgs()
    b.fwd = call.args
    keep = [ops._f32c(t) for t in gs]
    b.g_rgb, b.g_depth_pred, b.g_depth_gt = (L.ptr(t) for t in keep)
    b.g_weights, b.g_c2w, b.g_cam, b.g_scale_shift = (L.ptr(t) for t in g)
    fn = L.lib.nnb_render_frame_train_bwd_engine if suffix else L.lib.nnb_render_frame_train_bwd
    L.check(fn(C.byref(b), ops._stream()), "train_bwd" + suffix)
    torch.cuda.synchronize()
    call.release()
    return outs, g


def test_tensor_core_engine_calls_unchanged():
    from nope_nerf_b200 import _lib as L
    for N, S, D, seed in ((300, 48, 128, 1), (129, 16, 64, 2), (37, 1024, 256, 3)):
        flat, c2w, cam, kw, gs = _case(N, S, D, seed=seed)
        assert (L.lib.nnb_render_frame_bwd_workspace_bytes_engine(N, S, D, L.ENGINE_TC)
                == L.lib.nnb_render_frame_bwd_workspace_bytes(N, S, D))
        nz = _noise(kw, seed)
        _assert_equal(_tc_pair_direct(flat, c2w, cam, kw, gs, nz, "_engine"), _tc_pair_direct(flat, c2w, cam, kw, gs, nz, ""), (N, S))
        # one call: ops.render_frame_bwd runs nnb_render_frame_bwd_engine, the pair without noise nnb_render_frame_train_*
        _assert_equal(_one_call(flat, c2w, cam, kw, gs, engine=L.ENGINE_TC), _tc_pair_direct(flat, c2w, cam, kw, gs, None, ""), (N, S))


# ---- (7) memory --------------------------------------------------------------------------------------------------------------------
def test_workspace_and_a_large_call():
    from nope_nerf_b200 import ops, _lib as L
    N = 4096
    ws = lambda S: L.lib.nnb_render_frame_bwd_workspace_bytes_engine(N, S, 256, L.ENGINE_SIMT)
    stash = lambda S: L.lib.nnb_workspace_bytes_dim(N, S, L.STASH, L.ENGINE_SIMT, 256)
    print("exact frame bwd workspace (N=4096, D=256):", {S: ws(S) for S in (8, 16, 32, 128, 512, 1024)},
          "exact stash workspace:", {S: stash(S) for S in (8, 16, 32, 128, 512, 1024)})
    ops._pool.free.clear(); gc.collect(); torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    print("free %.2f GB of %.2f GB; exact stash workspace at S = 1024: %.2f GB" % (free / 1e9, total / 1e9, stash(1024) / 1e9))
    # the stash path's workspace alone takes more than nine tenths of an 80 GB card, the frame's one thirtieth of that
    assert stash(1024) > 0.9 * total and ws(1024) < stash(1024) // 30
    flat, c2w, cam, kw, gs = _case(N, 1024, 256, seed=9)
    outs, grads = _one_call(flat, c2w, cam, kw, gs)
    torch.cuda.synchronize()
    assert all(torch.isfinite(g).all() for g in grads) and grads[0].abs().max() > 0
    ref = ops.render_frame_engine(flat, c2w, cam, engine=L.ENGINE_SIMT, **kw)
    for x, y in zip(outs, ref):
        assert torch.equal(x, y)
    ops._pool.free.clear()


# ---- (8) Trainer -------------------------------------------------------------------------------------------------------------------
FULL = {"full_loss": dict(full=True), "full_loss_focal": dict(full=True, focal=(2, False))}
EXACT = dict(frame_grad=True, frame_grad_engine="simt")


@pytest.mark.parametrize("case", list(FULL))
def test_trainer_graph_replay_equals_eager_bits(case, monkeypatch):
    """the captured step and the same step body launched eagerly give bit-identical losses and parameters over 5 full-loss steps; the
    first step's losses equal those of the default exact path (frame_grad=False), whose forward has the same bits"""
    from nope_nerf_b200 import ops
    ops.set_default_engine("simt")
    opts = FULL[case]
    ge = GO._run(opts, "eager", monkeypatch, steps=5, **EXACT)
    gg = GO._run(opts, "graph", monkeypatch, steps=5, **EXACT)
    assert ge["tr"].frame_grad_engine == "simt" and gg["tr"].frame_grad_engine == "simt"
    assert len(gg["gsteps"]) == 1 and gg["gsteps"][0].graph is not None and gg["gsteps"][0].calls == 5
    assert ge["losses"][:, 4].min() > 0 and ge["losses"][:, 5].min() > 0
    for k in ("losses", "w", "r", "t", "scales", "shifts", "focal"):
        if k in ge:
            assert ge[k].tobytes() == gg[k].tobytes(), (k, np.abs(ge[k] - gg[k]).max())
    fs = GO._run(opts, "graph", monkeypatch, steps=1)
    assert not fs["tr"].frame_grad
    assert gg["losses"][0].tobytes() == fs["losses"][0].tobytes()


def test_trainer_step_below_the_tensor_core_range():
    """a graph step at S = 8 (the tensor-core pair cannot run there) on the exact pair, in its own memory"""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    N, S, H, W, V, hd, wd = 1024, 8, 96, 128, 3, 24, 32
    ops.set_default_engine("tc")
    cfg = default_cfg()
    cfg["rendering"]["num_points"] = S; cfg["training"]["n_training_points"] = N
    dev = torch.device("cuda")
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=9, hf_damp=True).items()})
    model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
    pose = mdl.LearnPose(V, True, True, cfg).to(dev); dist = mdl.Learn_Distortion(V, True, True, cfg).to(dev)
    tr = mdl.Trainer(model, torch.optim.Adam(model.parameters(), lr=1e-3), cfg["training"], device=dev,
                     optimizer_pose=torch.optim.Adam(pose.parameters(), lr=5e-4), pose_param_net=pose,
                     optimizer_distortion=torch.optim.Adam(dist.parameters(), lr=5e-4), distortion_net=dist, use_cuda_graph=True, **EXACT)
    count = {"n": 0}
    base_call = ops.ExactFrameRenderCall

    class CountingCall(base_call):
        def __init__(self, *a, **k):
            count["n"] += 1
            super().__init__(*a, **k)
    ops.ExactFrameRenderCall = CountingCall
    try:
        g = torch.Generator().manual_seed(4)
        cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
        data = {"img": torch.rand(1, 3, H, W, generator=g).cuda(), "img.idx": torch.tensor([1]),
                "img.dpt": (torch.rand(1, hd, wd, generator=g) * 3 + 2).cuda(), "img.camera_mat": cam, "img.scale_mat": torch.eye(4)[None],
                "img.ref_imgs": torch.rand(1, 3, H, W, generator=g).cuda(), "img.ref_dpts": (torch.rand(1, hd, wd, generator=g) * 3 + 2).cuda(),
                "img.ref_idxs": torch.tensor([2])}
        losses = [float(tr.train_step(data, it=it, epoch=0, scheduling_start=10000, render_path=None)["loss"]) for it in range(3)]
    finally:
        ops.ExactFrameRenderCall = base_call
    torch.cuda.synchronize()
    gsteps = [v for v in tr._gsteps.values() if v]
    assert len(gsteps) == 1 and gsteps[0].graph is not None and gsteps[0].calls == 3
    assert count["n"] >= 1
    assert np.isfinite(losses).all() and torch.isfinite(net.flat_weights()).all()


@pytest.fixture
def exact_frame_trainer(monkeypatch):
    """every Trainer built in the test gets frame_grad=True, frame_grad_engine='simt'; counts the renders that ran the exact pair"""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    count = {"frame": 0}
    base, base_call = mdl.Trainer, ops.ExactFrameRenderCall

    class FrameTrainer(base):
        def __init__(self, *a, **k):
            super().__init__(*a, **dict(k, **EXACT))

    class CountingCall(base_call):
        def __init__(self, *a, **k):
            count["frame"] += 1
            super().__init__(*a, **k)
    monkeypatch.setattr(mdl, "Trainer", FrameTrainer)
    monkeypatch.setattr(ops, "ExactFrameRenderCall", CountingCall)
    return count


@pytest.mark.parametrize("name,with_ref", [("train_render_only", False), ("train_full_losses", True)])
def test_parity_golden(name, with_ref, exact_frame_trainer, monkeypatch):
    GP.test_trainer_step_vs_reference_golden(name, with_ref, "simt", monkeypatch)
    assert exact_frame_trainer["frame"] >= 2


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("name,with_ref", SC.TRAIN)
def test_sample_count_golden(name, with_ref, graph, exact_frame_trainer, monkeypatch):
    SC.test_trainer_steps_vs_reference_golden(name, with_ref, "simt", graph, monkeypatch)
    assert exact_frame_trainer["frame"] >= 2


# ---- (9) Renderer ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,sample_option", [(16, "uniform"), (64, "ndc"), (8, "uniform")])
def test_renderer_frame_grad_simt(S, sample_option):
    """Renderer(frame_grad=True, frame_grad_engine='simt').nope_nerf against the default exact path (render_autograd on the exact
    engine): the same outputs, and gradients to the MLP, the pose and the prior depth within 1e-4 of each tensor's maximum"""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops, _lib as L
    from _cfg import default_cfg
    cfg = default_cfg()
    cfg["rendering"]["num_points"] = S; cfg["rendering"]["sample_option"] = sample_option
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=9, hf_damp=True).items()})
    net = net.cuda()
    N, H, W = 700, 240, 320
    gen = torch.Generator().manual_seed(9)
    pix = torch.stack([torch.randint(0, W, (N,), generator=gen), torch.randint(0, H, (N,), generator=gen)], -1).float()
    pix = torch.stack([2 * pix[:, 0] / W - 1, 2 * pix[:, 1] / H - 1], -1).cuda()
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], device="cuda").view(1, 4, 4)
    depth0 = (torch.rand(N, generator=gen) * 2 + 0.5).cuda()
    r0, t0 = (torch.randn(1, 3, generator=gen) * 0.05).cuda(), (torch.randn(1, 3, generator=gen) * 0.05).cuda()
    gC = (torch.randn(1, N, 3, generator=gen)).cuda()
    res = []
    for kw in (dict(engine=L.ENGINE_SIMT), dict(engine=L.ENGINE_TC, frame_grad=True, frame_grad_engine="simt")):
        rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), **kw)
        net.zero_grad(set_to_none=True)
        r, t = r0.clone().requires_grad_(True), t0.clone().requires_grad_(True)
        depth = depth0.clone().requires_grad_(True)
        out = rend.nope_nerf(pix[None], depth, cam, None, None, add_noise=False, it=0, c2w=ops.pose_c2w(r, t, None, 0))
        ((out["rgb"] * gC).sum() + out["depth_pred"].sum() * 0.1).backward()
        grads = [p.grad.clone() for p in net.parameters() if p.grad is not None]
        res.append((out["rgb"].detach(), out["depth_pred"].detach(), grads, r.grad.clone(), t.grad.clone(), depth.grad.clone()))
    (rgb0, dp0, g0, r0g, t0g, d0g), (rgb1, dp1, g1, r1g, t1g, d1g) = res
    assert torch.equal(rgb0, rgb1) and torch.equal(dp0, dp1)
    assert len(g0) == len(g1) and len(g0) > 0
    worst = max((_rel(a, b) for a, b in zip(g1, g0) if b.abs().max() > 0), default=0.0)
    e = dict(dW=worst, r=_rel(r1g, r0g), t=_rel(t1g, t0g), depth=_rel(d1g, d0g))
    print("Renderer frame_grad_engine='simt' vs exact render_autograd S=%d %s:" % (S, sample_option), e)
    assert max(e.values()) < 1e-4, e
    if S <= 32:   # one chunk: the stash path's bits
        assert all(torch.equal(a, b) for a, b in zip(g1, g0)) and torch.equal(d1g, d0g)

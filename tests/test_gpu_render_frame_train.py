"""GPU: nnb_render_frame_train_fwd / nnb_render_frame_train_bwd (FrameRenderCall) and Trainer(frame_grad=True), the
differentiable frame as a forward / backward pair for training, with jitter.
(1) the forward equals nnb_render_fwd on the tensor-core engine bit for bit, with and without noise, over both density heads, NDC and
uniform sampling, dist_alpha, white_background, D = 64, 128 and 256, S = 16 ... 1024 and ragged N; (2) without noise the pair gives
nnb_render_frame_bwd's outputs and gradients bit for bit; (3) with noise its gradients agree with RenderCall(stash=True) + backward to
1e-4 of each tensor's maximum; (4) repeated pairs, workspaces filled with 0x00, 0xFF and 0x7E, two interleaved pairs and the pair
replayed from a CUDA graph give the same bits; (5) Trainer(frame_grad=True): graph replay equals the eager step body bit for bit over 5
full-loss steps, with and without a learned focal, and against frame_grad=False the first step's losses are equal and 5 steps agree
within the gates of graph-vs-eager; (6) the stored reference Trainer results under the default path's tolerances; (7) a graph step at
N = 4096, S = 512, D = 256 in a small part of the stash path's memory."""
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


def _pair(flat, c2w, cam, kw, gs, noise=None):
    """FrameRenderCall + backward: (rgb, depth_pred, depth_gt, mask), (g_weights, g_c2w, g_cam, g_scale_shift[, g_depth])"""
    from nope_nerf_b200 import ops
    call = ops.FrameRenderCall(flat, c2w, cam, engine=None, noise=noise, **kw)
    outs = (call.rgb, call.depth_pred, call.depth_gt, call.mask)
    g_w, g_c, g_k, g_ss = _grads(kw["hidden_dim"])
    g_d = torch.empty(kw["N"], device="cuda") if kw.get("depth") is not None else None
    call.backward(*gs, g_w, g_c, g_k, g_d, g_ss)
    return outs, (g_w, g_c, g_k, g_ss) + ((g_d,) if g_d is not None else ())


def _fwd_bits(flat, c2w, cam, kw, noise):
    from nope_nerf_b200 import ops, _lib as L
    ref = ops.RenderCall(flat, c2w, cam, engine=L.ENGINE_TC, stash=False, noise=noise, **kw)
    got = ops.FrameRenderCall(flat, c2w, cam, engine=None, noise=noise, **kw)
    got.release()
    torch.cuda.synchronize()
    for name in ("rgb", "depth_pred", "depth_gt", "mask"):
        assert torch.equal(getattr(got, name), getattr(ref, name)), name
    return got


# ---- (1) forward bits ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("opt", range(len(OPTS)))
@pytest.mark.parametrize("occ", ["softplus", "relu"])
def test_forward_bits_over_options(opt, occ, noise):
    flat, c2w, cam, kw, _ = _case(301, 48, 128, OPTS[opt], occ=occ, seed=opt)
    got = _fwd_bits(flat, c2w, cam, kw, _noise(kw, opt) if noise else None)
    if noise and OPTS[opt].get("sample_option") == "ndc":      # jitter is ignored under NDC
        plain = _fwd_bits(flat, c2w, cam, kw, None)
        for name in ("rgb", "depth_pred", "depth_gt", "mask"):
            assert torch.equal(getattr(got, name), getattr(plain, name)), name


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("N,S", [(257, 16), (1000, 48), (129, 128), (77, 300), (130, 512), (37, 1024)])
def test_forward_bits_over_sizes(N, S, D, noise):
    flat, c2w, cam, kw, _ = _case(N, S, D, seed=N + S)
    _fwd_bits(flat, c2w, cam, kw, _noise(kw, S) if noise else None)


def test_forward_bits_eval_and_depth_input():
    flat, c2w, cam, kw, _ = _case(200, 64, 256, eval_=True)
    _fwd_bits(flat, c2w, cam, kw, _noise(kw, 1))
    kw = dict(kw); kw.pop("depth_map")
    kw["depth"] = cuda(np.random.default_rng(2).uniform(0.6, 7.2, kw["N"]).astype(np.float32))
    _fwd_bits(flat, c2w, cam, kw, _noise(kw, 3))


# ---- (2) the split equals the one-call backward ----------------------------------------------------------------------------------
def _one_call(flat, c2w, cam, kw, gs):
    from nope_nerf_b200 import ops
    g_w, g_c, g_k, g_ss = _grads(kw["hidden_dim"])
    g_d = torch.empty(kw["N"], device="cuda") if kw.get("depth") is not None else None
    outs = ops.render_frame_bwd(flat, c2w, cam, *gs, g_w, g_c, g_k, g_d, g_ss, **kw)
    return outs, (g_w, g_c, g_k, g_ss) + ((g_d,) if g_d is not None else ())


SPLIT = [(300, 48, 128, 0, "softplus", False), (300, 48, 128, 1, "relu", False), (300, 48, 64, 2, "softplus", False),
         (300, 48, 256, 3, "relu", False), (300, 48, 128, 4, "softplus", False), (129, 128, 256, 0, "softplus", True),
         (130, 512, 64, 0, "softplus", False), (37, 1024, 256, 1, "softplus", False), (257, 16, 128, 0, "softplus", True)]


@pytest.mark.parametrize("case", range(len(SPLIT)))
def test_split_equals_one_call_backward(case):
    N, S, D, opt, occ, depth_in = SPLIT[case]
    flat, c2w, cam, kw, gs = _case(N, S, D, OPTS[opt], occ=occ, seed=case)
    if depth_in:                                              # g_depth through an explicit depth[N]
        kw = dict(kw); kw.pop("depth_map")
        kw["depth"] = cuda(np.random.default_rng(case).uniform(0.6, 7.2, N).astype(np.float32))
    po, pg = _pair(flat, c2w, cam, kw, gs)
    oo, og = _one_call(flat, c2w, cam, kw, gs)
    torch.cuda.synchronize()
    for x, y in zip(po + pg, oo + og):
        assert torch.equal(x, y)
    assert pg[0].abs().max() > 0 and pg[1].abs().max() > 0


# ---- (3) with noise, against the stash path -------------------------------------------------------------------------------------
def _stash(flat, c2w, cam, kw, gs, noise):
    from nope_nerf_b200 import ops, _lib as L
    call = ops.RenderCall(flat, c2w, cam, engine=L.ENGINE_TC, stash=True, noise=noise, **kw)
    outs = (call.rgb, call.depth_pred, call.depth_gt, call.mask)
    g_w, g_c, g_k, g_ss = _grads(kw["hidden_dim"])
    call.backward(*gs, g_w, g_c, g_k, None, g_ss)
    return outs, (g_w, g_c, g_k, g_ss)


NOISY = [(300, 48, 128, 0, "softplus"), (300, 48, 128, 1, "relu"), (300, 48, 128, 2, "softplus"), (300, 48, 128, 3, "softplus"),
         (300, 48, 128, 4, "relu"), (257, 16, 64, 0, "softplus"), (129, 128, 256, 0, "relu"), (77, 300, 128, 1, "softplus"),
         (130, 512, 256, 0, "softplus"), (37, 1024, 64, 0, "softplus")]


@pytest.mark.parametrize("case", range(len(NOISY)))
def test_jittered_pair_matches_stash_backward(case):
    from nope_nerf_b200.model.official_nerf import param_slices
    N, S, D, opt, occ = NOISY[case]
    flat, c2w, cam, kw, gs = _case(N, S, D, OPTS[opt], occ=occ, seed=10 + case)
    noise = _noise(kw, case)
    po, pg = _pair(flat, c2w, cam, kw, gs, noise)
    so, sg = _stash(flat, c2w, cam, kw, gs, noise)
    torch.cuda.synchronize()
    for x, y in zip(po, so):
        assert torch.equal(x, y)
    worst = 0.0
    for (o, n, shape) in param_slices(D):
        ref = sg[0][o:o + n]
        if ref.abs().max() == 0:
            assert pg[0][o:o + n].abs().max() == 0
            continue
        e = _rel(pg[0][o:o + n], ref)
        worst = max(worst, e)
        assert e < 1e-4, (o, shape, e)
    e_pose = [_rel(pg[i], sg[i]) for i in (1, 2, 3)]
    print("train pair (jitter) vs stash bwd N=%d S=%d D=%d: worst dW %.2e, g_c2w %.2e, g_cam %.2e, g_scale_shift %.2e"
          % (N, S, D, worst, *e_pose))
    assert max(e_pose) < 1e-4, e_pose


# ---- (4) determinism and isolation ----------------------------------------------------------------------------------------------
def _flat_bits(res):
    outs, grads = res
    return [t.clone() for t in outs + grads]


def test_repeated_and_workspace_independent():
    from nope_nerf_b200 import ops, _lib as L
    flat, c2w, cam, kw, gs = _case(500, 80, 256, dict(dist_alpha=True), seed=5)
    noise = _noise(kw, 5)
    ref = _flat_bits(_pair(flat, c2w, cam, kw, gs, noise))
    for _ in range(2):
        for x, y in zip(_flat_bits(_pair(flat, c2w, cam, kw, gs, noise)), ref):
            assert torch.equal(x, y)
    nbytes = L.lib.nnb_render_frame_bwd_workspace_bytes(kw["N"], kw["S"], 256)
    for fill in (0x00, 0xFF, 0x7E):
        ops._pool.free.clear()
        ops._pool.give(torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda"))   # the next RenderCall takes this workspace
        for x, y in zip(_flat_bits(_pair(flat, c2w, cam, kw, gs, noise)), ref):
            assert torch.equal(x, y), fill
    ops._pool.free.clear()


def test_interleaved_pairs_on_separate_workspaces():
    from nope_nerf_b200 import ops
    A = _case(400, 96, 128, seed=21); B = _case(250, 96, 128, dict(white_background=True), seed=22)
    nA, nB = _noise(A[3], 21), _noise(B[3], 22)
    solo = [_flat_bits(_pair(*A, nA)), _flat_bits(_pair(*B, nB))]
    calls, outs = [], []
    for (flat, c2w, cam, kw, gs), noise in ((A, nA), (B, nB)):            # fwd A, fwd B
        calls.append(ops.FrameRenderCall(flat, c2w, cam, engine=None, noise=noise, **kw))
    assert calls[0].ws.data_ptr() != calls[1].ws.data_ptr()
    for call, (flat, c2w, cam, kw, gs) in zip(calls, (A, B)):              # bwd A, bwd B
        grads = _grads(kw["hidden_dim"])
        call.backward(*gs, grads[0], grads[1], grads[2], None, grads[3])
        outs.append([t.clone() for t in (call.rgb, call.depth_pred, call.depth_gt, call.mask) + grads])
    for got, ref in zip(outs, solo):
        for x, y in zip(got, ref):
            assert torch.equal(x, y)


def test_pair_replayed_from_a_cuda_graph():
    from nope_nerf_b200 import ops
    flat, c2w, cam, kw, gs = _case(300, 160, 128, seed=31)
    noise = _noise(kw, 31)
    ref = _flat_bits(_pair(flat, c2w, cam, kw, gs, noise))                 # eager: also the one-time set-up
    grads = _grads(kw["hidden_dim"])
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for g in grads:
            g.zero_()
        call = ops.FrameRenderCall(flat, c2w, cam, engine=None, noise=noise, **kw)
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


# ---- (5) Trainer on injected draws ---------------------------------------------------------------------------------------------
FULL = {"full_loss": dict(full=True), "full_loss_focal": dict(full=True, focal=(2, False))}


@pytest.mark.parametrize("case", list(FULL))
def test_trainer_graph_replay_equals_eager_bits(case, monkeypatch):
    """test_gpu_graph_options' injected draws (those of test_gpu_full_loss_repro) with full losses from the first step: the captured
    frame_grad step and the same step body launched eagerly give bit-identical losses, weights, r, t, scales and shifts over 5 steps"""
    opts = FULL[case]
    ge = GO._run(opts, "eager", monkeypatch, steps=5, frame_grad=True)
    gg = GO._run(opts, "graph", monkeypatch, steps=5, frame_grad=True)
    assert ge["tr"].frame_grad and gg["tr"].frame_grad
    assert len(gg["gsteps"]) == 1 and gg["gsteps"][0].graph is not None and gg["gsteps"][0].calls == 5
    assert ge["losses"][:, 4].min() > 0 and ge["losses"][:, 5].min() > 0
    for k in ("losses", "w", "r", "t", "scales", "shifts", "focal"):
        if k in ge:
            assert ge[k].tobytes() == gg[k].tobytes(), (k, np.abs(ge[k] - gg[k]).max())


@pytest.mark.parametrize("case", list(FULL))
def test_trainer_frame_grad_against_stash_path(case, monkeypatch):
    """frame_grad True against False on the same draws (graph steps).  Step 1's forward is the same bits, so its losses are equal; its
    gradients differ in the order of their sums only (<= 1e-4 of each part's maximum, as the ops-level gate).  Such differences are of
    the size the captured-vs-eager comparison of test_gpu_graph_options sees from its forked-stream atomics, and Adam's first steps
    (about lr x sign(g)) amplify them the same way for near-zero gradients, so after 5 steps its gates apply."""
    opts = FULL[case]
    ff = GO._run(opts, "graph", monkeypatch, steps=5, frame_grad=True)
    fs = GO._run(opts, "graph", monkeypatch, steps=5)
    assert ff["tr"].frame_grad and not fs["tr"].frame_grad
    assert ff["losses"][0].tobytes() == fs["losses"][0].tobytes()
    n_mlp = ff["tr"].model.renderer.model.num_params
    V = GO.V
    w0 = O.flatten_params(O.init_params(seed=9, hf_damp=True)).astype(np.float64)
    r0 = (torch.randn(V, 3, generator=torch.Generator().manual_seed(5)) * 0.03).numpy().astype(np.float64)
    t0 = (torch.randn(V, 3, generator=torch.Generator().manual_seed(6)) * 0.03).numpy().astype(np.float64)
    upd = lambda k, p0: np.linalg.norm((ff[k] - p0) - (fs[k] - p0)) / max(np.linalg.norm(fs[k] - p0), 1e-30)
    le, lf = fs["losses"], ff["losses"]
    e = dict(g1_mlp=GO._relmax(ff["g_first"][:n_mlp], fs["g_first"][:n_mlp]), g1_pose=GO._relmax(ff["g_first"][n_mlp:], fs["g_first"][n_mlp:]),
             loss=np.abs(le - lf).max() / np.abs(le).max(), w=np.linalg.norm((ff["w"] - w0) - (fs["w"] - w0)) / np.linalg.norm(fs["w"] - w0),
             r=upd("r", r0), t=upd("t", t0), r_abs=np.abs(ff["r"] - fs["r"]).max(), t_abs=np.abs(ff["t"] - fs["t"]).max(),
             shifts=GO._relmax(ff["shifts"], fs["shifts"]))
    if "focal" in fs:
        e["focal"] = np.abs(ff["focal"] - fs["focal"]).max() / np.abs(fs["focal"]).max()
    print("frame_grad vs stash", case, e)
    assert e["g1_mlp"] < 1e-4 and e["g1_pose"] < 1e-4, e
    assert e.get("focal", 0.0) <= 1e-5, e
    assert e["loss"] < 1e-5, e
    assert e["w"] < 2e-2 and e["r"] < 0.1 and e["t"] < 0.1 and e["r_abs"] < 5e-4 and e["t_abs"] < 5e-4 and e["shifts"] < 1e-3, e


# ---- (6) the stored reference results --------------------------------------------------------------------------------------------
@pytest.fixture
def frame_trainer(monkeypatch):
    """every Trainer built in the test gets frame_grad=True; counts the training renders that ran the frame pair"""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    count = {"frame": 0}
    base, base_call = mdl.Trainer, ops.FrameRenderCall

    class FrameTrainer(base):
        def __init__(self, *a, **k):
            super().__init__(*a, **dict(k, frame_grad=True))

    class CountingCall(base_call):
        def __init__(self, *a, **k):
            count["frame"] += 1
            super().__init__(*a, **k)
    monkeypatch.setattr(mdl, "Trainer", FrameTrainer)
    monkeypatch.setattr(ops, "FrameRenderCall", CountingCall)
    return count


@pytest.mark.parametrize("name,with_ref", [("train_render_only", False), ("train_full_losses", True)])
def test_parity_golden(name, with_ref, frame_trainer, monkeypatch):
    GP.test_trainer_step_vs_reference_golden(name, with_ref, "tc", monkeypatch)
    assert frame_trainer["frame"] >= 2


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("name,with_ref", SC.TRAIN)
def test_sample_count_golden(name, with_ref, graph, frame_trainer, monkeypatch):
    SC.test_trainer_steps_vs_reference_golden(name, with_ref, "tc", graph, monkeypatch)
    assert frame_trainer["frame"] >= 2


# ---- (7) memory -------------------------------------------------------------------------------------------------------------------
def test_large_graph_step_memory(monkeypatch):
    """a frame_grad graph step at N = 4096, S = 512, D = 256 runs, and its peak allocation is far below the stash path's workspace.
    The peak is counted above what was allocated before the Trainer was built: memory that earlier test modules of the same process
    still hold (module-level caches, live tensors) is not the step's."""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops, _lib as L
    from _cfg import default_cfg
    N, S, H, W, V, hd, wd = 4096, 512, 128, 160, 3, 32, 40
    stash_ws = L.lib.nnb_workspace_bytes_dim(N, S, L.STASH, L.ENGINE_TC, 256)
    ops.set_default_engine("tc")
    ops._pool.free.clear(); gc.collect(); torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    cfg = default_cfg()
    cfg["rendering"]["num_points"] = S; cfg["training"]["n_training_points"] = N
    cfg["training"]["pc_weight"] = [0.0, 0.0]; cfg["training"]["rgb_s_weight"] = [0.0, 0.0]
    dev = torch.device("cuda")
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=9, hf_damp=True).items()})
    model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
    pose = mdl.LearnPose(V, True, True, cfg).to(dev); dist = mdl.Learn_Distortion(V, True, True, cfg).to(dev)
    tr = mdl.Trainer(model, torch.optim.Adam(model.parameters(), lr=1e-3), cfg["training"], device=dev,
                     optimizer_pose=torch.optim.Adam(pose.parameters(), lr=5e-4), pose_param_net=pose,
                     optimizer_distortion=torch.optim.Adam(dist.parameters(), lr=5e-4), distortion_net=dist, use_cuda_graph=True,
                     frame_grad=True)
    g = torch.Generator().manual_seed(4)
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
    data = {"img": torch.rand(1, 3, H, W, generator=g).cuda(), "img.idx": torch.tensor([1]), "img.dpt": (torch.rand(1, hd, wd, generator=g) * 3 + 2).cuda(),
            "img.camera_mat": cam, "img.scale_mat": torch.eye(4)[None], "img.ref_imgs": torch.rand(1, 3, H, W, generator=g).cuda(),
            "img.ref_dpts": (torch.rand(1, hd, wd, generator=g) * 3 + 2).cuda(), "img.ref_idxs": torch.tensor([2])}
    losses = []
    for it in range(3):                                        # eager warm-up, capture, replay
        ld = tr.train_step(data, it=it, epoch=0, scheduling_start=10000, render_path=None)
        losses.append(float(ld["loss"]))
    torch.cuda.synchronize()
    gsteps = [v for v in tr._gsteps.values() if v]
    assert len(gsteps) == 1 and gsteps[0].graph is not None and gsteps[0].calls == 3
    assert np.isfinite(losses).all() and torch.isfinite(net.flat_weights()).all()
    peak = torch.cuda.max_memory_allocated() - base
    print("frame_grad graph step N=%d S=%d D=256: peak %.2f GB above %.2f GB held before, stash workspace %.2f GB, frame workspace %.2f GB"
          % (N, S, peak / 1e9, base / 1e9, stash_ws / 1e9, L.lib.nnb_render_frame_bwd_workspace_bytes(N, S, 256) / 1e9))
    assert peak < stash_ws / 4, (peak, stash_ws)
    del tr, gsteps, model, net
    gc.collect(); torch.cuda.empty_cache()

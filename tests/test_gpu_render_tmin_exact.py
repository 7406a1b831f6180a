"""GPU: nnb_render_fwd_tmin_engine / nnb_render_bwd_tmin_engine on the exact-fp32 engine (ops.exact_stash_render_call(t_min),
Trainer(train_t_min=t, train_t_min_engine='simt')), training with early ray termination on the exact engine's per-sample stash.
(1) at S <= 32 (one round) every output and gradient is RenderCall(engine=ENGINE_SIMT, stash=True) + backward()'s bit for bit, over
S = 2, 8, 17 and 32, both density heads, D = 64, 128 and 256, ragged N, with and without noise, and n_eval == S;
(2) at t_min = 0 and S = 33, 128, 512 the outputs are RenderCall(engine=ENGINE_SIMT)'s bits and g_c2w, g_cam and g_scale_shift
ExactFrameRenderCall's (the same per-ray sums in the same order); dW / db are within DW_GATE of each tensor's maximum of
ExactFrameRenderCall's, whose weight-gradient stage runs once per round;
(3) at t_min > 0 without noise, rgb, depth_pred, depth_gt, mask and n_eval are render_frame_engine(engine=ENGINE_SIMT)'s bits on the seeded
surface field (every ray stops after chunk 0) and on the scattered plant s256 (rays stop in at least 4 rounds);
(4) the gradients at t_min > 0, with and without noise, against float64 autograd of the truncated render under the gate of
test_gpu_render_frame_train_tmin, which the untruncated render and the suffix started at the last chunk both exceed;
(5) on the seeded surface field at t_min = 1e-4 the tensor-core and exact pairs give the same n_eval, and outputs and gradients within
test_gpu_parity's tensor-core-versus-exact tolerances;
(6) repeated pairs, workspaces filled with 0x00, 0xFF (NaN) and 0x7E (large values), interleaved pairs and a graph-captured pair replayed
after the weights change the stop pattern give the same bits, and a pose-only backward runs;
(7) nnb_render_fwd_tmin_engine / _bwd_tmin_engine on NNB_ENGINE_TC give nnb_render_fwd_tmin / _bwd_tmin's bits;
(8) Trainer: train_t_min=0.0 gives the default exact step's first losses; at S = 8 five captured steps give the default exact Trainer's
losses and parameters bit for bit; at 1e-4 the captured step equals its eager body over 5 full-loss steps, with and without a learned
focal.

Largest values measured (NVIDIA H100 80GB HBM3, 700 W power limit): (2) dW / db 4.8e-6 of each tensor's maximum (gate 5e-5); (4) 4.1e-5
(g_cam, s256 without noise; 2.5e-5 with noise) under the 3.6e-3 gate, wrong answers at least 9.7e-3 (untruncated) and 7.2e-3 (suffix
from the last chunk); (5) outputs 2.2e-7, pose gradients 3.0e-6 (gate 1e-4), dW 2.8e-4 (gate 5e-4), depth_gt and mask equal.
"""
import gc

import numpy as np
import pytest
import torch

from nope_nerf_b200 import _lib as L
from oracle import nerf_oracle as O
from test_gpu_render_frame_grad import _case, _rel
from test_gpu_render_frame_train_tmin import _equal, _grads, _noise, truncated_reference
import test_gpu_graph_options as GO
import test_gpu_ray_local as RL
import test_gpu_render_frame_local as FL

pytestmark = pytest.mark.gpu
DW_GATE = 5e-5   # (2): dW / db against ExactFrameRenderCall, relative to each tensor's maximum


@pytest.fixture(autouse=True)
def _keep_default_engine(monkeypatch):
    from nope_nerf_b200 import ops
    monkeypatch.setattr(ops, "_DEFAULT_ENGINE", list(ops._DEFAULT_ENGINE))


@pytest.fixture(scope="module", autouse=True)
def _release_pool():
    yield
    from nope_nerf_b200 import ops
    ops._pool.free.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _cls(t):
    from nope_nerf_b200 import ops
    return ops.exact_stash_render_call(t)


def _pair(cls, flat, c2w, cam, kw, gs, noise=None, engine=L.ENGINE_SIMT):
    """cls(...) + backward: [rgb, depth_pred, depth_gt, mask, g_weights, g_c2w, g_cam, g_scale_shift], n_eval (or None)"""
    call = cls(flat, c2w, cam, engine=engine, noise=noise, stash=True, **kw)
    g = _grads(kw["hidden_dim"])
    call.backward(*gs, *g[:3], None, g[3])
    torch.cuda.synchronize()
    return [t.clone() for t in (call.rgb, call.depth_pred, call.depth_gt, call.mask) + g], getattr(call, "n_eval", None)


def _planted(name):
    P, inp, flags, D = FL.planted(name)
    return (FL._cu(O.flatten_params(P)), FL._cu(inp["c2w"]), FL._cu(inp["cam"]), FL._call_kw(inp, flags, D),
            (FL._cu(inp["g_rgb"]), FL._cu(inp["g_dp"]), FL._cu(inp["g_dg"])))


def _dw_worst(got, ref, D):
    from nope_nerf_b200.model.official_nerf import param_slices
    worst = 0.0
    for (o, n, shape) in param_slices(D):
        r = ref[o:o + n]
        if r.abs().max() > 0:
            worst = max(worst, _rel(got[o:o + n], r))
    return worst


# ---- (1) one round: the exact stash path's bits ----------------------------------------------------------------------------------
ONE = [(257, 2, 64, "softplus"), (301, 8, 128, "relu"), (129, 17, 256, "softplus"), (130, 32, 64, "relu"), (77, 17, 128, "relu"),
       (37, 32, 256, "softplus"), (1000, 8, 256, "relu")]


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("case", range(len(ONE)))
def test_one_round_is_the_exact_stash_path(case, noise):
    from nope_nerf_b200 import ops
    N, S, D, occ = ONE[case]
    flat, c2w, cam, kw, gs = _case(N, S, D, dict(dist_alpha=case % 2 == 1), occ=occ, seed=60 + case)
    nz = _noise(kw, case) if noise else None
    ref, _ = _pair(ops.RenderCall, flat, c2w, cam, kw, gs, nz)
    for t in (1e-4, 0.0):
        got, n_eval = _pair(_cls(t), flat, c2w, cam, kw, gs, nz, engine=L.ENGINE_TC)   # the engine argument is ignored
        _equal(got, ref, "case %d t %g" % (case, t))
        assert (n_eval == S).all()
    assert ref[4].abs().max() > 0 and ref[5].abs().max() > 0


# ---- (2) t_min = 0 over several rounds -----------------------------------------------------------------------------------------
ZERO = [(301, 33, 128, "relu"), (129, 128, 256, "softplus"), (130, 512, 64, "relu"), (37, 512, 256, "softplus")]


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("case", range(len(ZERO)))
def test_t_min_zero_against_the_exact_frame_pair(case, noise):
    from nope_nerf_b200 import ops
    N, S, D, occ = ZERO[case]
    flat, c2w, cam, kw, gs = _case(N, S, D, dict(dist_alpha=case % 2 == 1), occ=occ, seed=70 + case)
    nz = _noise(kw, case) if noise else None
    got, n_eval = _pair(_cls(0.0), flat, c2w, cam, kw, gs, nz)
    assert (n_eval == S).all()
    plain = ops.RenderCall(flat, c2w, cam, engine=L.ENGINE_SIMT, noise=nz, **kw)
    torch.cuda.synchronize()
    _equal(got[:4], [plain.rgb, plain.depth_pred, plain.depth_gt, plain.mask], "outputs vs RenderCall(ENGINE_SIMT)")
    ref, _ = _pair(ops.ExactFrameRenderCall, flat, c2w, cam, kw, gs, nz)
    _equal(got[5:], ref[5:], "g_c2w, g_cam, g_scale_shift vs ExactFrameRenderCall")
    worst = _dw_worst(got[4], ref[4], D)
    print("S <= 1024 t=0 case", case, "noise", noise, "dW worst vs exact frame pair %.2e" % worst)
    assert worst <= DW_GATE, worst
    assert ref[4].abs().max() > 0 and ref[5].abs().max() > 0


# ---- (3) the forward at t_min > 0 ------------------------------------------------------------------------------------------------
def _field(name):
    if name == "seeded":
        return _case(1000, 128, 256, seed=3)
    return _planted(name)


@pytest.mark.parametrize("name,t", [("seeded", 1e-4), ("s256", 1e-3)])
def test_forward_is_render_frame_engine(name, t):
    from nope_nerf_b200 import ops
    flat, c2w, cam, kw, gs = _field(name)
    S, C = kw["S"], (kw["S"] + 31) // 32
    got, n_eval = _pair(_cls(t), flat, c2w, cam, kw, gs)
    *outs, n_ref, _ = ops.render_frame_engine(flat, c2w, cam, engine=L.ENGINE_SIMT, t_min=t, want_stats=True, **kw)
    torch.cuda.synchronize()
    _equal(got[:4] + [n_eval], outs + [n_ref], name)
    rounds = ((n_eval + 31) // 32 - 1).cpu().numpy()
    print(name, "t", t, "rays per stop round", np.bincount(rounds, minlength=C))
    if name == "seeded":
        assert (n_eval == 32).all(), "the seeded surface field stops every ray after chunk 0"
    else:
        assert len(set(rounds[rounds < C - 1].tolist())) >= 4


# ---- (4) gradients against float64 of the truncated render ---------------------------------------------------------------------
@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("name,t,kind", [("s256", 1e-3, "scattered"), ("t100", 1.0, "round0"), ("t100-relu", 1.0, "round0")])
def test_gradients_against_float64_truncated(name, t, kind, noise, monkeypatch):
    from nope_nerf_b200 import ops
    P, inp, flags, D = FL.planted(name)
    N, S = inp["N"], inp["S"]
    C = (S + 31) // 32
    kw = FL._call_kw(inp, flags, D)
    nz = FL._cu(inp["noise"]) if noise else None
    ops._pool.free.clear()   # a workspace of large floats: a value read without being written shows in the gradients
    ops._pool.give(torch.full((L.lib.nnb_render_tmin_workspace_bytes_engine(N, S, D, L.ENGINE_SIMT),), 0x7E, dtype=torch.uint8, device="cuda"))
    call = _cls(t)(FL._cu(O.flatten_params(P)), FL._cu(inp["c2w"]), FL._cu(inp["cam"]), engine=None, noise=nz, **kw)
    outs = (call.rgb.clone(), call.depth_pred.clone(), call.depth_gt.clone())
    n_eval = call.n_eval.clone()
    g = FL._grads(D, N)
    call.backward(FL._cu(inp["g_rgb"]), FL._cu(inp["g_dp"]), FL._cu(inp["g_dg"]), g["w"], g["g_c2w"], g["g_cam"], None, g["g_scale_shift"])
    torch.cuda.synchronize()
    ops._pool.free.clear()
    got = FL._got(outs, g, D, False)
    stop_round = ((n_eval + 31) // 32 - 1).cpu().numpy()
    if kind == "scattered" and not noise:
        assert len(set(stop_round[stop_round < C - 1].tolist())) >= 4, np.bincount(stop_round)
    elif kind == "round0":
        assert (n_eval == 32).all()
    st = FL.stash_run(P, inp, flags, D, "simt", noise=noise)
    s_gate = (st["rec"][:, 4] > 0).double()
    gates = [x.double() for x in st["gates"]]
    mask = (torch.arange(S, device="cuda")[None, :] < n_eval[:, None]).double()
    if noise:   # the reference's samples with the same jitter
        ray_stage = RL.ray_stage
        monkeypatch.setattr(RL, "ray_stage", lambda A, q, fl, S_, nzr: ray_stage(A, q, fl, S_, A.t(inp["noise"], "cuda") if nzr is None else nzr))
    ref_outs, G, wrong = truncated_reference(P, inp, flags, gates, s_gate, mask)
    ref = dict(ref_outs, **G)
    err = FL.compare(got, ref)
    gate = FL.E2E_GATES["scattered"]["tc"]
    worst = max(err.items(), key=lambda kv: kv[1])
    teeth = {bug: max(float((got[k].double() - Gw[k]).abs().max()) / max(float(ref[k].abs().max()), 1e-300) for k in G)
             for bug, Gw in wrong.items()}
    print(name, "t_min", t, "noise", noise, "rays per stop round", np.bincount(stop_round, minlength=C), "worst", worst, "gate", gate,
          "wrong", teeth)
    assert worst[1] <= gate, (worst, gate)
    for bug, sc in teeth.items():
        assert sc > gate, (bug, sc, gate)


# ---- (5) the two engines' pairs ---------------------------------------------------------------------------------------------------
def test_engines_agree_on_the_seeded_field():
    from nope_nerf_b200 import ops
    flat, c2w, cam, kw, gs = _case(1000, 128, 256, seed=3)
    nz = _noise(kw, 7)
    tc, n_tc = _pair(ops.stash_render_call(1e-4), flat, c2w, cam, kw, gs, nz, engine=L.ENGINE_TC)
    ex, n_ex = _pair(_cls(1e-4), flat, c2w, cam, kw, gs, nz)
    assert torch.equal(n_tc, n_ex) and (n_ex < kw["S"]).all()
    rel = lambda x, y: ((x - y).abs().max() / x.abs().max().clamp_min(1e-30)).item()
    e = dict(rgb=rel(ex[0], tc[0]), dp=rel(ex[1], tc[1]), dg=rel(ex[2], tc[2]), gw=rel(ex[4], tc[4]), gc=rel(ex[5], tc[5]),
             gcam=rel(ex[6], tc[6]), gss=rel(ex[7], tc[7]))
    print("exact vs tensor-core stash pair, seeded field, t_min 1e-4:", e)
    assert torch.equal(ex[3], tc[3])
    assert max(e["rgb"], e["dp"], e["dg"], e["gc"], e["gcam"], e["gss"]) < 1e-4 and e["gw"] < 5e-4, e


# ---- (6) determinism, workspace state, interleaving, graph replay ---------------------------------------------------------------
def test_repeated_interleaved_and_workspace_independent():
    from nope_nerf_b200 import ops
    flat, c2w, cam, kw, gs = _planted("s256")
    nz = _noise(kw, 5)
    cls = _cls(1e-3)
    ref, n0 = _pair(cls, flat, c2w, cam, kw, gs, nz)
    assert (n0 < kw["S"]).any() and (n0 == kw["S"]).any()
    for _ in range(2):
        _equal(_pair(cls, flat, c2w, cam, kw, gs, nz)[0], ref, "repeat")
    nbytes = L.lib.nnb_render_tmin_workspace_bytes_engine(kw["N"], kw["S"], kw["hidden_dim"], L.ENGINE_SIMT)
    for fill in (0x00, 0xFF, 0x7E):
        ops._pool.free.clear()
        ops._pool.give(torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda"))
        _equal(_pair(cls, flat, c2w, cam, kw, gs, nz)[0], ref, fill)
    ops._pool.free.clear()
    a = cls(flat, c2w, cam, engine=None, noise=nz, **kw)   # two forwards in flight, their backwards in the other order
    b = cls(flat, c2w, cam, engine=None, noise=nz, **kw)
    ga, gb = _grads(kw["hidden_dim"]), _grads(kw["hidden_dim"])
    b.backward(*gs, *gb[:3], None, gb[3])
    a.backward(*gs, *ga[:3], None, ga[3])
    torch.cuda.synchronize()
    for call, g in ((a, ga), (b, gb)):
        _equal([call.rgb, call.depth_pred, call.depth_gt, call.mask] + list(g), ref, "interleaved")


def test_graph_replay_after_weights_change():
    P, inp, flags, D = FL.planted("s256")
    c2w, cam, kw = FL._cu(inp["c2w"]), FL._cu(inp["cam"]), FL._call_kw(inp, flags, D)
    gs = (FL._cu(inp["g_rgb"]), FL._cu(inp["g_dp"]), FL._cu(inp["g_dg"]))
    nz = FL._cu(inp["noise"])
    cls = _cls(1e-3)
    w_a = FL._cu(O.flatten_params(P))
    P_b = dict(P); P_b["fc_density.bias"] = P["fc_density.bias"] - np.float32(1.5)   # fewer rays stop, later
    w_b = FL._cu(O.flatten_params(P_b))
    ref_a, n_a = _pair(cls, w_a, c2w, cam, kw, gs, nz)
    ref_b, n_b = _pair(cls, w_b, c2w, cam, kw, gs, nz)
    assert not torch.equal(n_a, n_b), "the stop pattern changes with the weights"
    flat = w_a.clone()
    grads = _grads(D)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for g in grads:
            g.zero_()
        call = cls(flat, c2w, cam, engine=None, noise=nz, **kw)
        call.pooled = False
        ws = call.ws
        call.backward(*gs, *grads[:3], None, grads[3])
    for w, ref, n_ref in ((w_b, ref_b, n_b), (w_a, ref_a, n_a), (w_b, ref_b, n_b)):
        flat.copy_(w)
        graph.replay()
        torch.cuda.synchronize()
        _equal([call.rgb, call.depth_pred, call.depth_gt, call.mask] + list(grads), ref, "graph replay")
        assert torch.equal(call.n_eval, n_ref)
    del graph, ws


def test_pose_only_backward():
    flat, c2w, cam, kw, gs = _planted("s256")
    ref, _ = _pair(_cls(1e-3), flat, c2w, cam, kw, gs)
    call = _cls(1e-3)(flat, c2w, cam, engine=None, **kw)
    g = _grads(kw["hidden_dim"])
    call.backward(*gs, None, g[1], g[2], None, g[3])
    torch.cuda.synchronize()
    _equal([g[1], g[2], g[3]], ref[5:], "pose only")


# ---- (7) the _engine calls on the tensor-core engine ----------------------------------------------------------------------------
def test_engine_calls_on_tc_are_the_plain_calls(monkeypatch):
    from nope_nerf_b200 import ops
    flat, c2w, cam, kw, gs = _planted("s256")
    nz = _noise(kw, 3)
    cls = ops.stash_render_call(1e-3)
    ref, n_ref = _pair(cls, flat, c2w, cam, kw, gs, nz, engine=L.ENGINE_TC)
    monkeypatch.setattr(L.lib, "nnb_render_fwd_tmin", L.lib.nnb_render_fwd_tmin_engine)
    monkeypatch.setattr(L.lib, "nnb_render_bwd_tmin", L.lib.nnb_render_bwd_tmin_engine)
    got, n_got = _pair(cls, flat, c2w, cam, kw, gs, nz, engine=L.ENGINE_TC)
    _equal(got, ref, "_engine on NNB_ENGINE_TC")
    assert torch.equal(n_got, n_ref) and (n_ref < kw["S"]).any()


# ---- (8) Trainer ----------------------------------------------------------------------------------------------------------------------
EXACT = dict(train_t_min_engine="simt")


def test_trainer_t_min_zero_first_step_is_the_default_exact_step(monkeypatch):
    from nope_nerf_b200 import ops
    ops.set_default_engine("simt")
    opts = dict(full=True)
    a = GO._run(opts, "graph", monkeypatch, steps=1)
    b = GO._run(opts, "graph", monkeypatch, steps=1, train_t_min=0.0, **EXACT)
    assert b["tr"]._train_render_call(True) is ops.exact_stash_render_call(0.0)
    assert a["losses"].tobytes() == b["losses"].tobytes(), (a["losses"], b["losses"])


def test_trainer_one_round_equals_the_default_exact_trainer(monkeypatch):
    """at S = 8 the pair's gradients are the exact stash path's bits, so five captured steps give the same losses and parameters"""
    from nope_nerf_b200 import ops
    ops.set_default_engine("simt")
    monkeypatch.setattr(GO, "S", 8)
    opts = dict(full=True)
    a = GO._run(opts, "graph", monkeypatch, steps=5)
    b = GO._run(opts, "graph", monkeypatch, steps=5, train_t_min=1e-4, **EXACT)
    assert len(b["gsteps"]) == 1 and b["gsteps"][0].graph is not None and b["gsteps"][0].calls == 5
    for k in ("losses", "w", "r", "t", "scales", "shifts"):
        assert a[k].tobytes() == b[k].tobytes(), (k, np.abs(a[k] - b[k]).max())


@pytest.mark.parametrize("opts", [dict(full=True), dict(full=True, focal=(2, False))], ids=["full", "full_focal"])
def test_trainer_graph_equals_eager(monkeypatch, opts):
    ge = GO._run(opts, "eager", monkeypatch, steps=5, train_t_min=1e-4, **EXACT)
    gg = GO._run(opts, "graph", monkeypatch, steps=5, train_t_min=1e-4, **EXACT)
    assert gg["tr"].train_t_min_engine == "simt"
    assert len(gg["gsteps"]) == 1 and gg["gsteps"][0].graph is not None and gg["gsteps"][0].calls == 5
    for k in ("losses", "w", "r", "t", "scales", "shifts", "focal"):
        if k in ge:
            assert ge[k].tobytes() == gg[k].tobytes(), (k, np.abs(ge[k] - gg[k]).max())

"""GPU: nnb_render_fwd_tmin / nnb_render_bwd_tmin (ops.stash_render_call(t_min), Trainer(train_t_min=t)), training with early ray
termination on the per-sample stash: each sample evaluated once, rows packed round by round, one weight-gradient stage.
(1) rgb, depth_pred, depth_gt, mask and n_eval are the frame tmin pair's (ops.frame_render_call) bits at the same t_min, with and without
noise, over both density heads, D = 64, 128 and 256, S = 16, 33, 128 and 512 and ragged N, on the seeded surface field (every ray stops
after chunk 0) and the scattered plant of test_gpu_render_frame_local (rays stop in at least 4 rounds); at t_min = 0 they are
RenderCall(stash=True)'s bits.  g_c2w, g_cam and g_scale_shift equal the frame pair's bit for bit (the same per-sample arithmetic, the
same per-ray sums in the same order); every dW / db is within DW_GATE of its tensor's maximum: the weight-gradient sums run once over
the packed rows instead of once per round, so they add the same terms in another order (worst measured 3.2e-5 on the scattered plant
s256 and 1.7e-5 at D = 64, S = 512, where (2) finds both pairs equally close to float64; at most 9.7e-6 on the other fields);
(2) the gradients against float64 autograd of the truncated render under the gate of test_gpu_render_frame_train_tmin, which the
untruncated render and the suffix started at the last chunk exceed;
(3) repeated pairs, workspaces filled with 0x00, 0xFF (NaN) and 0x7E (large values), interleaved pairs and a graph-captured pair replayed
after the weights change the stop pattern give the same bits;
(4) Trainer: train_t_min=0.0 gives the default step's first losses, the captured step at 1e-4 equals its eager body over 5 full-loss steps
with and without a learned focal, and a pose-only backward (g_weights=None) runs.
"""
import gc

import numpy as np
import pytest
import torch

from nope_nerf_b200 import _lib as L
from oracle import nerf_oracle as O
from test_gpu_render_frame_grad import _case, _rel
from test_gpu_render_frame_train_tmin import _equal, _grads, _noise, _pair, truncated_reference, ZERO
import test_gpu_graph_options as GO
import test_gpu_render_frame_local as FL

pytestmark = pytest.mark.gpu
DW_GATE = 5e-5   # dW / db against the frame tmin pair, relative to each tensor's maximum (see (1))


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


def _planted(name):
    P, inp, flags, D = FL.planted(name)
    return (FL._cu(O.flatten_params(P)), FL._cu(inp["c2w"]), FL._cu(inp["cam"]), FL._call_kw(inp, flags, D),
            (FL._cu(inp["g_rgb"]), FL._cu(inp["g_dp"]), FL._cu(inp["g_dg"])))


def _against_frame_pair(flat, c2w, cam, kw, gs, t, nz, what):
    """the stash pair against the frame tmin pair: outputs, n_eval and pose gradients bitwise, dW within 1e-5 of each tensor's max"""
    from nope_nerf_b200 import ops
    from nope_nerf_b200.model.official_nerf import param_slices
    ref, n_ref = _pair(ops.frame_render_call(t), flat, c2w, cam, kw, gs, nz)
    got, n_got = _pair(ops.stash_render_call(t), flat, c2w, cam, kw, gs, nz)
    _equal(got[:4], ref[:4], what + " outputs")
    assert torch.equal(n_got, n_ref), what
    _equal(got[5:], ref[5:], what + " g_c2w, g_cam, g_scale_shift")
    worst = 0.0
    for (o, n, shape) in param_slices(kw["hidden_dim"]):
        r = ref[4][o:o + n]
        if r.abs().max() > 0:
            worst = max(worst, _rel(got[4][o:o + n], r))
    assert worst <= DW_GATE, (what, worst)
    assert ref[4].abs().max() > 0 and ref[5].abs().max() > 0
    return got, n_got, worst


# ---- (1) the frame tmin pair's bits ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", [0.0, 1e-3])
@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("case", range(len(ZERO)))
def test_matches_frame_tmin_pair(case, noise, t):
    from nope_nerf_b200 import ops
    N, S, D, occ = ZERO[case]
    flat, c2w, cam, kw, gs = _case(N, S, D, dict(dist_alpha=case % 2 == 1), occ=occ, seed=40 + case)
    nz = _noise(kw, case) if noise else None
    got, n_eval, worst = _against_frame_pair(flat, c2w, cam, kw, gs, t, nz, "case %d" % case)
    if t == 0.0:
        assert (n_eval == S).all()
        call = ops.RenderCall(flat, c2w, cam, engine=None, noise=nz, stash=True, **kw)
        call.release()
        torch.cuda.synchronize()
        _equal(got[:4], [call.rgb, call.depth_pred, call.depth_gt, call.mask], "t = 0 vs RenderCall(stash=True)")
    print("case", case, "noise", noise, "t", t, "mean n_eval %.1f" % n_eval.float().mean(), "dW worst %.2e" % worst)


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("name,t", [("seeded", 1e-4), ("s256", 1e-3), ("t100", 1.0)])
def test_matches_frame_tmin_pair_on_stopping_fields(name, t, noise):
    if name == "seeded":
        flat, c2w, cam, kw, gs = _case(1000, 128, 256, seed=3)
    else:
        flat, c2w, cam, kw, gs = _planted(name)
    nz = _noise(kw, 11) if noise else None
    _, n_eval, worst = _against_frame_pair(flat, c2w, cam, kw, gs, t, nz, name)
    S, C = kw["S"], (kw["S"] + 31) // 32
    rounds = ((n_eval + 31) // 32 - 1).cpu().numpy()
    print(name, "t", t, "noise", noise, "rays per stop round", np.bincount(rounds, minlength=C), "dW worst %.2e" % worst)
    if name == "s256" and not noise:
        assert len(set(rounds[rounds < C - 1].tolist())) >= 4
    if name == "seeded":
        assert (n_eval == 32).all(), "the seeded surface field stops every ray after chunk 0"


# ---- (2) gradients against float64 of the truncated render ---------------------------------------------------------------------
def _stash_grads(P, inp, flags, D, t):
    """the stash pair in a workspace filled with 0x7E (large floats): a value read without being written shows in the gradients"""
    from nope_nerf_b200 import ops
    ops._pool.free.clear()
    ops._pool.give(torch.full((L.lib.nnb_render_tmin_workspace_bytes(inp["N"], inp["S"], D),), 0x7E, dtype=torch.uint8, device="cuda"))
    call = ops.stash_render_call(t)(FL._cu(O.flatten_params(P)), FL._cu(inp["c2w"]), FL._cu(inp["cam"]), engine=None,
                                    **FL._call_kw(inp, flags, D))
    outs = (call.rgb.clone(), call.depth_pred.clone(), call.depth_gt.clone())
    n_eval = call.n_eval.clone()
    g = FL._grads(D, inp["N"])
    call.backward(FL._cu(inp["g_rgb"]), FL._cu(inp["g_dp"]), FL._cu(inp["g_dg"]), g["w"], g["g_c2w"], g["g_cam"], None, g["g_scale_shift"])
    torch.cuda.synchronize()
    return FL._got(outs, g, D, False), n_eval


@pytest.mark.parametrize("name,t,kind", [("s256", 1e-3, "scattered"), ("t100", 1.0, "round0"), ("t100-relu", 1.0, "round0")])
def test_gradients_against_float64_truncated(name, t, kind):
    P, inp, flags, D = FL.planted(name)
    S = inp["S"]
    C = (S + 31) // 32
    got, n_eval = _stash_grads(P, inp, flags, D, t)
    stop_round = ((n_eval + 31) // 32 - 1).cpu().numpy()
    if kind == "scattered":
        assert len(set(stop_round[stop_round < C - 1].tolist())) >= 4, np.bincount(stop_round)
    else:
        assert (n_eval == 32).all()
    st = FL.stash_run(P, inp, flags, D, "tc", noise=False)
    s_gate = (st["rec"][:, 4] > 0).double()
    gates = [g.double() for g in st["gates"]]
    mask = (torch.arange(S, device="cuda")[None, :] < n_eval[:, None]).double()
    outs, G, wrong = truncated_reference(P, inp, flags, gates, s_gate, mask)
    ref = dict(outs, **G)
    err = FL.compare(got, ref)
    gate = FL.E2E_GATES["scattered"]["tc"]
    worst = max(err.items(), key=lambda kv: kv[1])
    teeth = {bug: max(float((got[k].double() - Gw[k]).abs().max()) / max(float(ref[k].abs().max()), 1e-300) for k in G)
             for bug, Gw in wrong.items()}
    print(name, "t_min", t, "rays per stop round", np.bincount(stop_round, minlength=C), "worst", worst, "gate", gate, "wrong", teeth)
    assert worst[1] <= gate, (worst, gate)
    for bug, sc in teeth.items():
        assert sc > gate, (bug, sc, gate)


# ---- (3) determinism, workspace state, interleaving, graph replay ---------------------------------------------------------------
def test_repeated_interleaved_and_workspace_independent():
    from nope_nerf_b200 import ops
    flat, c2w, cam, kw, gs = _planted("s256")
    nz = _noise(kw, 5)
    cls = ops.stash_render_call(1e-3)
    ref, n0 = _pair(cls, flat, c2w, cam, kw, gs, nz)
    assert (n0 < kw["S"]).any() and (n0 == kw["S"]).any()
    for _ in range(2):
        _equal(_pair(cls, flat, c2w, cam, kw, gs, nz)[0], ref, "repeat")
    nbytes = L.lib.nnb_render_tmin_workspace_bytes(kw["N"], kw["S"], kw["hidden_dim"])
    for fill in (0x00, 0xFF, 0x7E):
        ops._pool.free.clear()
        ops._pool.give(torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda"))
        _equal(_pair(cls, flat, c2w, cam, kw, gs, nz)[0], ref, fill)
    ops._pool.free.clear()
    # two forwards in flight, their backwards in the other order
    a = cls(flat, c2w, cam, engine=None, noise=nz, **kw)
    b = cls(flat, c2w, cam, engine=None, noise=nz, **kw)
    ga, gb = _grads(kw["hidden_dim"]), _grads(kw["hidden_dim"])
    b.backward(*gs, *gb[:3], None, gb[3])
    a.backward(*gs, *ga[:3], None, ga[3])
    torch.cuda.synchronize()
    for call, g in ((a, ga), (b, gb)):
        _equal([call.rgb, call.depth_pred, call.depth_gt, call.mask] + list(g), ref, "interleaved")


def test_graph_replay_after_weights_change():
    from nope_nerf_b200 import ops
    P, inp, flags, D = FL.planted("s256")
    c2w, cam, kw = FL._cu(inp["c2w"]), FL._cu(inp["cam"]), FL._call_kw(inp, flags, D)
    gs = (FL._cu(inp["g_rgb"]), FL._cu(inp["g_dp"]), FL._cu(inp["g_dg"]))
    nz = FL._cu(inp["noise"])
    cls = ops.stash_render_call(1e-3)
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
    from nope_nerf_b200 import ops
    flat, c2w, cam, kw, gs = _planted("s256")
    ref, _ = _pair(ops.stash_render_call(1e-3), flat, c2w, cam, kw, gs)
    call = ops.stash_render_call(1e-3)(flat, c2w, cam, engine=None, **kw)
    g = _grads(kw["hidden_dim"])
    call.backward(*gs, None, g[1], g[2], None, g[3])
    torch.cuda.synchronize()
    _equal([g[1], g[2], g[3]], ref[5:], "pose only")


# ---- (4) Trainer ----------------------------------------------------------------------------------------------------------------------
def test_trainer_t_min_zero_first_step_is_default(monkeypatch):
    opts = dict(full=True)
    a = GO._run(opts, "graph", monkeypatch, steps=1)
    b = GO._run(opts, "graph", monkeypatch, steps=1, train_t_min=0.0)
    assert b["tr"]._train_render_call(True).t_min == 0.0
    assert a["losses"].tobytes() == b["losses"].tobytes(), (a["losses"], b["losses"])


@pytest.mark.parametrize("opts", [dict(full=True), dict(full=True, focal=(2, False))], ids=["full", "full_focal"])
def test_trainer_t_min_graph_equals_eager(monkeypatch, opts):
    ge = GO._run(opts, "eager", monkeypatch, steps=5, train_t_min=1e-4)
    gg = GO._run(opts, "graph", monkeypatch, steps=5, train_t_min=1e-4)
    assert len(gg["gsteps"]) == 1 and gg["gsteps"][0].graph is not None and gg["gsteps"][0].calls == 5
    for k in ("losses", "w", "r", "t", "scales", "shifts"):
        assert ge[k].tobytes() == gg[k].tobytes(), (k, np.abs(ge[k] - gg[k]).max())

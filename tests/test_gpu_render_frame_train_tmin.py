"""GPU: nnb_render_frame_train_fwd_tmin / nnb_render_frame_train_bwd_tmin (ops.frame_render_call(t_min), Trainer(frame_grad_t_min=t)),
the frame's training pair with early ray termination: reverse round k visits only the rays that evaluated chunk k.
(1) at t_min = 0 the _tmin pair gives the plain pair's outputs and gradients bit for bit, with and without noise, over both density
heads, D = 64, 128 and 256, S = 16, 33, 128 and 512, ragged N and permuted rays; _bwd_tmin after the plain forward gives the same bits;
(2) at t_min > 0 without noise the forward equals render_frame(t_min, want_stats=True) bit for bit (rgb, depth_pred, depth_gt, mask,
n_eval); with noise, rays with n_eval == S keep the t_min = 0 bits and stopped rays stay within the header's bound of them;
(3) the gradients against float64 autograd of the truncated render (test_gpu_render_frame_local's reference with every sample past the
ray's n_eval given zero opacity, the engine's own n_eval and ReLU gates) on its scattered plant (rays stop in at least 4 rounds, asserted)
and on a field where every ray stops in round 0, under that module's end-to-end gate; two wrong answers, the untruncated float64 render
and the truncated field pull-back of the untruncated compositing adjoint (what a suffix started at chunk C - 1 carries), must exceed it;
(4) with zero cotangents on every stopped ray, every dW / db and g_c2w agrees with the t_min = 0 pair within 1e-5 of its tensor's maximum;
(5) repeated pairs, workspaces filled with 0x00, 0xFF (NaN) and 0x7E (large values), and a graph-captured pair replayed after the
weights change in place (so the stop pattern changes) give the eager bits; (6) Trainer: frame_grad_t_min=0.0 gives the frame_grad=True
losses and parameters bit for bit over 5 full-loss graph steps, and at t = 1e-4 the captured step equals its eager body bit for bit.

Largest errors measured (NVIDIA H100 80GB HBM3, 700 W power limit), per tensor |got - ref|max / |ref|max, gate 3.6e-3 (the scattered
end-to-end gate of test_gpu_render_frame_local): scattered plant s256 at t_min = 1e-3 (rays stop in rounds 1, 2, 3, 5 and 6; 228 of 301
never stop) 7.2e-5 (g_cam); every ray stopped in round 0 (t100, t100-relu at t_min = 1) 1.6e-5 and 2.0e-5.  Wrong answers: untruncated
render 1.1e-2 / 1.58 / 4.2, suffix carried from the untruncated render 7.2e-3 / 0.99 / 4.4.  Zero cotangent on stopped rays: dW within
2.1e-6 of the t = 0 pair at D = 256, g_c2w equal.
Mutation check (one line in frame_chunk_adjoint_live on a scratch build: the suffix starts at k == C - 1 instead of k == c_n - 1): the
three float64 cases fail (inf / NaN from the 0x7E-filled workspace) and so does the workspace-independence test.
"""
import gc

import numpy as np
import pytest
import torch

from nope_nerf_b200 import _lib as L
from oracle import nerf_oracle as O
from test_gpu_parity import cuda
from test_gpu_render_frame_grad import _case, _rel
import test_gpu_graph_options as GO
import test_gpu_ray_local as RL
import test_gpu_render_frame_local as FL

pytestmark = pytest.mark.gpu


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


def _noise(kw, seed):
    return cuda(np.random.default_rng(seed).uniform(0, 1, (kw["N"], kw["S"])).astype(np.float32))


def _grads(D):
    return (torch.zeros(L.num_params(D), device="cuda"), torch.zeros(4, 4, device="cuda"), torch.zeros(4, 4, device="cuda"),
            torch.zeros(2, device="cuda"))


def _pair(cls, flat, c2w, cam, kw, gs, noise=None, bwd_tmin=None):
    """cls(...) + backward: [rgb, depth_pred, depth_gt, mask, g_weights, g_c2w, g_cam, g_scale_shift], n_eval (or None).
    bwd_tmin: run backward() through the _tmin call whatever the forward was"""
    call = cls(flat, c2w, cam, engine=None, noise=noise, **kw)
    if bwd_tmin is not None:
        call.t_min = bwd_tmin
    g = _grads(kw["hidden_dim"])
    call.backward(*gs, *g[:3], None, g[3])
    torch.cuda.synchronize()
    return [t.clone() for t in (call.rgb, call.depth_pred, call.depth_gt, call.mask) + g], getattr(call, "n_eval", None)


def _equal(a, b, what=""):
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (what, i)


# ---- (1) t_min = 0 ---------------------------------------------------------------------------------------------------------------
ZERO = [(257, 16, 64, "softplus"), (301, 33, 128, "relu"), (129, 128, 256, "softplus"), (130, 512, 64, "relu"), (77, 128, 128, "relu"),
        (37, 512, 256, "softplus")]


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("case", range(len(ZERO)))
def test_tmin_zero_is_the_plain_pair(case, noise):
    from nope_nerf_b200 import ops
    N, S, D, occ = ZERO[case]
    flat, c2w, cam, kw, gs = _case(N, S, D, dict(dist_alpha=case % 2 == 1), occ=occ, seed=40 + case)
    nz = _noise(kw, case) if noise else None
    ref, _ = _pair(ops.FrameRenderCall, flat, c2w, cam, kw, gs, nz)
    got, n_eval = _pair(ops.frame_render_call(0.0), flat, c2w, cam, kw, gs, nz)
    _equal(got, ref, "tmin pair")
    assert (n_eval == S).all()
    mixed, _ = _pair(ops.FrameRenderCall, flat, c2w, cam, kw, gs, nz, bwd_tmin=0.0)   # plain forward, _bwd_tmin
    _equal(mixed, ref, "plain fwd + bwd_tmin")
    assert ref[4].abs().max() > 0 and ref[5].abs().max() > 0


# ---- (2) the forward at t_min > 0 ------------------------------------------------------------------------------------------------
FWD = [("s256", 1e-3), ("seeded", 1e-4)]


def _fwd_case(name, D=256):
    if name == "seeded":
        flat, c2w, cam, kw, gs = _case(1000, 128, D, seed=3)
        return flat, c2w, cam, kw, gs
    P, inp, flags, D = FL.planted(name)
    return (FL._cu(O.flatten_params(P)), FL._cu(inp["c2w"]), FL._cu(inp["cam"]), FL._call_kw(inp, flags, D),
            (FL._cu(inp["g_rgb"]), FL._cu(inp["g_dp"]), FL._cu(inp["g_dg"])))


@pytest.mark.parametrize("name,t", FWD)
def test_forward_at_t_min(name, t):
    from nope_nerf_b200 import ops
    flat, c2w, cam, kw, gs = _fwd_case(name)
    N, S = kw["N"], kw["S"]
    call = ops.frame_render_call(t)(flat, c2w, cam, engine=None, **kw)
    call.release()
    *outs, n_eval, t_final = ops.render_frame(flat, c2w, cam, engine=None, t_min=t, want_stats=True, **kw)
    torch.cuda.synchronize()
    _equal([call.rgb, call.depth_pred, call.depth_gt, call.mask, call.n_eval], outs + [n_eval], "forward vs render_frame")
    print(name, "t_min", t, "rays per n_eval:", dict(zip(*[x.tolist() for x in torch.unique(n_eval, return_counts=True)])))
    # with noise: rays that never stop keep the t = 0 bits; stopped rays within the bound of the t = 0 output
    nz = _noise(kw, 9)
    c0 = ops.FrameRenderCall(flat, c2w, cam, engine=None, noise=nz, **kw); c0.release()
    ct = ops.frame_render_call(t)(flat, c2w, cam, engine=None, noise=nz, **kw); ct.release()
    torch.cuda.synchronize()
    live = ct.n_eval == S
    assert torch.equal(ct.rgb[live], c0.rgb[live]) and torch.equal(ct.depth_pred[live], c0.depth_pred[live])
    if (~live).any():
        d = (ct.rgb[~live] - c0.rgb[~live]).abs().max()
        assert d <= 1.002 * t + 1e-6, (float(d), t)


# ---- (3) gradients against float64 of the truncated render ----------------------------------------------------------------------
def truncated_reference(P, inp, flags, gates, s_gate, mask, dev="cuda"):
    """float64 autograd of the render with every sample where mask == 0 given zero opacity (the truncated render; no dist_alpha, whose
    last sample is opaque by definition).  Returns (outputs, gradients, wrong answers {name: gradients})."""
    N, S = inp["N"], inp["S"]
    M = N * S
    A = RL.Arith()
    t64 = lambda x: torch.as_tensor(np.asarray(x, np.float64), device=dev)
    Wt = {k: t64(v).requires_grad_(True) for k, v in P.items()}
    c2w, cam = t64(inp["c2w"]).requires_grad_(True), t64(inp["cam"]).requires_grad_(True)
    q_in = dict(N=N, S=S, H=FL.H, W=FL.W, near=inp["near"], far=inp["far"], c2w=c2w, cam=cam, ray_idx=inp["ray_idx"])
    sc, sf = t64(inp["scale"]).requires_grad_(True), t64(inp["shift"]).requires_grad_(True)
    q_in.update(raw=inp["raw"], raw_rint=inp["raw"], scale=sc, shift=sf)
    leaves = dict(Wt, g_c2w=c2w, g_cam=cam, g_scale=sc, g_shift=sf)
    p, z, v, _ = RL.ray_stage(A, RL._rowq(A, q_in, (N, S), dev), flags, S, None)
    rgb_s, a_s = FL.field_ref(Wt, p.reshape(M, 3), v.reshape(M, 3), gates, s_gate, flags)
    q = RL._rowq(A, q_in, (N,), dev)
    ray = RL._ray_scalars(RL.setup_ray(A, q, flags), q)
    seeds = {k: t64(inp[k]) for k in ("g_rgb", "g_dp", "g_dg")}
    names = list(leaves)

    def render(m):
        rec = dict(r=rgb_s[:, 0].reshape(N, S), g=rgb_s[:, 1].reshape(N, S), b=rgb_s[:, 2].reshape(N, S), a=a_s.reshape(N, S) * m, z=z)
        _, rgb, dp, dg = RL.composite_fwd_ref(A, rec, ray, flags)
        loss = (seeds["g_rgb"] * rgb).sum() + (seeds["g_dp"] * dp).sum() + (seeds["g_dg"] * dg).sum()
        return dict(rgb=rgb.detach(), depth_pred=dp.detach(), depth_gt=dg.detach()), loss

    def grads(loss):
        g = torch.autograd.grad(loss, [leaves[k] for k in names] + [rgb_s, a_s], retain_graph=True, allow_unused=True)
        G = {k: (torch.zeros_like(leaves[k]) if x is None else x) for k, x in zip(names, g)}
        return FL._grad_tensors(G), g[len(names):]

    outs, loss = render(mask)
    G, _ = grads(loss)
    _, loss_full = render(torch.ones_like(mask))
    G_full, (g_rgb_full, g_a_full) = grads(loss_full)
    mrow = mask.reshape(M)
    pb = torch.autograd.grad([rgb_s, a_s], [Wt[k] for k in P], [g_rgb_full * mrow[:, None], g_a_full * mrow], retain_graph=True,
                             allow_unused=True)
    G_suffix = dict(G, **{k: (torch.zeros_like(Wt[k]) if x is None else x) for k, x in zip(P, pb)})
    return outs, G, dict(untruncated=G_full, suffix_from_last_chunk=G_suffix)


def _tmin_grads(P, inp, flags, D, t):
    """the _tmin pair in a workspace filled with 0x7E (large floats), so that a value the pair reads without writing it first (a stale
    suffix carry or lane partial of a ray outside a round's list) shows in its gradients"""
    from nope_nerf_b200 import ops
    ops._pool.free.clear()
    ops._pool.give(torch.full((L.lib.nnb_render_frame_bwd_workspace_bytes(inp["N"], inp["S"], D),), 0x7E, dtype=torch.uint8, device="cuda"))
    cls = ops.frame_render_call(t)
    call = cls(FL._cu(O.flatten_params(P)), FL._cu(inp["c2w"]), FL._cu(inp["cam"]), engine=None, **FL._call_kw(inp, flags, D))
    outs = (call.rgb.clone(), call.depth_pred.clone(), call.depth_gt.clone())
    n_eval = call.n_eval.clone()
    g = FL._grads(D, inp["N"])
    call.backward(FL._cu(inp["g_rgb"]), FL._cu(inp["g_dp"]), FL._cu(inp["g_dg"]), g["w"], g["g_c2w"], g["g_cam"], None, g["g_scale_shift"])
    torch.cuda.synchronize()
    return FL._got(outs, g, D, False), n_eval


GRAD = [("s256", 1e-3, "scattered"), ("t100", 1.0, "round0"), ("t100-relu", 1.0, "round0")]


@pytest.mark.parametrize("name,t,kind", GRAD)
def test_gradients_against_float64_truncated(name, t, kind):
    P, inp, flags, D = FL.planted(name)
    N, S = inp["N"], inp["S"]
    C = (S + 31) // 32
    assert not flags & L.DIST_ALPHA
    got, n_eval = _tmin_grads(P, inp, flags, D, t)
    stop_round = ((n_eval + 31) // 32 - 1).cpu().numpy()
    if kind == "scattered":
        assert len(set(stop_round[stop_round < C - 1].tolist())) >= 4, np.bincount(stop_round)
    else:
        assert (n_eval == 32).all(), "every ray stops in round 0"
    st = FL.stash_run(P, inp, flags, D, "tc", noise=False)
    s_gate = (st["rec"][:, 4] > 0).double()
    gates = [g.double() for g in st["gates"]]
    mask = (torch.arange(S, device="cuda")[None, :] < n_eval[:, None]).double()
    outs, G, wrong = truncated_reference(P, inp, flags, gates, s_gate, mask)
    ref = dict(outs, **G)
    err = FL.compare(got, ref)
    gate = FL.E2E_GATES["scattered"]["tc"]
    worst = max(err.items(), key=lambda kv: kv[1])
    teeth = {}
    for bug, Gw in wrong.items():
        teeth[bug] = max(float((got[k].double() - Gw[k]).abs().max()) / max(float(ref[k].abs().max()), 1e-300) for k in G)
    print(name, "t_min", t, "rays per stop round", np.bincount(stop_round, minlength=C), "worst", worst, "gate", gate, "wrong", teeth)
    assert worst[1] <= gate, (worst, gate)
    for bug, sc in teeth.items():
        assert sc > gate, (bug, sc, gate)


# ---- (4) zero cotangent on stopped rays -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 128, 256])
def test_stopped_rays_with_zero_cotangent(D):
    from nope_nerf_b200 import ops
    name = {64: "t100-d64", 128: "t100-d128", 256: "s256"}[D]
    P, inp, flags, D = FL.planted(name)
    flat, c2w, cam, kw = FL._cu(O.flatten_params(P)), FL._cu(inp["c2w"]), FL._cu(inp["cam"]), FL._call_kw(inp, flags, D)
    # a t_min that leaves a mix of stopped and live rays: 1e-3 on the scattered plant, bisected on the translucent ones (t_min = 0 stops
    # no ray, t_min = 1 every ray after chunk 0)
    def live_at(t):
        probe = ops.frame_render_call(t)(flat, c2w, cam, engine=None, **kw); probe.release()
        torch.cuda.synchronize()
        return (probe.n_eval == inp["S"]).float()
    lo, hi = 0.0, 1.0
    t = 1e-3 if name == "s256" else 0.5
    for _ in range(30):
        live = live_at(t)
        if 0 < live.sum() < inp["N"] or name == "s256":
            break
        lo, hi = (t, hi) if live.sum() == inp["N"] else (lo, t)
        t = 0.5 * (lo + hi)
    assert 0 < live.sum() < inp["N"], "a mix of stopped and live rays"
    gs = (FL._cu(inp["g_rgb"]) * live[:, None], FL._cu(inp["g_dp"]) * live, FL._cu(inp["g_dg"]) * live)
    ref, _ = _pair(ops.FrameRenderCall, flat, c2w, cam, kw, gs)
    got, _ = _pair(ops.frame_render_call(t), flat, c2w, cam, kw, gs)
    from nope_nerf_b200.model.official_nerf import param_slices
    worst = 0.0
    for (o, n, shape) in param_slices(D):
        r = ref[4][o:o + n]
        if r.abs().max() == 0:
            continue
        worst = max(worst, _rel(got[4][o:o + n], r))
    e_pose = _rel(got[5], ref[5])
    print(name, "D", D, "zero cotangent on stopped rays: worst dW %.2e, g_c2w %.2e" % (worst, e_pose))
    assert worst <= 1e-5 and e_pose <= 1e-5, (worst, e_pose)


# ---- (5) determinism, workspace state, graph replay -----------------------------------------------------------------------------
def test_repeated_and_workspace_independent():
    from nope_nerf_b200 import ops
    P, inp, flags, D = FL.planted("s256")
    flat, c2w, cam, kw = FL._cu(O.flatten_params(P)), FL._cu(inp["c2w"]), FL._cu(inp["cam"]), FL._call_kw(inp, flags, D)
    gs = (FL._cu(inp["g_rgb"]), FL._cu(inp["g_dp"]), FL._cu(inp["g_dg"]))
    nz = FL._cu(inp["noise"])
    cls = ops.frame_render_call(1e-3)
    ref, n0 = _pair(cls, flat, c2w, cam, kw, gs, nz)
    assert (n0 < inp["S"]).any()
    for _ in range(2):
        _equal(_pair(cls, flat, c2w, cam, kw, gs, nz)[0], ref, "repeat")
    nbytes = L.lib.nnb_render_frame_bwd_workspace_bytes(kw["N"], kw["S"], D)
    for fill in (0x00, 0xFF, 0x7E):
        ops._pool.free.clear()
        ops._pool.give(torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda"))
        _equal(_pair(cls, flat, c2w, cam, kw, gs, nz)[0], ref, fill)
    ops._pool.free.clear()


def test_graph_replay_after_weights_change():
    from nope_nerf_b200 import ops
    P, inp, flags, D = FL.planted("s256")
    c2w, cam, kw = FL._cu(inp["c2w"]), FL._cu(inp["cam"]), FL._call_kw(inp, flags, D)
    gs = (FL._cu(inp["g_rgb"]), FL._cu(inp["g_dp"]), FL._cu(inp["g_dg"]))
    nz = FL._cu(inp["noise"])
    cls = ops.frame_render_call(1e-3)
    w_a = FL._cu(O.flatten_params(P))
    P_b = dict(P); P_b["fc_density.bias"] = P["fc_density.bias"] - np.float32(1.5)   # fewer rays stop, later
    w_b = FL._cu(O.flatten_params(P_b))
    ref_a, n_a = _pair(cls, w_a, c2w, cam, kw, gs, nz)                  # eager: also the one-time set-up
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


# ---- (6) Trainer --------------------------------------------------------------------------------------------------------------------
def test_trainer_t_min_zero_is_frame_grad(monkeypatch):
    opts = dict(full=True)
    a = GO._run(opts, "graph", monkeypatch, steps=5, frame_grad=True)
    b = GO._run(opts, "graph", monkeypatch, steps=5, frame_grad=True, frame_grad_t_min=0.0)
    assert b["tr"]._train_render_call(True).t_min == 0.0
    for k in ("losses", "w", "r", "t", "scales", "shifts"):
        assert a[k].tobytes() == b[k].tobytes(), (k, np.abs(a[k] - b[k]).max())


def test_trainer_t_min_graph_equals_eager(monkeypatch):
    opts = dict(full=True)
    ge = GO._run(opts, "eager", monkeypatch, steps=5, frame_grad=True, frame_grad_t_min=1e-4)
    gg = GO._run(opts, "graph", monkeypatch, steps=5, frame_grad=True, frame_grad_t_min=1e-4)
    assert len(gg["gsteps"]) == 1 and gg["gsteps"][0].graph is not None and gg["gsteps"][0].calls == 5
    for k in ("losses", "w", "r", "t", "scales", "shifts"):
        assert ge[k].tobytes() == gg[k].tobytes(), (k, np.abs(ge[k] - gg[k]).max())

"""GPU: the tensor-core second-order field backward (nnb_field_hvp_tc: tc_points_vjp_fwd, tc_points_hvp, tc_points_tangent and the
weight-gradient stage of csrc/nnb_tc.cu) and its Python path (field.field_normal / OfficialStaticNerf.gradient_grad with engine='tc',
grad_engine='tc', Renderer(normal_engine='tc', normal_grad_engine='tc')).

For a cotangent u on the normals n = d s / d p of the density logit s, the call returns d(u . n)/d p and d(u . n)/d weights.  Checks:
- the normals under autograd are the detached gradient(engine='tc') normals, bit for bit, and a third derivative raises;
- g_pts and every dW against float64 torch double backward of the logit, evaluated with the ReLU gates this call's forward wrote (read
  from its workspace), within TOL of each tensor's maximum; every bias slot and every colour slot of g_weights is left as it was;
- with u restricted to the rows both engines gate alike, agreement with the exact engine's nnb_field_hvp within the same bounds;
- a point's g_pts depends on that point alone (permuted, split into uneven calls), repeated calls give the same bits, and a workspace of
  zeros, NaN bytes or 0x7E7E7E7E words gives the same bits;
- every error code, with nothing launched;
- the C2-shaped Renderer.nope_nerf with normal_loss on this path: finite MLP and pose gradients, which agree with the exact engine's
  renderer when the loss weights only the rays whose surface points both engines gate alike.

Largest measured (NVIDIA H100 80GB HBM3, 700 W power limit), relative to the tensor's maximum at D = 64 / 128 / 256: every dW against
float64 2.2e-5 / 3.6e-5 / 7.9e-5, g_pts 1.7e-5 / 1.2e-5 / 1.1e-5 (1.2e-5 / 8.9e-6 / 7.5e-6 for the calls of 1 and 127 points); against
nnb_field_hvp on the rows both engines gate alike 2.1e-5 / 3.7e-5 / 7.9e-5; the C2 renderer's MLP and pose gradients against the exact
engine's 4.7e-5.  Run with -s to print them per case.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
from test_gpu_field_grad_tc import grad_gates, param_slices, COLOUR, _net
from test_gpu_field_hvp import logit, TRUNK
from test_gpu_relu_mask import layout
from test_gpu_field_vjp import relmax, bits

pytestmark = pytest.mark.gpu

TOL = 1e-4
SIZES = (1, 127, 128, 129, 4097, 131072)
WEIGHTS = {"%s.%d.weight" % t for t in TRUNK} | {"fc_density.weight"}


def _lib():
    from nope_nerf_b200 import _lib as L, ops
    return L, ops


def hvp_tc(flat, D, p, u, ws=None, gp=None, gw=None, want_p=True, want_w=True, ws_bytes=None, flags=None, engine=None):
    """one nnb_field_hvp_tc call; u (M, 3) or (M, 4).  Returns (rc, g_pts (M, 4) | None, g_weights | None, workspace)"""
    L, ops = _lib()
    M = p.shape[0]
    if ws is None:
        ws = torch.empty(max(L.lib.nnb_field_hvp_tc_workspace_bytes(M, 0, D), 256), dtype=torch.uint8, device="cuda")
    u4 = u if u.shape[-1] == 4 else torch.cat([u, torch.zeros(M, 1, device="cuda")], 1).contiguous()
    if gp is None and want_p:
        gp = torch.full((M, 4), float("nan"), device="cuda")
    if gw is None and want_w:
        gw = torch.zeros(L.num_params(D), device="cuda")
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p); a.dirs = None; a.N = M; a.S = 1; a.flags = 0 if flags is None else flags
    a.engine = L.ENGINE_TC if engine is None else engine; a.hidden_dim = D
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel() if ws_bytes is None else ws_bytes
    rc = L.lib.nnb_field_hvp_tc(C.byref(a), L.ptr(u4), L.ptr(gp), L.ptr(gw), ops._stream())
    torch.cuda.synchronize()
    return rc, gp, gw, ws


def hvp_exact(flat, D, p, u):
    """nnb_field_hvp (exact engine): (g_pts (M, 4), g_weights, the forward's h > 0 per trunk layer)"""
    L, ops = _lib()
    M = p.shape[0]
    flags = L.STASH | L.HVP | L.RAW_DENSITY
    ws = torch.empty(L.lib.nnb_workspace_bytes_dim(M, 1, flags, L.ENGINE_SIMT, D), dtype=torch.uint8, device="cuda")
    u4 = torch.cat([u, torch.zeros(M, 1, device="cuda")], 1).contiguous()
    gp = torch.empty(M, 4, device="cuda"); gw = torch.zeros(L.num_params(D), device="cuda")
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p); a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_SIMT; a.hidden_dim = D
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    L.check(L.lib.nnb_field_hvp(C.byref(a), L.ptr(u4), L.ptr(gp), L.ptr(gw), ops._stream()), "nnb_field_hvp")
    torch.cuda.synchronize()
    lay = layout(M, 1, D)
    masks = [ws[o:o + lay["Mpad"] * D * 4].view(torch.float32).view(lay["Mpad"], D)[:M] > 0 for o in lay["h"]]
    return gp, gw, masks


def make_inputs(D, M, seed):
    """hf_damp weights, points in [-1.5, 1.5]^3, u ~ N(0, 1) with every 7th row zero"""
    rng = np.random.default_rng(seed)
    P = O.init_params(seed=11 + D, D=D, hf_damp=True)
    p = rng.uniform(-1.5, 1.5, (M, 3)).astype(np.float32)
    u = rng.normal(size=(M, 3)).astype(np.float32)
    u[::7] = 0.0
    flat = torch.from_numpy(O.flatten_params(P)).cuda()
    return flat, torch.from_numpy(p).cuda(), torch.from_numpy(u).cuda()


def double_backward64(flat, D, p, u, gates):
    """float64 d(u . d s / d p)/d (p, W) of the logit with each ReLU replaced by the given gates (bool (M, D) per trunk layer)"""
    W = {n: flat[o:o + k].double().view(s).clone().requires_grad_(True) for n, o, k, s in param_slices(D)}
    p64 = p.double().clone().requires_grad_(True)
    s = logit(W, p64, [g.double() for g in gates])
    n, = torch.autograd.grad(s.sum(), p64, create_graph=True)
    names = list(W)
    grads = torch.autograd.grad((n * u.double()).sum(), [p64] + [W[k] for k in names], allow_unused=True)
    return grads[0], {k: (torch.zeros_like(W[k]) if g is None else g) for k, g in zip(names, grads[1:])}


@pytest.mark.parametrize("D", [64, 128, 256])
def test_float64_and_exact_engine(D):
    """g_pts and every dW against float64 with this call's gates; bias and colour slots untouched; agreement with nnb_field_hvp where
    both engines gate a row alike"""
    L, _ = _lib()
    worst = {}
    for M in SIZES:
        flat, p, u = make_inputs(D, M, seed=500 + M)
        sentinel = torch.randn(L.num_params(D), device="cuda", generator=torch.Generator("cuda").manual_seed(M))
        rc, gp, gw, ws = hvp_tc(flat, D, p, u)
        assert rc == 0, L.lib.nnb_last_error()
        rc, _, gw_sent, _ = hvp_tc(flat, D, p, u, gw=sentinel.clone(), want_p=False)
        assert rc == 0
        assert torch.isfinite(gp).all() and (gp[:, 3] == 0).all() and (gp[::7, :3] == 0).all()
        gates = grad_gates(ws, M, D, True)
        ref_p, ref_w = double_backward64(flat, D, p, u, gates)
        e = {"g_pts": relmax(gp[:, :3].cpu().numpy(), ref_p.cpu().numpy())}
        for n, o, k, s in param_slices(D):
            if n in WEIGHTS:
                e[n] = relmax(gw[o:o + k].cpu().numpy(), ref_w[n].reshape(-1).cpu().numpy())
            else:   # no bias term and no colour term: the slot keeps its bits
                assert torch.equal(bits(gw_sent[o:o + k]), bits(sentinel[o:o + k])), n
                assert float(ref_w[n].abs().max()) == 0.0, n
        # the exact engine, with u on the rows both engines gate alike
        _, _, masks = hvp_exact(flat, D, p, torch.zeros_like(u))
        same = torch.stack([(a_ == b_).all(1) for a_, b_ in zip(gates, masks)]).all(0)
        u_same = u * same[:, None]
        gp_s, gw_s, _ = hvp_exact(flat, D, p, u_same)
        rc, gp_t, gw_t, _ = hvp_tc(flat, D, p, u_same)
        assert rc == 0
        e["g_pts_exact"] = relmax(gp_t[:, :3].cpu().numpy(), gp_s[:, :3].double().cpu().numpy())
        for n, o, k, s in param_slices(D):
            if n in WEIGHTS:
                e["x:" + n] = relmax(gw_t[o:o + k].cpu().numpy(), gw_s[o:o + k].double().cpu().numpy())
        bad = {k: v for k, v in e.items() if v > TOL}
        assert not bad, (D, M, bad)
        summary = dict(g_pts=e["g_pts"], weights=max(v for k, v in e.items() if k in WEIGHTS),
                       exact=max(v for k, v in e.items() if k == "g_pts_exact" or k.startswith("x:")),
                       rows_gates_differ=float(1.0 - same.float().mean()))
        if M < 128:
            summary["g_pts_below_128_rows"] = summary.pop("g_pts")
        for k, v in summary.items():
            worst[k] = max(worst.get(k, 0.0), v)
    print("field_hvp_tc D=%d: %s" % (D, " ".join("%s %.2e" % kv for kv in sorted(worst.items()))))


@pytest.mark.parametrize("D", [64, 128, 256])
def test_row_independence_determinism_and_poison(D):
    """g_pts of a row is the same bits permuted, split into uneven calls, repeated, or with a poisoned workspace; g_weights repeats bit
    for bit and does not depend on what the workspace held"""
    L, _ = _lib()
    M = 4097
    flat, p, u = make_inputs(D, M, seed=77)
    rc, gp, gw, _ = hvp_tc(flat, D, p, u)
    assert rc == 0, L.lib.nnb_last_error()
    rc, gp2, gw2, _ = hvp_tc(flat, D, p, u)
    assert rc == 0 and torch.equal(bits(gp), bits(gp2)) and torch.equal(bits(gw), bits(gw2))
    perm = torch.randperm(M, generator=torch.Generator().manual_seed(3)).cuda()
    rc, gpp, _, _ = hvp_tc(flat, D, p[perm].contiguous(), u[perm].contiguous(), want_w=False)
    assert rc == 0 and torch.equal(bits(gpp), bits(gp[perm]))
    for a0, b0 in ((0, 1), (1, 130), (130, 1000), (1000, M)):
        rc, gpc, _, _ = hvp_tc(flat, D, p[a0:b0].contiguous(), u[a0:b0].contiguous(), want_w=False)
        assert rc == 0 and torch.equal(bits(gpc), bits(gp[a0:b0])), (a0, b0)
    need = L.lib.nnb_field_hvp_tc_workspace_bytes(M, 0, D)
    for fill in (0x00, 0xFF, 0x7E):
        ws = torch.full((need,), fill, dtype=torch.uint8, device="cuda")
        rc, gpf, gwf, _ = hvp_tc(flat, D, p, u, ws=ws)
        assert rc == 0 and torch.equal(bits(gpf), bits(gp)) and torch.equal(bits(gwf), bits(gw)), fill
    # g_weights accumulates, and each output is optional
    x0 = torch.randn(L.num_params(D), device="cuda", generator=torch.Generator("cuda").manual_seed(5))
    rc, _, gwa, _ = hvp_tc(flat, D, p, u, gw=x0.clone())
    assert rc == 0 and torch.equal(bits(gwa), bits(x0 + gw))
    rc, gpo, gwo, _ = hvp_tc(flat, D, p, u, want_w=False)
    assert rc == 0 and gwo is None and torch.equal(bits(gpo), bits(gp))
    rc, gpo, gwo, _ = hvp_tc(flat, D, p, u, want_p=False)
    assert rc == 0 and gpo is None and torch.equal(bits(gwo), bits(gw))


def test_error_paths():
    """each rejected call launches nothing (g_pts keeps its NaNs, g_weights its sentinel)"""
    L, ops = _lib()
    D, M = 64, 100
    flat, p, u = make_inputs(D, M, seed=41)
    u4 = torch.cat([u, torch.zeros(M, 1, device="cuda")], 1).contiguous()
    err = lambda: L.lib.nnb_last_error().decode()
    need = L.lib.nnb_field_hvp_tc_workspace_bytes(M, 0, D)
    ws = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    gp = torch.full((M + 8, 4), float("nan"), device="cuda")
    gw = torch.full((L.num_params(D) + 8,), -7.0, device="cuda")
    untouched = lambda: bool(torch.isnan(gp).all() and (gw == -7.0).all())
    cases = [
        (dict(engine=L.ENGINE_SIMT), -4, "engine"),
        (dict(flags=1 << 16), -7, "not defined"),
        (dict(flags=L.STASH), -6, "NNB_STASH"),
        (dict(flags=L.HVP), -6, "NNB_HVP"),
        (dict(D=96), -8, "hidden_dim"),
        (dict(N=-1), -3, "negative"),
        (dict(ws_bytes=need - 1), -5, "too small"),
        (dict(ws=ws[16:], ws_bytes=need), -5, "aligned"),
        (dict(p=None), -3, "pts"),
        (dict(flat=None), -3, "weights"),
        (dict(u=None), -3, "u"),
        (dict(gp=None, gw=None), -3, "g_pts, g_weights"),
        (dict(gp=gp.view(-1)[1:1 + 4 * M].view(M, 4)), -3, "aligned"),
        (dict(u=u4.view(-1)[1:1 + 4 * (M - 1)].view(M - 1, 4)), -3, "aligned"),
        (dict(gw_off=2), -3, "g_weights"),
    ]
    for kw, code, word in cases:
        a = L.RenderArgs()
        a.weights = L.ptr(kw["flat"]) if "flat" in kw else L.ptr(flat)
        a.pts = L.ptr(kw["p"]) if "p" in kw else L.ptr(p)
        a.N = kw.get("N", M); a.S = 1; a.flags = kw.get("flags", 0); a.engine = kw.get("engine", L.ENGINE_TC); a.hidden_dim = kw.get("D", D)
        w_ = kw.get("ws", ws)
        a.workspace = L.ptr(w_); a.workspace_bytes = kw.get("ws_bytes", w_.numel())
        gw_ptr = (L.ptr(gw) + kw.get("gw_off", 0)) if kw.get("gw", gw) is not None else None
        rc = L.lib.nnb_field_hvp_tc(C.byref(a), L.ptr(kw["u"]) if "u" in kw else L.ptr(u4),
                                    L.ptr(kw["gp"]) if "gp" in kw else L.ptr(gp), gw_ptr, ops._stream())
        torch.cuda.synchronize()
        assert rc == code and word in err() and untouched(), (kw.keys(), rc, code, err())
    rc, *_ = hvp_tc(flat, D, p[:0], u[:0], ws=ws, gp=gp, gw=gw)
    assert rc == 0 and untouched()
    rc, *_ = hvp_tc(flat, D, p, u4, ws=ws, gp=gp, gw=gw)
    assert rc == 0 and bool(torch.isfinite(gp[:M]).all()), err()
    assert bool((gw[L.num_params(D):] == -7.0).all()) and bool(torch.isnan(gp[M:]).all())


def _nodes(t):
    """names of the autograd nodes behind t"""
    names, stack = set(), [t.grad_fn]
    while stack:
        f = stack.pop()
        if f is not None:
            names.add(type(f).__name__)
            stack += [x[0] for x in f.next_functions]
    return names


@pytest.mark.parametrize("D", [64, 128, 256])
def test_python_path(D):
    """gradient_grad(p, engine='tc', grad_engine='tc'): the normals are gradient(engine='tc')'s bits; the gradients in p and every
    parameter are nnb_field_hvp_tc's with the cotangent on -n; a third derivative raises"""
    L, _ = _lib()
    net = _net(D)
    M = 5000
    gen = torch.Generator().manual_seed(4)
    p0 = (torch.rand(M, 3, generator=gen) * 3 - 1.5).cuda()
    w = torch.randn(M, 3, generator=gen).cuda()
    p = p0.clone().requires_grad_(True)
    net.zero_grad(set_to_none=True)
    n = net.gradient_grad(p, 0, engine="tc", grad_engine="tc")
    with torch.no_grad():
        n_det = net.gradient(p0, 0, engine="tc")
    assert n.grad_fn is not None and torch.equal(bits(n), bits(n_det))
    (n[:, 0, :] * w).sum().backward()
    rc, gp_ref, gw_ref, _ = hvp_tc(net.flat_weights(), D, p0, -w)
    assert rc == 0
    assert torch.equal(bits(p.grad), bits(gp_ref[:, :3].contiguous()))
    for name, q, (o, k, s) in zip([n_ for n_, _ in net.named_parameters()], net.parameters(), net.param_slices):
        if name in WEIGHTS:
            assert torch.equal(bits(q.grad.reshape(-1)), bits(gw_ref[o:o + k])), name
        else:
            assert q.grad is None or not q.grad.any(), name
    # the default keeps the exact engine's second-order backward
    p = p0.clone().requires_grad_(True)
    assert "_GradTcFnBackward" in _nodes(n) and "_GradFnBackward" not in _nodes(n)
    assert "_GradFnBackward" in _nodes(net.gradient(p, 0, engine="tc")) and "_GradFnBackward" in _nodes(net.gradient_grad(p, 0, engine="tc"))
    # a third derivative raises, as on the exact engine
    p = p0[:300].clone().requires_grad_(True)
    g, = torch.autograd.grad(net.gradient_grad(p, 0, engine="tc", grad_engine="tc").sum(), p, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()


def _renderer_run(cfg, net, grad_engine, wts_fn, pp_log):
    """C2-shaped Renderer.nope_nerf with normal_loss; loss = sum(wts * out['normal']^2); returns (loss inputs, MLP and pose gradients)"""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    kw = dict(normal_engine="tc", normal_grad_engine="tc") if grad_engine == "tc" else {}
    rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), **kw)
    N, S = 1024, int(cfg["rendering"]["num_points"])
    gen = torch.Generator().manual_seed(9)
    H, W = 240, 320
    pix = torch.stack([torch.randint(0, W, (N,), generator=gen), torch.randint(0, H, (N,), generator=gen)], -1).float()
    pix = torch.stack([2 * pix[:, 0] / W - 1, 2 * pix[:, 1] / H - 1], -1).cuda()
    r = (torch.randn(1, 3, generator=gen) * 0.05).cuda().requires_grad_(True)
    t = (torch.randn(1, 3, generator=gen) * 0.05).cuda().requires_grad_(True)
    c2w = ops.pose_c2w(r, t, None, 0)
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], device="cuda").view(1, 4, 4)
    depth = (torch.rand(N, generator=gen) * 2 + 0.5).cuda()
    orig_g, orig_gg = net.gradient, net.gradient_grad
    pp_grad = []

    def log(pp):   # the surface points and, after the backward, the loss's gradient in them
        pp_log.append(pp.detach().clone())
        pp.register_hook(lambda g_: pp_grad.append(g_.detach().clone()))
    net.gradient = lambda pp, it, *a, **k: (log(pp), orig_g(pp, it, *a, **k))[1]
    net.gradient_grad = lambda pp, it, *a, **k: (log(pp), orig_gg(pp, it, *a, **k))[1]
    try:
        net.zero_grad(set_to_none=True)
        torch.manual_seed(123)   # the same neighbour offsets on both engines
        out = rend.nope_nerf(pix[None], depth, cam, None, None, add_noise=False, it=0, c2w=c2w)
    finally:
        del net.gradient, net.gradient_grad
    dn = out["normal"]
    (wts_fn(dn) * dn ** 2).sum().backward()
    grads = {n_: (torch.zeros_like(q) if q.grad is None else q.grad.clone()) for n_, q in net.named_parameters()}
    grads["pose_r"], grads["pose_t"] = r.grad.clone(), t.grad.clone()
    # the pose gradients sum the points' gradients, which largely cancel: their scale is the sum of the terms' magnitudes
    gpp, pp = pp_grad[0], pp_log[-1]
    scale = {"pose_t": float(gpp.abs().sum()), "pose_r": float((gpp.norm(dim=1) * pp.norm(dim=1)).sum())}
    return dn.detach(), grads, scale


def test_renderer_normal_loss_c2():
    """Renderer(normal_engine='tc', normal_grad_engine='tc').nope_nerf with normal_loss at N = 1024, S = 128, D = 256: forward and
    backward run, the MLP and pose gradients of a loss on out['normal'] are finite, and with the loss weighted to the rays whose two
    surface points both engines gate alike they agree with the exact engine's renderer within TOL: each MLP gradient relative to its
    tensor's maximum, each pose gradient relative to the summed magnitudes of the per-point terms it adds up"""
    from _cfg import default_cfg
    import nope_nerf_b200.model as mdl
    L, _ = _lib()
    cfg = default_cfg()
    cfg["model"]["hidden_dim"] = 256
    cfg["rendering"]["normal_loss"] = True
    cfg["rendering"]["num_points"] = 128
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=61, D=256, hf_damp=True).items()})
    net = net.cuda()
    log = []
    dn_t, g_t, _ = _renderer_run(cfg, net, "tc", lambda dn: torch.ones_like(dn), log)
    assert len(log) == 1 and dn_t.numel() > 0 and torch.isfinite(dn_t).all()
    for k, v in g_t.items():
        assert torch.isfinite(v).all(), k
    assert g_t["layers0.0.weight"].abs().max() > 0 and g_t["pose_r"].abs().max() > 0
    # the rays whose two surface points both engines gate alike
    pp = log[0]
    Nv = pp.shape[0] // 2
    _, _, _, ws = hvp_tc(net.flat_weights(), 256, pp.contiguous(), torch.zeros_like(pp), want_p=False)
    g_tc = grad_gates(ws, pp.shape[0], 256, True)
    _, _, masks = hvp_exact(net.flat_weights(), 256, pp.contiguous(), torch.zeros_like(pp))
    same = torch.stack([(a_ == b_).all(1) for a_, b_ in zip(g_tc, masks)]).all(0)
    ray_same = (same[:Nv] & same[Nv:]).float()
    _, g_t, _ = _renderer_run(cfg, net, "tc", lambda dn: ray_same, [])
    _, g_s, scale = _renderer_run(cfg, net, None, lambda dn: ray_same, [])
    e = {k: relmax(g_t[k].cpu().numpy(), g_s[k].double().cpu().numpy()) for k in g_s if k not in scale and float(g_s[k].abs().max()) > 0}
    for k, sc in scale.items():
        e[k] = float((g_t[k] - g_s[k]).abs().max()) / sc
    print("renderer normal_loss C2: rays %d, gated differently %d; largest relative difference %.2e (%s)"
          % (Nv, int(Nv - ray_same.sum()), max(e.values()), max(e, key=e.get)))
    assert max(e.values()) <= TOL, e

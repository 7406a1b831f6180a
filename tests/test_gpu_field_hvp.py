"""GPU: nnb_field_hvp (the second-order field backward behind OfficialStaticNerf.gradient's autograd) against float64, from the kernel's
own inputs.

For a cotangent u on n = d s / d p (s the density logit), the library returns d(u . n)/d p and d(u . n)/d weights.  The reference is
float64 torch double backward of a test-local restatement of infer_occ (official_nerf.py:60-67) at the fp32 points and weights, with
the kernel's own ReLU masks read from the workspace's stash (h_l > 0), so a gate that flips between fp32 and fp64 cannot enter.  The
same quantities are also spelled out explicitly (tangent chain, gated output gradients, the encoding's second derivative: DESIGN.md
§4) and must equal the double backward to float64 rounding.

Each element's error is normalised by its own operands: u_32 times the same sum with every operand replaced by its magnitude, propagated
through the chains (|W| products of |dy| and |x'|, f^2 |delta sin| + f^2 |delta cos| for the point term).  The data- and tangent-chain
errors feed the weight- and point-gradient sums; that magnitude scale bounds chains of 16 GEMMs of up to D + 63 terms, and the kernel stays
far inside it (largest normalised error 0.1 over all cases below), so the gate is 8.
"""
import ctypes as C
import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
from test_gpu_relu_mask import layout

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GATE = 8.0   # largest measured: 0.1 (D = 64 and 128, M = 1; NVIDIA H100 80GB HBM3, 700 W power limit)
TRUNK = [("layers0", 0), ("layers0", 2), ("layers0", 4), ("layers0", 6), ("layers1", 0), ("layers1", 2), ("layers1", 4), ("layers1", 6)]


def _align(x, a):
    return (x + a - 1) // a * a


def hvp_call(P, D, p, u, want_p=True, want_w=True):
    """one nnb_field_hvp call on its own workspace; returns (g_pts [M,3] | None, g_weights flat | None, workspace)"""
    from nope_nerf_b200 import _lib as L, ops
    M = p.shape[0]
    flat = torch.from_numpy(np.concatenate([np.asarray(P[n], np.float32).reshape(-1) for n, _ in O.param_shapes(D)])).cuda()
    flags = L.STASH | L.HVP | L.SOFTPLUS
    nbytes = L.lib.nnb_workspace_bytes_dim(M, 1, flags, L.ENGINE_SIMT, D)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    p_c = torch.from_numpy(np.ascontiguousarray(p, np.float32)).cuda()
    u4 = torch.zeros(M, 4, device="cuda"); u4[:, :3] = torch.from_numpy(u.astype(np.float32)).cuda()
    g_p = torch.full((M, 4), float("nan"), device="cuda") if want_p else None
    g_w = torch.zeros(flat.numel(), device="cuda") if want_w else None
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p_c); a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_SIMT; a.hidden_dim = D
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    L.check(L.lib.nnb_field_hvp(C.byref(a), L.ptr(u4), L.ptr(g_p), L.ptr(g_w), ops._stream()), "nnb_field_hvp")
    torch.cuda.synchronize()
    return (None if g_p is None else g_p[:, :3].clone()), (None if g_w is None else g_w.clone()), ws


def stash_masks(ws, M, D):
    """the forward's h_l > 0 for l = 0..7 (SIMT layout of make_layout with NNB_STASH)"""
    lay = layout(M, 1, D)
    return [(ws[o:o + lay["Mpad"] * D * 4].view(torch.float32).view(lay["Mpad"], D)[:M] > 0).double() for o in lay["h"]]


def encode(p):
    out = [p]
    for i in range(10):
        out += [torch.sin(2.0 ** i * p), torch.cos(2.0 ** i * p)]
    return torch.cat(out, -1)


def logit(W, p, masks):
    """infer_occ with the ReLUs replaced by the fixed masks"""
    e = encode(p)
    x = e
    for l, (blk, i) in enumerate(TRUNK):
        if l == 4:
            x = torch.cat([x, e], -1)
        x = (x @ W["%s.%d.weight" % (blk, i)].T + W["%s.%d.bias" % (blk, i)]) * masks[l]
    return x @ W["fc_density.weight"].T + W["fc_density.bias"]


def explicit(W, p, u, masks, D):
    """the derivation of DESIGN.md §4 and its magnitude chains: values and scales of d s'/d p and d s'/d W_l, d s'/d w_sigma"""
    Ws = [W["%s.%d.weight" % t] for t in TRUNK]
    cols = [u]; acols = [u.abs()]
    for i in range(10):
        f = 2.0 ** i
        cols += [f * torch.cos(f * p) * u, -f * torch.sin(f * p) * u]
        acols += [(f * torch.cos(f * p) * u).abs(), (f * torch.sin(f * p) * u).abs()]
    ed, aed = torch.cat(cols, -1), torch.cat(acols, -1)
    xs, axs = [], []
    x, ax = ed, aed
    for l in range(8):
        if l == 4:
            x = torch.cat([x, ed], -1); ax = torch.cat([ax, aed], -1)
        xs.append(x); axs.append(ax)
        x = (x @ Ws[l].T) * masks[l]; ax = (ax @ Ws[l].abs().T) * masks[l]
    h7, ah7 = x, ax
    dy = [None] * 8; ady = [None] * 8
    g, ag = W["fc_density.weight"].expand(p.shape[0], D), W["fc_density.weight"].abs().expand(p.shape[0], D)
    denc = 0; adenc = 0
    for l in range(7, -1, -1):
        dy[l] = g * masks[l]; ady[l] = ag * masks[l]
        gin, agin = dy[l] @ Ws[l], ady[l] @ Ws[l].abs()
        if l == 4:
            denc = denc + gin[:, D:]; adenc = adenc + agin[:, D:]
        if l == 0:
            denc = denc + gin; adenc = adenc + agin
        g, ag = gin[:, :D], agin[:, :D]
    gp = torch.zeros_like(p); agp = torch.zeros_like(p)
    for i in range(10):
        f = 2.0 ** i
        ds, dc = denc[:, 3 + 6 * i:6 + 6 * i], denc[:, 6 + 6 * i:9 + 6 * i]
        ads, adc = adenc[:, 3 + 6 * i:6 + 6 * i], adenc[:, 6 + 6 * i:9 + 6 * i]
        gp = gp - f * f * (ds * torch.sin(f * p) + dc * torch.cos(f * p)) * u
        agp = agp + f * f * (ads * torch.sin(f * p).abs() + adc * torch.cos(f * p).abs()) * u.abs()
    gW = {("%s.%d.weight" % TRUNK[l]): (dy[l].T @ xs[l], ady[l].T @ axs[l]) for l in range(8)}
    gW["fc_density.weight"] = (h7.sum(0, keepdim=True), ah7.sum(0, keepdim=True))
    return gp, agp, gW


def nerr(got, ref, scale):
    d = (got - ref).abs()
    return float(torch.where(d == 0, torch.zeros_like(d), d / (U * scale).clamp_min(1e-300)).max())


def case(D, M, seed=3):
    rng = np.random.default_rng(seed + M + D)
    P = O.init_params(seed=seed, D=D)
    p = rng.uniform(-1.2, 1.2, (M, 3)).astype(np.float32)
    u = rng.normal(0, 1, (M, 3)).astype(np.float32)
    return P, p, u


@pytest.mark.parametrize("M", [1, 63, 64, 65, 2048, 5000])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_field_hvp_vs_float64(D, M):
    P, p, u = case(D, M)
    errs = {}
    for mode in ("p_and_w", "w_only", "p_only"):
        g_p, g_w, ws = hvp_call(P, D, p, u, want_p=mode != "w_only", want_w=mode != "p_only")
        masks = stash_masks(ws, M, D)
        W = {k: torch.from_numpy(np.asarray(v, np.float64)).cuda() for k, v in P.items()}
        for v in W.values():
            v.requires_grad_(True)
        p64 = torch.from_numpy(p.astype(np.float64)).cuda().requires_grad_(True)
        u64 = torch.from_numpy(u.astype(np.float64)).cuda()
        s = logit(W, p64, masks)
        n, = torch.autograd.grad(s.sum(), p64, create_graph=True)
        names = [k for k, _ in O.param_shapes(D)]
        grads = torch.autograd.grad((n * u64).sum(), [p64] + [W[k] for k in names], allow_unused=True)
        ref_p = grads[0]
        ref_w = {k: (torch.zeros_like(W[k]) if g is None else g) for k, g in zip(names, grads[1:])}
        with torch.no_grad():
            gp_x, agp, gW = explicit({k: v.detach() for k, v in W.items()}, p64.detach(), u64, masks, D)
        # the explicit derivation is the double backward (float64 rounding apart)
        assert nerr(gp_x, ref_p, agp) < 1e-3
        for k, (val, _) in gW.items():
            assert float((val - ref_w[k]).abs().max()) <= 1e-9 * max(float(ref_w[k].abs().max()), 1e-30), k
        if g_p is not None:
            assert torch.isfinite(g_p).all()
            errs[mode + ":p"] = nerr(g_p.double(), ref_p, agp)
        if g_w is not None:
            got = {k: torch.from_numpy(v.astype(np.float64)).cuda() for k, v in O.unflatten_params(g_w.cpu().numpy(), D).items()}
            for k in names:
                if k in gW:
                    errs[mode + ":" + k] = nerr(got[k], ref_w[k], gW[k][1])
                else:   # biases and the rgb branch: exactly zero
                    assert float(got[k].abs().max()) == 0.0, k
    worst = max(errs.values())
    print("D=%d M=%d worst normalised error %.1f (%s)" % (D, M, worst, max(errs, key=errs.get)))
    assert worst < GATE, errs


@pytest.mark.parametrize("D", [64, 256])
def test_field_hvp_same_bits(D):
    """two calls on the same inputs give the same bytes (fixed-order sums, no float atomics)"""
    P, p, u = case(D, 3000, seed=8)
    a = hvp_call(P, D, p, u)
    b = hvp_call(P, D, p, u)
    assert a[0].cpu().numpy().tobytes() == b[0].cpu().numpy().tobytes()
    assert a[1].cpu().numpy().tobytes() == b[1].cpu().numpy().tobytes()


def test_field_hvp_workspace_sizing_and_checks():
    """NNB_HVP adds the tangent stash only when set; the call refuses a workspace sized without it, a null u, N <= 0"""
    from nope_nerf_b200 import _lib as L, ops
    for D in (64, 128, 256):
        for M in (1, 65, 5000):
            base = L.lib.nnb_workspace_bytes_dim(M, 1, L.STASH, L.ENGINE_SIMT, D)
            hvp = L.lib.nnb_workspace_bytes_dim(M, 1, L.STASH | L.HVP, L.ENGINE_SIMT, D)
            Mpad = _align(M, 128)
            assert hvp == base + 8 * _align(Mpad * D * 4, 256) + _align(Mpad * 64 * 4, 256)
            assert L.lib.nnb_workspace_bytes_dim(M, 1, L.HVP, L.ENGINE_SIMT, D) == L.lib.nnb_workspace_bytes_dim(M, 1, 0, L.ENGINE_SIMT, D)
    D, M = 64, 100
    P, p, u = case(D, M)
    flat = torch.from_numpy(np.concatenate([np.asarray(P[n], np.float32).reshape(-1) for n, _ in O.param_shapes(D)])).cuda()
    p_c = torch.from_numpy(p).cuda(); u4 = torch.zeros(M, 4, device="cuda"); g_p = torch.zeros(M, 4, device="cuda")
    ws = torch.empty(L.lib.nnb_workspace_bytes_dim(M, 1, L.STASH, L.ENGINE_SIMT, D), dtype=torch.uint8, device="cuda")
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p_c); a.N = M; a.S = 1; a.engine = L.ENGINE_SIMT; a.hidden_dim = D
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    a.flags = L.STASH                      # no NNB_HVP
    assert L.lib.nnb_field_hvp(C.byref(a), L.ptr(u4), L.ptr(g_p), None, ops._stream()) < 0
    a.flags = L.STASH | L.HVP              # flag set, workspace too small
    assert L.lib.nnb_field_hvp(C.byref(a), L.ptr(u4), L.ptr(g_p), None, ops._stream()) < 0
    assert b"workspace too small" in L.lib.nnb_last_error()
    ws2 = torch.empty(L.lib.nnb_workspace_bytes_dim(M, 1, L.STASH | L.HVP, L.ENGINE_SIMT, D), dtype=torch.uint8, device="cuda")
    a.workspace = L.ptr(ws2); a.workspace_bytes = ws2.numel()
    assert L.lib.nnb_field_hvp(C.byref(a), None, L.ptr(g_p), None, ops._stream()) < 0            # null u
    assert L.lib.nnb_field_hvp(C.byref(a), L.ptr(u4), None, None, ops._stream()) < 0             # nothing to compute
    a.N = 0
    assert L.lib.nnb_field_hvp(C.byref(a), L.ptr(u4), L.ptr(g_p), None, ops._stream()) < 0
    a.N = M
    assert L.lib.nnb_field_hvp(C.byref(a), L.ptr(u4), L.ptr(g_p), None, ops._stream()) == 0
    torch.cuda.synchronize()

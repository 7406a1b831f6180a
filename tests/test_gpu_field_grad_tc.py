"""GPU: the tensor-core backward of explicit-point field queries with weight gradients (nnb_field_grad: tc_points_grad_fwd,
tc_points_grad and the weight-gradient stage of csrc/nnb_tc.cu), and its Python path (forward / infer_occ with engine='tc',
grad_engine='tc').

Checks:
- bits shared with the existing calls: out_rgba is nnb_field_fwd's on tensor cores, g_pts / g_dirs are nnb_field_vjp's;
- every dW / db, g_pts and g_dirs against float64 torch autograd of the field evaluated with the ReLU gates this call's forward wrote
  (read from its workspace), within 1e-4 of each tensor's maximum (DESIGN.md §2) on every row;
- agreement with the exact engine (nnb_field_fwd + nnb_field_bwd) with the cotangent restricted to the rows both engines gate alike;
- two calls give the same bits, g_weights accumulates (x + the result from zeros, bit for bit), the occupancy-only call leaves the colour
  parameters' slots untouched, and a workspace of zeros, NaN bytes or large finite words gives the same bits (rows past N add nothing);
- every error code, with nothing launched.

Largest measured over all cases below (NVIDIA H100 80GB HBM3, 700 W power limit), relative to the tensor's maximum (D = 64 / 128 / 256):
every dW / db against float64 3.3e-5 / 5.1e-5 / 9.4e-5; g_pts 1.4e-5 / 2.3e-5 / 1.5e-5 and g_dirs 1.4e-5 / 7.9e-6 / 6.2e-6 from 128 points
on, and g_pts of the calls of 1 and 127 points up to 2.2e-4 (SMALL_TOL); against the exact engine on the rows both gate alike
3.2e-5 / 5.2e-5 / 9.4e-5; deepest gate that differs from float64's 5.8e-7 of the layer's largest pre-activation.  One Adam step: the steps
agree to 3e-5 lr where the gradient is above 1e-2 of its maximum.  Run with -s to print them per case.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
import _fullsize_cases as FC
from test_gpu_relu_mask import layout, decode
from test_gpu_field_vjp import vjp_call, field_fwd, relmax, bits, FLIP_DEPTH

pytestmark = pytest.mark.gpu

TOL = 1e-4
SMALL_TOL = 5e-4   # g_pts / g_dirs of a call with fewer than 128 points (see test_bits_float64_and_exact_engine)
SIZES = (1, 127, 128, 129, 16901, 131072)


def _lib():
    from nope_nerf_b200 import _lib as L, ops
    return L, ops


def grad_call(flat, D, p, d, g, flags, gw=None, ws=None, out=True, g_dirs=True, o=None, gp=None, gd=None, ws_bytes=None, engine=None,
              weights=True):
    """one nnb_field_grad call; returns (rc, out_rgba, g_pts, g_dirs, g_weights) with fresh NaN-filled outputs and zeroed g_weights
    unless given"""
    L, ops = _lib()
    M = p.shape[0]
    nan = lambda: torch.full((M, 4), float("nan"), device="cuda")
    if ws is None:
        ws = torch.empty(max(L.lib.nnb_field_grad_workspace_bytes(M, flags, D), 256), dtype=torch.uint8, device="cuda")
    o = (nan() if out else None) if o is None else o
    gp = nan() if gp is None else gp
    gd = (nan() if g_dirs else None) if gd is None else gd
    if gw is None and weights:
        gw = torch.zeros(L.num_params(D), device="cuda")
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p); a.dirs = L.ptr(d); a.N = M; a.S = 1; a.flags = flags
    a.engine = L.ENGINE_TC if engine is None else engine; a.hidden_dim = D
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel() if ws_bytes is None else ws_bytes
    rc = L.lib.nnb_field_grad(C.byref(a), L.ptr(g), L.ptr(o), L.ptr(gp), L.ptr(gd), L.ptr(gw), ops._stream())
    torch.cuda.synchronize()
    return rc, o, gp, gd, gw


def exact_grad(flat, D, p, d, g, flags):
    """nnb_field_fwd (NNB_STASH) + nnb_field_bwd on the exact engine: (g_pts, g_dirs, g_weights from zeros, workspace)"""
    L, ops = _lib()
    M = p.shape[0]
    a, ws, _ = field_fwd(flat, D, p, d, flags | L.STASH, L.ENGINE_SIMT)
    gp = torch.empty(M, 4, device="cuda"); gd = torch.empty(M, 4, device="cuda"); gw = torch.zeros(L.num_params(D), device="cuda")
    assert L.lib.nnb_field_bwd(C.byref(a), L.ptr(g), L.ptr(gp), L.ptr(gd), L.ptr(gw), ops._stream()) == 0, L.lib.nnb_last_error()
    torch.cuda.synchronize()
    return gp, gd, gw, ws


def make_inputs(D, M, seed, with_dirs=True):
    rng = np.random.default_rng(seed)
    P = O.init_params(seed=7 + D, D=D, hf_damp=True)
    p = rng.uniform(-1.5, 1.5, (M, 3)).astype(np.float32)
    d = rng.normal(size=(M, 3)); d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    g = rng.normal(size=(M, 4)).astype(np.float32)
    flat = torch.from_numpy(O.flatten_params(P)).cuda()
    cu = lambda x: None if x is None else torch.from_numpy(x).cuda()
    return flat, cu(p), cu(d if with_dirs else None), cu(g)


def grad_gates(ws, N, D, occ):
    """the ReLU gate bits nnb_field_grad's forward wrote (make_layout's gates region): [bool (N, D)] x 8 and, unless occ, [bool (N, D/2)]"""
    lay = layout(N, 1, D)
    w = ws[lay["gates"]:lay["gates"] + lay["Mpad"] * D + lay["Mpad"] * D // 16].cpu().numpy()
    n_tiles, mp = lay["n_tiles"], lay["Mpad"]
    out = []
    for layer in range(8 if occ else 9):
        cols = D if layer < 8 else D // 2
        off = layer * mp * D // 8 if layer < 8 else mp * D
        out.append(torch.from_numpy(decode(w[off:off + mp * cols // 8], n_tiles, cols)[:N]).cuda())
    return out


def param_slices(D):
    from nope_nerf_b200.model.official_nerf import param_slices as ps, param_shapes
    return [(n, o, k, s) for (n, _), (o, k, s) in zip(param_shapes(D), ps(D))]


COLOUR = ("fc_feature.weight", "fc_feature.bias", "rgb_layers.0.weight", "rgb_layers.0.bias", "fc_rgb.weight", "fc_rgb.bias")


def field64(flat, D, p, d, g, flags, gates, occ):
    """float64 torch autograd of OfficialStaticNerf.forward at the fp32 inputs, each ReLU replaced by the gate the tensor-core forward
    wrote: returns (g_pts, g_dirs, {name: dW}, flip) with flip the largest |pre-activation| / (that layer's largest) over the units whose
    gate differs from the sign of float64's pre-activation"""
    L, _ = _lib()
    W = {n: flat[o:o + k].double().view(s).clone().requires_grad_(True) for n, o, k, s in param_slices(D)}
    P = p.double().clone().requires_grad_(True)
    Dd = (torch.ones_like(P) if d is None else d.double()).clone().requires_grad_(True)
    enc = lambda x, n: torch.cat([x] + [f(2.0 ** i * x) for i in range(n) for f in (torch.sin, torch.cos)], -1)
    e = enc(P, 10)
    x, flip = e, 0.0
    names = [("layers0", i) for i in (0, 2, 4, 6)] + [("layers1", i) for i in (0, 2, 4, 6)]
    for l, (blk, i) in enumerate(names):
        if l == 4:
            x = torch.cat([x, e], -1)
        y = x @ W["%s.%d.weight" % (blk, i)].T + W["%s.%d.bias" % (blk, i)]
        diff = gates[l] != (y.detach() > 0)
        if diff.any():
            flip = max(flip, float(y.detach()[diff].abs().max() / y.detach().abs().max()))
        x = y * gates[l].double()
    s = (x @ W["fc_density.weight"].T + W["fc_density.bias"])[:, 0]
    if flags & L.RAW_DENSITY:
        a = s
    else:
        sigma = torch.nn.functional.softplus(s) if flags & L.SOFTPLUS else torch.relu(s)
        a = sigma if flags & L.DIST_ALPHA else 1 - torch.exp(-sigma)
    loss = (a * g[:, 3].double()).sum()
    if not occ:
        feat = x @ W["fc_feature.weight"].T + W["fc_feature.bias"]
        yr = torch.cat([feat, enc(Dd, 4)], -1) @ W["rgb_layers.0.weight"].T + W["rgb_layers.0.bias"]
        diff = gates[8] != (yr.detach() > 0)
        if diff.any():
            flip = max(flip, float(yr.detach()[diff].abs().max() / yr.detach().abs().max()))
        rgb = torch.sigmoid((yr * gates[8].double()) @ W["fc_rgb.weight"].T + W["fc_rgb.bias"])
        loss = loss + (rgb * g[:, :3].double()).sum()
    loss.backward()
    G = {n: (w.grad if w.grad is not None else torch.zeros_like(w)) for n, w in W.items()}
    return P.grad, (None if occ else Dd.grad), G, flip


def act_flags(occ_act, dist_alpha, raw):
    L, _ = _lib()
    return (L.SOFTPLUS if occ_act == "softplus" else 0) | (L.DIST_ALPHA if dist_alpha else 0) | (L.RAW_DENSITY if raw else 0)


@pytest.mark.parametrize("mode", ["dirs", "ones", "occ"])
@pytest.mark.parametrize("raw", [False, True], ids=["act", "raw"])
@pytest.mark.parametrize("dist_alpha", [False, True], ids=["alpha", "sigma"])
@pytest.mark.parametrize("occ_act", ["softplus", "relu"])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_bits_float64_and_exact_engine(D, occ_act, dist_alpha, raw, mode):
    """out_rgba bit for bit against nnb_field_fwd (TC), g_pts / g_dirs against nnb_field_vjp; every dW / db, g_pts, g_dirs against float64
    with this call's gates; agreement with the exact engine on the rows both engines gate alike.  131 072 points for one activation."""
    L, _ = _lib()
    occ = mode == "occ"
    flags = act_flags(occ_act, dist_alpha, raw) | (L.OCC_ONLY if occ else 0)
    sizes = SIZES if (occ_act == "softplus" and not dist_alpha and not raw) else SIZES[:-1]
    worst, small = {}, 0.0
    for M in sizes:
        flat, p, d, g = make_inputs(D, M, seed=3000 + M, with_dirs=(mode == "dirs"))
        ws = torch.empty(L.lib.nnb_field_grad_workspace_bytes(M, flags, D), dtype=torch.uint8, device="cuda")
        rc, out, gp, gd, gw = grad_call(flat, D, p, d, g, flags, ws=ws, g_dirs=not occ)
        assert rc == 0, L.lib.nnb_last_error()
        _, _, fwd = field_fwd(flat, D, p, d, flags, L.ENGINE_TC)
        torch.cuda.synchronize()
        assert torch.equal(bits(out), bits(fwd))
        rc, _, gp_v, gd_v = vjp_call(flat, D, p, d, g, flags, out=False, g_dirs=not occ)
        assert rc == 0 and torch.equal(bits(gp), bits(gp_v)), L.lib.nnb_last_error()
        if not occ:
            assert torch.equal(bits(gd), bits(gd_v))
        assert torch.isfinite(gw).all() and (gp[:, 3] == 0).all()
        gates = grad_gates(ws, M, D, occ)
        gp64, gd64, G64, flip = field64(flat, D, p, d, g, flags, gates, occ)
        e = dict(gp64=relmax(gp[:, :3].cpu().numpy(), gp64.cpu().numpy()))
        if not occ:
            e["gd64"] = relmax(gd[:, :3].cpu().numpy(), gd64.cpu().numpy())
        for n, o, k, s in param_slices(D):
            if occ and n in COLOUR:
                assert (gw[o:o + k] == 0).all(), n   # not touched: still the zeros it started from
                continue
            ref = G64[n].reshape(-1)
            if float(ref.abs().max()) > 0:
                e["w:" + n] = relmax(gw[o:o + k].cpu().numpy(), ref.cpu().numpy())
        # the exact engine, with the cotangent restricted to the rows both engines gate alike
        _, _, _, ws_s = exact_grad(flat, D, p, d, torch.zeros_like(g), flags & ~L.OCC_ONLY)
        lay = layout(M, 1, D)
        take = lambda off, cols: ws_s[off:off + lay["Mpad"] * cols * 4].view(torch.float32).view(lay["Mpad"], cols)[:M] > 0
        gs = [take(o_, D) for o_ in lay["h"]] + [take(lay["hr"], D // 2)]
        same = torch.stack([(a_ == b_).all(1) for a_, b_ in zip(gates, gs)]).all(0)
        g_same = g * same[:, None]
        if occ:
            g_same[:, :3] = 0
        gp_s, gd_s, gw_s, _ = exact_grad(flat, D, p, d, g_same, flags & ~L.OCC_ONLY)
        rc, _, gp_t, gd_t, gw_t = grad_call(flat, D, p, d, g_same, flags, g_dirs=not occ, out=False)
        assert rc == 0
        e["gp_exact"] = relmax(gp_t[:, :3].cpu().numpy(), gp_s[:, :3].double().cpu().numpy())
        if not occ:
            e["gd_exact"] = relmax(gd_t[:, :3].cpu().numpy(), gd_s[:, :3].double().cpu().numpy())
        for n, o, k, s in param_slices(D):
            if occ and n in COLOUR:
                continue
            ref = gw_s[o:o + k].double()
            if float(ref.abs().max()) > 0:
                e["x:" + n] = relmax(gw_t[o:o + k].cpu().numpy(), ref.cpu().numpy())
        # g_pts of a point is a sum of encoding terms up to 512 p that largely cancel, so its error is set by the terms, not by the result;
        # over a tensor of one or a few rows the maximum is that of those few points (measured: 1.4e-4 at N = 1, the bits of nnb_field_vjp)
        tol_rows = TOL if M >= 128 else SMALL_TOL
        bad = {k: v for k, v in e.items() if v > (tol_rows if k in ("gp64", "gd64", "gp_exact", "gd_exact") else TOL)}
        assert not bad and flip <= FLIP_DEPTH, (D, flags, M, bad, flip)
        if M < 128:
            small = max(small, e["gp64"], e.get("gd64", 0.0), e["gp_exact"], e.get("gd_exact", 0.0))
            e = {k: v for k, v in e.items() if k not in ("gp64", "gd64", "gp_exact", "gd_exact")}
            e.update(gp64=0.0, gp_exact=0.0)
        summary = dict(g_pts=e["gp64"], g_dirs=e.get("gd64", 0.0), weights=max(v for k, v in e.items() if k.startswith("w:")),
                       exact=max(v for k, v in e.items() if k.endswith("_exact") or k.startswith("x:")), flip=flip,
                       rows_gates_differ=float(1.0 - same.float().mean()))
        worst = {k: max(worst.get(k, 0.0), v) for k, v in summary.items()}
    worst["point_grads_below_128_rows"] = small
    print("field_grad D=%d flags=0x%x %s: %s" % (D, flags, mode, " ".join("%s %.2e" % kv for kv in sorted(worst.items()))))


@pytest.mark.parametrize("occ", [False, True], ids=["full", "occ_only"])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_determinism_accumulation_and_workspace_poison(D, occ):
    """two calls give the same bits; g_weights prefilled with x gives x + (the result from zeros) bit for bit; occupancy-only leaves the
    colour slots as they were; a workspace of zeros, of NaN bytes or of large finite words gives the same bits, so the rows of the last
    tile past N add exactly nothing"""
    L, _ = _lib()
    M = 16901
    flags = L.SOFTPLUS | (L.OCC_ONLY if occ else 0)
    flat, p, d, g = make_inputs(D, M, seed=91)
    d = None if occ else d
    need = L.lib.nnb_field_grad_workspace_bytes(M, flags, D)
    ref = grad_call(flat, D, p, d, g, flags, g_dirs=not occ)
    assert ref[0] == 0, L.lib.nnb_last_error()
    again = grad_call(flat, D, p, d, g, flags, g_dirs=not occ)
    for x, y in zip(ref[1:], again[1:]):
        if x is not None:
            assert torch.equal(bits(x), bits(y))
    x0 = torch.randn(L.num_params(D), device="cuda", generator=torch.Generator("cuda").manual_seed(5))
    rc, *_, gw = grad_call(flat, D, p, d, g, flags, gw=x0.clone(), g_dirs=not occ)
    assert rc == 0 and torch.equal(bits(gw), bits(x0 + ref[4]))
    if occ:
        for n, o, k, s in param_slices(D):
            if n in COLOUR:
                assert torch.equal(bits(gw[o:o + k]), bits(x0[o:o + k])), n
    for fill in (0x00, 0xFF, 0x7E):   # 0x7E7E7E7E is about 8.5e37
        ws = torch.full((need,), fill, dtype=torch.uint8, device="cuda")
        res = grad_call(flat, D, p, d, g, flags, ws=ws, g_dirs=not occ)
        assert res[0] == 0
        for x, y in zip(ref[1:], res[1:]):
            if x is not None:
                assert torch.equal(bits(x), bits(y)), fill
    # without g_weights the call is nnb_field_vjp
    rc, o, gp, gd, gw = grad_call(flat, D, p, d, g, flags, g_dirs=not occ, weights=False)
    assert rc == 0 and gw is None and torch.equal(bits(gp), bits(ref[2])) and torch.equal(bits(o), bits(ref[1]))


def test_error_paths():
    """each rejected call launches nothing (its outputs keep their NaNs, g_weights its sentinel); the same buffers then succeed"""
    L, _ = _lib()
    D, M = 64, 100
    flat, p, d, g = make_inputs(D, M, seed=41)
    err = lambda: L.lib.nnb_last_error().decode()
    need = L.lib.nnb_field_grad_workspace_bytes(M, L.SOFTPLUS, D)
    ws = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    o, gp, gd = (torch.full((M + 8, 4), float("nan"), device="cuda") for _ in range(3))
    gw = torch.full((L.num_params(D) + 8,), -7.0, device="cuda")
    untouched = lambda: bool(torch.isnan(o).all() and torch.isnan(gp).all() and torch.isnan(gd).all() and (gw == -7.0).all())
    cases = [
        (dict(engine=L.ENGINE_SIMT), -4, "engine"),
        (dict(engine=7), -4, "engine"),
        (dict(flags=L.SOFTPLUS | 512), -7, "not defined"),
        (dict(flags=L.SOFTPLUS | (1 << 16)), -7, "not defined"),
        (dict(flags=L.SOFTPLUS | L.STASH), -6, "NNB_STASH"),
        (dict(flags=L.SOFTPLUS | L.HVP), -6, "NNB_HVP"),
        (dict(flags=L.SOFTPLUS | L.OCC_ONLY), -6, "g_dirs"),
        (dict(D=96), -8, "hidden_dim"),
        (dict(ws_bytes=need - 1), -5, "too small"),
        (dict(ws=ws[16:], ws_bytes=need), -5, "aligned"),
        (dict(p=None), -3, "pts"),
        (dict(flat=None), -3, "weights"),
        (dict(g=None), -3, "g_rgba"),
        (dict(gp=None), -3, "g_pts"),
        (dict(gp=gp.view(-1)[1:1 + 4 * M].view(M, 4)), -3, "aligned"),
        (dict(o=o.view(-1)[2:2 + 4 * M].view(M, 4)), -3, "aligned"),
        (dict(gd=gd.view(-1)[3:3 + 4 * M].view(M, 4)), -3, "aligned"),
        (dict(g=g.view(-1)[1:1 + 4 * (M - 1)].view(M - 1, 4)), -3, "aligned"),
        (dict(gw_off=2), -3, "g_weights"),
    ]
    for kw, code, word in cases:
        kw = dict(kw)
        a = L.RenderArgs()
        a.weights = L.ptr(kw["flat"]) if "flat" in kw else L.ptr(flat)
        a.pts = L.ptr(kw["p"]) if "p" in kw else L.ptr(p)
        a.dirs = L.ptr(d); a.N = M; a.S = 1; a.flags = kw.get("flags", L.SOFTPLUS); a.engine = kw.get("engine", L.ENGINE_TC)
        a.hidden_dim = kw.get("D", D)
        w_ = kw.get("ws", ws)
        a.workspace = L.ptr(w_); a.workspace_bytes = kw.get("ws_bytes", w_.numel())
        gw_ptr = L.ptr(gw) + kw.get("gw_off", 0)   # a float pointer off by 2 bytes
        _, ops = _lib()
        rc = L.lib.nnb_field_grad(C.byref(a), L.ptr(kw["g"]) if "g" in kw else L.ptr(g), L.ptr(kw.get("o", o)),
                                  L.ptr(kw["gp"]) if "gp" in kw else L.ptr(gp), L.ptr(kw.get("gd", gd)), gw_ptr, ops._stream())
        torch.cuda.synchronize()
        assert rc == code and word in err() and untouched(), (kw.keys(), rc, code, err())
    rc, *_ = grad_call(flat, D, p[:0], d[:0], g[:0], L.SOFTPLUS, ws=ws, o=o, gp=gp, gd=gd, gw=gw)
    assert rc == 0 and untouched()
    rc, *_ = grad_call(flat, D, p, d, g, L.SOFTPLUS, ws=ws, o=o, gp=gp, gd=gd, gw=gw)
    assert rc == 0 and bool(torch.isfinite(o[:M]).all() and torch.isfinite(gp[:M]).all() and torch.isfinite(gd[:M]).all()), err()
    assert bool((gw[L.num_params(D):] == -7.0).all())   # past the parameters: not written


def _net(D, seed=3):
    import nope_nerf_b200.model as mdl
    cfg = FC.default_cfg(); cfg["model"]["hidden_dim"] = D
    net = mdl.OfficialStaticNerf(cfg).cuda()
    P = O.init_params(seed=seed + D, D=D, hf_damp=True)
    net.load_state_dict({k: torch.from_numpy(np.asarray(P[k], np.float32)).reshape(v.shape) for k, v in net.state_dict().items()})
    return net


@pytest.mark.parametrize("D", [64, 128, 256])
def test_python_path(D):
    """forward(p, d, engine='tc', grad_engine='tc') and infer_occ(p, engine='tc', grad_engine='tc'): outputs are the inference query's
    bits, and the gradients in p, d and every parameter are nnb_field_grad's bit for bit.  One Adam step from the same start on both
    engines moves every parameter whose gradient is above 1e-2 of its tensor's maximum by the same amount to 1e-2 of the step."""
    L, _ = _lib()
    net = _net(D)
    flags = L.SOFTPLUS
    M = 20000
    gen = torch.Generator().manual_seed(2)
    p0 = (torch.rand(M, 3, generator=gen) * 3 - 1.5).cuda()
    d0 = torch.nn.functional.normalize(torch.randn(M, 3, generator=gen), dim=1).cuda()
    g = torch.randn(M, 4, generator=gen).cuda()
    flat = net.flat_weights()
    rc, _, gp_ref, gd_ref, gw_ref = grad_call(flat, D, p0, d0, g, flags, out=False)
    assert rc == 0
    p = p0.clone().requires_grad_(True); d = d0.clone().requires_grad_(True)
    net.zero_grad(set_to_none=True)
    rgb, a = net(p, d, return_addocc=True, engine="tc", grad_engine="tc")
    with torch.no_grad():
        rgb_i, a_i = net(p0, d0, return_addocc=True, engine="tc")
    assert torch.equal(bits(rgb), bits(rgb_i)) and torch.equal(bits(a), bits(a_i))
    ((rgb * g[:, :3]).sum() + (a[:, 0] * g[:, 3]).sum()).backward()
    assert torch.equal(bits(p.grad), bits(gp_ref[:, :3])) and torch.equal(bits(d.grad), bits(gd_ref[:, :3]))
    for q, (o, k, s) in zip(net.parameters(), net.param_slices):
        assert torch.equal(bits(q.grad.reshape(-1)), bits(gw_ref[o:o + k])), s
    # infer_occ: the occupancy-only backward on the raw logit
    occ_flags = L.SOFTPLUS | L.RAW_DENSITY | L.OCC_ONLY
    rc, _, gp_o, _, gw_o = grad_call(flat, D, p0, None, g, occ_flags, out=False, g_dirs=False)
    assert rc == 0
    p = p0.clone().requires_grad_(True)
    net.zero_grad(set_to_none=True)
    _, s = net.infer_occ(p, engine="tc", grad_engine="tc")
    (s[:, 0] * g[:, 3]).sum().backward()
    assert torch.equal(bits(p.grad), bits(gp_o[:, :3]))
    for name, q, (o, k, sh) in zip([n for n, _ in net.named_parameters()], net.parameters(), net.param_slices):
        if name in COLOUR:
            assert q.grad is None or not q.grad.any(), name
        else:
            assert torch.equal(bits(q.grad.reshape(-1)), bits(gw_o[o:o + k])), name
    # one Adam step on each engine from the same start
    lr, start = 1e-3, [q.detach().clone() for q in net.parameters()]
    steps, grads = {}, {}
    for eng in ("exact", "tc"):
        with torch.no_grad():
            for q, s0 in zip(net.parameters(), start):
                q.copy_(s0)
        opt = torch.optim.Adam(net.parameters(), lr=lr)
        opt.zero_grad(set_to_none=True)
        kw = dict(engine="tc", grad_engine="tc") if eng == "tc" else {}
        rgb, a = net(p0, d0, return_addocc=True, **kw)
        ((rgb * g[:, :3]).sum() + (a[:, 0] * g[:, 3]).sum()).backward()
        grads[eng] = [q.grad.detach().clone() for q in net.parameters()]
        opt.step()
        steps[eng] = [q.detach() - s0 for q, s0 in zip(net.parameters(), start)]
    # Where a gradient is above 1e-2 of its tensor's maximum, the bound of 1e-4 of the maximum is at most 1 % of the element, and Adam's
    # first step lr g / (|g| + eps) moves by far less than that: the steps agree to 1e-2 lr there.  (Below, an element's sign may differ
    # between two valid gradients, and its step by up to 2 lr.)
    worst = 0.0
    for ge, se, st in zip(grads["exact"], steps["exact"], steps["tc"]):
        big = ge.abs() > 1e-2 * ge.abs().max()
        worst = max(worst, float((se - st)[big].abs().max()) / lr)
        assert float((se - st).abs().max()) <= 2 * lr * (1 + 1e-3)
    print("Adam step D=%d: largest difference of the steps where the gradient is above 1e-2 of its maximum: %.2e lr" % (D, worst))
    assert worst <= 1e-2

"""GPU: the tensor-core data gradient of explicit-point field queries (nnb_field_vjp: tc_points_vjp_fwd + tc_points_vjp in
csrc/nnb_tc.cu), OfficialStaticNerf.gradient(engine='tc') and the geometry view with Renderer(normal_engine='tc').

Reference: oracle/nerf_oracle.py's mlp_forward / mlp_backward in float64 at the fp32 points, directions and weights (drawn with
hf_damp, see oracle.nerf_oracle.init_params), the backward gated by the ReLU bits of the evaluation it is compared with (read from
nnb_field_vjp's workspace, or from the exact engine's fp32 stash).  Bound: 1e-4 of each tensor's maximum (DESIGN.md §2) on every
checked row; every gate that differs from float64's own must sit within FLIP_DEPTH (1e-5) of the layer's largest pre-activation.

Largest measured over all cases below (NVIDIA H100 80GB HBM3, 700 W power limit), relative to the tensor's maximum, every checked row:
g_pts 2.5e-5 against float64 (and against the exact engine on the rows both engines gate alike), g_dirs 1.1e-5, out_rgba 2.9e-7;
the normals of gradient(engine='tc') 1.4e-5; the exact engine itself 9.1e-7.  Deepest gate that differs from float64's: 7.7e-7 of the
layer's largest pre-activation on tensor cores, 1.3e-8 on the exact engine; the engines gate at most 0.07 % of the checked rows
differently.  Run with -s to print them per case.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
import _fullsize_cases as FC

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-4
SIZES = (1, 127, 128, 129, 16901, 200003)   # those of test_gpu_field_tc.py
ORACLE_ROWS = 4096


def _lib():
    from nope_nerf_b200 import _lib as L, ops
    return L, ops


def vjp_call(flat, D, p, d, g, flags, out=True, g_dirs=True, ws=None, gp=None, gd=None, o=None, ws_bytes=None, engine=None):
    """one nnb_field_vjp call; returns (rc, out_rgba, g_pts, g_dirs) with fresh NaN-filled outputs unless given"""
    L, ops = _lib()
    M = p.shape[0]
    nan = lambda: torch.full((M, 4), float("nan"), device="cuda")
    if ws is None:
        ws = torch.empty(max(L.lib.nnb_field_vjp_workspace_bytes(M, flags, D), 256), dtype=torch.uint8, device="cuda")
    o = (nan() if out else None) if o is None else o
    gp = nan() if gp is None else gp
    gd = (nan() if g_dirs else None) if gd is None else gd
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p); a.dirs = L.ptr(d); a.N = M; a.S = 1; a.flags = flags
    a.engine = L.ENGINE_TC if engine is None else engine; a.hidden_dim = D
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel() if ws_bytes is None else ws_bytes
    rc = L.lib.nnb_field_vjp(C.byref(a), L.ptr(g), L.ptr(o), L.ptr(gp), L.ptr(gd), ops._stream())
    torch.cuda.synchronize()
    return rc, o, gp, gd


def field_fwd(flat, D, p, d, flags, engine):
    L, ops = _lib()
    M = p.shape[0]
    ws = torch.empty(L.lib.nnb_workspace_bytes_dim(M, 1, flags, engine, D), dtype=torch.uint8, device="cuda")
    out = torch.empty(M, 4, device="cuda")
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p); a.dirs = L.ptr(d); a.N = M; a.S = 1; a.flags = flags; a.engine = engine; a.hidden_dim = D
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    assert L.lib.nnb_field_fwd(C.byref(a), L.ptr(out), ops._stream()) == 0, L.lib.nnb_last_error()
    return a, ws, out


def exact_vjp(flat, D, p, d, g, flags):
    """nnb_field_fwd + nnb_field_bwd on the exact-fp32 engine: (out, g_pts, g_dirs, workspace with the fp32 stash)"""
    L, ops = _lib()
    M = p.shape[0]
    a, ws, out = field_fwd(flat, D, p, d, flags | L.STASH, L.ENGINE_SIMT)
    gp = torch.empty(M, 4, device="cuda"); gd = torch.empty(M, 4, device="cuda")
    assert L.lib.nnb_field_bwd(C.byref(a), L.ptr(g), L.ptr(gp), L.ptr(gd), None, ops._stream()) == 0, L.lib.nnb_last_error()
    torch.cuda.synchronize()
    return out, gp, gd, ws


def make_inputs(D, M, seed, with_dirs=True):
    rng = np.random.default_rng(seed)
    P = O.init_params(seed=7 + D, D=D, hf_damp=True)
    p = rng.uniform(-1.5, 1.5, (M, 3)).astype(np.float32)
    d = rng.normal(size=(M, 3)); d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    g = rng.normal(size=(M, 4)).astype(np.float32)
    flat = torch.from_numpy(O.flatten_params(P)).cuda()
    return P, p, (d if with_dirs else None), g, flat


def act_flags(act):
    L, _ = _lib()
    return L.SOFTPLUS | {"alpha": 0, "sigma": L.DIST_ALPHA, "logit": L.RAW_DENSITY}[act]


def oracle64_forward(P, p, d, act):
    """float64 forward at the fp32 inputs: (rgb, fourth channel, cache for oracle64_backward)"""
    P64 = {k: np.asarray(v, np.float64) for k, v in P.items()}
    dd = np.ones_like(p, dtype=np.float64) if d is None else d.astype(np.float64)
    rgb, a, cache = O.mlp_forward(P64, p.astype(np.float64), dd, dist_alpha=(act == "sigma"), occ_activation="softplus")
    if act == "logit":   # the fourth channel is s itself: d channel / d s = 1 (relu' of a positive s, no exp(-sigma) factor)
        a = cache["s"]
        cache = dict(cache, occ="relu", dist_alpha=True, s=np.ones_like(cache["s"]))
    return rgb, a, dict(cache, P64=P64)


def oracle64_backward(cache, g, occ, gates):
    """float64 (g_pts, g_dirs) for the cotangent g (its rgb part ignored when occ), with the ReLU gates of an fp32 evaluation:
    gates = [bool (k, D)] x 8 for h0..h7 and, unless occ, [bool (k, D/2)] for the rgb hidden layer.  A gradient is discontinuous where
    a pre-activation crosses 0, so an fp32 evaluation whose rounding puts a pre-activation within about 1e-6 of 0 on the other side
    than float64 has another, equally valid gradient there; with the evaluation's own gates float64 gives the gradient it must match."""
    c = dict(cache, Y=[m.astype(np.float64) for m in gates[:8]])   # mlp_backward gates with Y > 0 and yr > 0
    if not occ:
        c["yr"] = gates[8].astype(np.float64)
    g64 = g.astype(np.float64)
    g_rgb = np.zeros_like(g64[:, :3]) if occ else g64[:, :3]
    _, g_pts, g_dirs = O.mlp_backward(c["P64"], c, g_rgb, g64[:, 3])
    return g_pts, g_dirs


def tc_gates(ws, N, D, rows, occ):
    """the ReLU gate bits nnb_field_vjp wrote to its workspace, for `rows`: [bool (k, D)] x 8 (h0..h7), and [bool (k, D/2)] for the
    rgb hidden layer unless occ.  Workspace: records (32 Npad bytes), then the gate_bits_off regions (nnb_workspace.cuh): thread t of a
    tile holds bit b = 4j + 2r + e = (row 64 (w / 4) + 16 (w % 4) + lane / 4 + 8 r, column 8 j + 2 (lane % 4) + e), w = t / 32, as bit
    W - 1 - b % W of its little-endian W-bit word b / W (W = 16 for the 16 bits of the rgb hidden layer at D = 64)."""
    w = ws.cpu().numpy()
    npad = (N + 127) // 128 * 128
    R = np.asarray(rows, np.int64)[:, None]
    rr = R % 128
    w16 = rr % 16
    out = []
    for layer in range(8 if occ else 9):
        cols = D if layer < 8 else D // 2
        nb = cols // 2
        W = 32 if nb >= 32 else 16
        off = npad * 32 + (layer * (npad // 128) * 16 * D if layer < 8 else npad * D)
        per_tile, per_thread = (16 * D, D // 16) if layer < 8 else (8 * D, D // 32)
        c = np.arange(cols)[None, :]
        t = 32 * (4 * (rr // 64) + (rr % 64) // 16) + 4 * (w16 % 8) + (c % 8) // 2
        b = 4 * (c // 8) + 2 * (w16 // 8) + c % 2
        byte = off + (R // 128) * per_tile + t * per_thread + (b // W) * (W // 8)
        word = sum(w[byte + k].astype(np.int64) << (8 * k) for k in range(W // 8))
        out.append(((word >> (W - 1 - b % W)) & 1).astype(bool))
    return out


def simt_gates(ws, N, D, rows):
    """h > 0 of the exact engine's fp32 stash (nnb_field_fwd with NNB_STASH) for `rows`: h0..h7 and the rgb hidden layer"""
    from test_gpu_relu_mask import layout
    lay = layout(N, 1, D)
    mp, r = lay["Mpad"], torch.from_numpy(np.asarray(rows, np.int64)).cuda()
    take = lambda off, cols: (ws[off:off + mp * cols * 4].view(torch.float32).view(mp, cols)[r] > 0).cpu().numpy()
    return [take(o, D) for o in lay["h"]] + [take(lay["hr"], D // 2)]


def flip_depth(gates, cache, occ):
    """the largest |float64 pre-activation| / (that layer's largest) over the units whose gate differs from float64's"""
    pre = list(cache["Y"]) + ([] if occ else [cache["yr"]])
    worst = 0.0
    for m, y in zip(gates, pre):
        diff = m != (y > 0)
        if diff.any():
            worst = max(worst, float(np.abs(y[diff]).max() / np.abs(y).max()))
    return worst


FLIP_DEPTH = 1e-5   # a gate may differ from float64's only where the pre-activation is within rounding of 0 (relative to the layer)


def relmax(x, ref):
    return float(np.abs(np.asarray(x, np.float64) - ref).max() / max(np.abs(ref).max(), 1e-30))


def bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("mode", ["dirs", "ones", "occ"])
@pytest.mark.parametrize("act", ["alpha", "sigma", "logit"])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_against_float64_and_exact_engine(D, act, mode):
    """g_pts, g_dirs and out_rgba against float64 and the exact engine on every checked row; out_rgba bit for bit against nnb_field_fwd
    on tensor cores.  The float64 gradients use the gates of the evaluation they are compared with (oracle64_backward), read from its
    workspace, and every gate that differs from float64's must sit within FLIP_DEPTH of 0.  The two engines are compared on the rows
    whose gates they share.  With NNB_OCC_ONLY the colour cotangent is NaN: it must not be read."""
    from test_gpu_relu_mask import decode
    L, _ = _lib()
    occ = mode == "occ"
    flags = act_flags(act) | (L.OCC_ONLY if occ else 0)
    worst = {}
    for M in SIZES:
        P, p, d, g, flat = make_inputs(D, M, seed=2000 + M, with_dirs=(mode == "dirs"))
        pc = torch.from_numpy(p).cuda(); dc = None if d is None else torch.from_numpy(d).cuda()
        gc = torch.from_numpy(g).cuda()
        g_in = gc.clone()
        if occ:
            g_in[:, :3] = float("nan")
        ws = torch.empty(L.lib.nnb_field_vjp_workspace_bytes(M, flags, D), dtype=torch.uint8, device="cuda")
        rc, out, gp, gd = vjp_call(flat, D, pc, dc, g_in, flags, g_dirs=not occ, ws=ws)
        assert rc == 0, L.lib.nnb_last_error()
        _, _, fwd = field_fwd(flat, D, pc, dc, flags, L.ENGINE_TC)
        torch.cuda.synchronize()
        assert torch.equal(bits(out), bits(fwd))
        g_ex = gc.clone()
        if occ:
            g_ex[:, :3] = 0.0
        out_s, gp_s, gd_s, ws_s = exact_vjp(flat, D, pc, dc, g_ex, act_flags(act))
        out, gp = out.cpu().numpy(), gp.cpu().numpy()
        assert np.isfinite(out).all() and np.isfinite(gp[:, :3]).all() and (gp[:, 3] == 0).all()
        rows = np.arange(M)
        if M > ORACLE_ROWS:
            last_tile = (M - 1) // 128 * 128
            rows = np.unique(np.concatenate([np.random.default_rng(M).choice(M, ORACLE_ROWS, replace=False), [0, last_tile - 1, last_tile, M - 1]]))
        gt = tc_gates(ws, M, D, rows, occ)
        if M <= 129:   # the row decoder above against the tile decoder of test_gpu_relu_mask
            n_tiles, npad = (M + 127) // 128, (M + 127) // 128 * 128
            wnp = ws.cpu().numpy()
            for layer, m in enumerate(gt):
                cols = m.shape[1]
                off = npad * 32 + (layer * npad * D // 8 if layer < 8 else npad * D)
                assert np.array_equal(decode(wnp[off:off + npad * cols // 8], n_tiles, cols)[rows], m), layer
        gs = simt_gates(ws_s, M, D, rows)[:len(gt)]
        rgb64, a64, cache = oracle64_forward(P, p[rows], None if d is None else d[rows], act)
        gp64, gd64 = oracle64_backward(cache, g[rows], occ, gt)
        gp64_s, gd64_s = oracle64_backward(cache, g[rows], occ, gs)
        same = np.logical_and.reduce([(a_ == b_).all(1) for a_, b_ in zip(gt, gs)])   # rows the two engines gate alike
        gp_s = gp_s[:, :3].cpu().numpy().astype(np.float64)[rows]
        e = dict(a64=relmax(out[rows, 3], a64), gp64=relmax(gp[rows, :3], gp64), gp_simt64=relmax(gp_s, gp64_s),
                 gp_simt=relmax(gp[rows][same, :3], gp_s[same]),
                 flip_tc=flip_depth(gt, cache, occ), flip_simt=flip_depth(gs, cache, occ))
        if not occ:
            gd = gd.cpu().numpy()
            assert np.isfinite(gd[:, :3]).all()
            gd_s = gd_s[:, :3].cpu().numpy().astype(np.float64)[rows]
            e.update(rgb64=relmax(out[rows, :3], rgb64), gd64=relmax(gd[rows, :3], gd64), gd_simt64=relmax(gd_s, gd64_s),
                     gd_simt=relmax(gd[rows][same, :3], gd_s[same]))
        else:
            assert (out[:, :3] == 0).all()
        flip = {k: e.pop(k) for k in ("flip_tc", "flip_simt")}
        assert max(e.values()) <= TOL and max(flip.values()) <= FLIP_DEPTH, (D, act, mode, M, e, flip)
        e.update(flip, rows_gates_differ=float(1.0 - same.mean()))
        worst = {k: max(worst.get(k, 0.0), v) for k, v in e.items()}
    print("field_vjp D=%d %s %s: %s" % (D, act, mode, " ".join("%s %.2e" % kv for kv in sorted(worst.items()))))


@pytest.mark.parametrize("occ", [False, True], ids=["full", "occ_only"])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_row_independence_workspace_and_sentinels(D, occ):
    """a point's outputs depend on that point alone: permuted and embedded among other points in a larger call, every row keeps its
    bits; a workspace of 0xFF bytes changes nothing; rows past N keep their sentinels"""
    L, _ = _lib()
    M, BIG, PAD, SENT = 3 * 128 + 77, 2 * 16896 + 1000, 200, -12345.5
    flags = L.SOFTPLUS | (L.OCC_ONLY if occ else 0)
    P, p, d, g, flat = make_inputs(D, BIG, seed=77)
    pc, dc, gc = (torch.from_numpy(x).cuda() for x in (p, d, g))
    rc, o1, gp1, gd1 = vjp_call(flat, D, pc[:M].contiguous(), dc[:M].contiguous(), gc[:M].contiguous(), flags, g_dirs=not occ)
    assert rc == 0, L.lib.nnb_last_error()
    perm = torch.from_numpy(np.random.default_rng(8).permutation(BIG)).cuda()
    rc, o2, gp2, gd2 = vjp_call(flat, D, pc[perm].contiguous(), dc[perm].contiguous(), gc[perm].contiguous(), flags, g_dirs=not occ)
    assert rc == 0, L.lib.nnb_last_error()
    inv = torch.argsort(perm)[:M]   # where each of the first M points went
    assert torch.equal(bits(o2[inv]), bits(o1)) and torch.equal(bits(gp2[inv]), bits(gp1))
    if not occ:
        assert torch.equal(bits(gd2[inv]), bits(gd1))
    ws = torch.full((L.lib.nnb_field_vjp_workspace_bytes(M, flags, D),), 0xFF, dtype=torch.uint8, device="cuda")
    bufs = [torch.full((M + PAD, 4), SENT, device="cuda") for _ in range(3)]
    rc, o3, gp3, gd3 = vjp_call(flat, D, pc[:M].contiguous(), dc[:M].contiguous(), gc[:M].contiguous(), flags, ws=ws,
                                o=bufs[0], gp=bufs[1], gd=None if occ else bufs[2], g_dirs=not occ)
    assert rc == 0, L.lib.nnb_last_error()
    assert torch.equal(bits(o3[:M]), bits(o1)) and torch.equal(bits(gp3[:M]), bits(gp1))
    if not occ:
        assert torch.equal(bits(gd3[:M]), bits(gd1))
    for b in bufs[:2] + ([] if occ else bufs[2:]):
        assert torch.equal(b[M:], torch.full((PAD, 4), SENT, device="cuda"))


def test_error_paths():
    """each rejected call launches nothing (its outputs keep their NaNs); the same buffers then succeed with valid arguments"""
    L, _ = _lib()
    D, M = 64, 100
    P, p, d, g, flat = make_inputs(D, M, seed=41)
    pc, dc, gc = (torch.from_numpy(x).cuda() for x in (p, d, g))
    err = lambda: L.lib.nnb_last_error().decode()
    need = L.lib.nnb_field_vjp_workspace_bytes(M, L.SOFTPLUS, D)
    ws = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    o, gp, gd = (torch.full((M + 8, 4), float("nan"), device="cuda") for _ in range(3))
    untouched = lambda: bool(torch.isnan(o).all() and torch.isnan(gp).all() and torch.isnan(gd).all())
    cases = [
        (dict(flags=L.SOFTPLUS, engine=L.ENGINE_SIMT), -4, "engine"),
        (dict(flags=L.SOFTPLUS, engine=7), -4, "engine"),
        (dict(flags=L.SOFTPLUS | 512), -7, "not defined"),
        (dict(flags=L.SOFTPLUS | (1 << 16)), -7, "not defined"),
        (dict(flags=L.SOFTPLUS | L.STASH), -6, "NNB_STASH"),
        (dict(flags=L.SOFTPLUS | L.HVP), -6, "NNB_HVP"),
        (dict(flags=L.SOFTPLUS, D=96), -8, "hidden_dim"),
        (dict(flags=L.SOFTPLUS, ws_bytes=need - 1), -5, "too small"),
        (dict(flags=L.SOFTPLUS, ws=ws[16:], ws_bytes=need), -5, "aligned"),
        (dict(flags=L.SOFTPLUS, p=None), -3, "pts"),
        (dict(flags=L.SOFTPLUS, g=None), -3, "g_rgba"),
        (dict(flags=L.SOFTPLUS, gp=None), -3, "g_pts"),
        (dict(flags=L.SOFTPLUS, gp=gp.view(-1)[1:1 + 4 * M].view(M, 4)), -3, "aligned"),
        (dict(flags=L.SOFTPLUS, o=o.view(-1)[2:2 + 4 * M].view(M, 4)), -3, "aligned"),
        (dict(flags=L.SOFTPLUS, gd=gd.view(-1)[3:3 + 4 * M].view(M, 4)), -3, "aligned"),
        (dict(flags=L.SOFTPLUS, g=gc.view(-1)[1:1 + 4 * (M - 1)].view(M - 1, 4)), -3, "aligned"),
        (dict(flags=L.SOFTPLUS | L.OCC_ONLY), -6, "g_dirs"),
    ]
    for kw, code, word in cases:
        kw = dict(kw)
        a_p = kw.pop("p", pc); a_g = kw.pop("g", gc); a_D = kw.pop("D", D); a_flags = kw.pop("flags")
        kw.setdefault("ws", ws); kw.setdefault("o", o); kw.setdefault("gp", gp); kw.setdefault("gd", gd)
        if a_p is None:   # a NULL pts: pass a placeholder of the right length to the helper, then clear the pointer
            L_, ops = _lib()
            a = L_.RenderArgs()
            a.weights = L_.ptr(flat); a.pts = None; a.N = M; a.S = 1; a.flags = a_flags; a.engine = L_.ENGINE_TC; a.hidden_dim = D
            a.workspace = L_.ptr(ws); a.workspace_bytes = ws.numel()
            rc = L_.lib.nnb_field_vjp(C.byref(a), L_.ptr(gc), L_.ptr(o), L_.ptr(gp), L_.ptr(gd), ops._stream())
            torch.cuda.synchronize()
        elif kw.get("gp", 0) is None or a_g is None:
            L_, ops = _lib()
            a = L_.RenderArgs()
            a.weights = L_.ptr(flat); a.pts = L_.ptr(pc); a.N = M; a.S = 1; a.flags = a_flags; a.engine = L_.ENGINE_TC; a.hidden_dim = D
            a.workspace = L_.ptr(ws); a.workspace_bytes = ws.numel()
            rc = L_.lib.nnb_field_vjp(C.byref(a), L_.ptr(a_g), L_.ptr(o), L_.ptr(kw["gp"]), L_.ptr(gd), ops._stream())
            torch.cuda.synchronize()
        else:
            rc, *_ = vjp_call(flat, a_D, a_p, dc, a_g, a_flags, **kw)
        assert rc == code and word in err() and untouched(), (kw, a_flags, rc, code, err())
    # N == 0: nothing to do, success
    rc, *_ = vjp_call(flat, D, pc[:0], dc[:0], gc[:0], L.SOFTPLUS, ws=ws, o=o, gp=gp, gd=gd)
    assert rc == 0 and untouched()
    # and the same buffers are fine when the arguments are
    rc, *_ = vjp_call(flat, D, pc, dc, gc, L.SOFTPLUS, ws=ws, o=o, gp=gp, gd=gd)
    assert rc == 0 and bool(torch.isfinite(o[:M]).all() and torch.isfinite(gp[:M]).all() and torch.isfinite(gd[:M]).all()), err()
    rc, *_ = vjp_call(flat, D, pc, None, gc, L.SOFTPLUS | L.OCC_ONLY, ws=ws, o=o, gp=gp, g_dirs=False)
    assert rc == 0, err()


def _net(D=256, seed=3):
    import nope_nerf_b200.model as mdl
    cfg = FC.default_cfg(); cfg["model"]["hidden_dim"] = D
    torch.manual_seed(seed)
    return mdl.OfficialStaticNerf(cfg).cuda(), cfg


def logit_gated(W, p, gates):
    """tests/_normals_ref.logit with the ReLU of trunk layer l replaced by the fixed gate gates[l] (float64 0 / 1, rows x D)"""
    import _normals_ref as NR
    e = [p]
    for i in range(10):
        e += [torch.sin(2.0 ** i * p), torch.cos(2.0 ** i * p)]
    e = torch.cat(e, -1)
    x = e
    for l, (blk, i) in enumerate(NR.TRUNK):
        if l == 4:
            x = torch.cat([x, e], -1)
        x = (x @ W["%s.%d.weight" % (blk, i)].T + W["%s.%d.bias" % (blk, i)]) * gates[l]
    return x @ W["fc_density.weight"].T + W["fc_density.bias"]


@pytest.mark.parametrize("D", [64, 128, 256])
def test_gradient_engine_tc(D):
    """gradient(p, 0, engine='tc') under no_grad is the library call bit for bit and matches float64 normals; a call that needs the
    graph (grad mode on, p requiring grad) runs on the exact engine: it equals gradient(p, 0) bit for bit"""
    L, _ = _lib()
    net, _ = _net(D)
    P = O.init_params(seed=50 + D, D=D, hf_damp=True)   # well-conditioned gates (see the module docstring)
    net.load_state_dict({k: torch.from_numpy(np.asarray(P[k], np.float32)).reshape(v.shape) for k, v in net.state_dict().items()})
    M = 5000
    gen = torch.Generator().manual_seed(11)
    p = (torch.rand(M, 3, generator=gen) * 2 - 1).cuda()
    with torch.no_grad():
        n_tc = net.gradient(p, 0, engine="tc")
        n_ex = net.gradient(p, 0)
    assert n_tc.shape == (M, 1, 3) and not n_tc.requires_grad
    g = torch.zeros(M, 4, device="cuda"); g[:, 3] = 1.0
    flat = net.flat_weights()
    ws = torch.empty(L.lib.nnb_field_vjp_workspace_bytes(M, L.RAW_DENSITY | L.OCC_ONLY, D), dtype=torch.uint8, device="cuda")
    rc, _, gp, _ = vjp_call(flat, D, p, None, g, L.RAW_DENSITY | L.OCC_ONLY, out=False, g_dirs=False, ws=ws)
    assert rc == 0
    assert torch.equal(bits(n_tc[:, 0]), bits(-gp[:, :3]))
    # float64 normals: the reference's autograd of infer_occ (tests/_normals_ref.logit), each with the ReLU gates of the engine it is
    # compared with (see oracle64_backward); every gate that differs from float64's own sits within FLIP_DEPTH of 0
    rows = np.arange(M)
    _, _, cache = oracle64_forward(P, p.cpu().numpy(), None, "logit")
    _, ws_s, _ = field_fwd(flat, D, p, None, L.RAW_DENSITY | L.STASH, L.ENGINE_SIMT)   # the forward gradient()'s exact path runs
    torch.cuda.synchronize()
    W = {k: v.detach().double().cpu() for k, v in net.state_dict().items()}
    errs = {}
    for name, n, gates in (("tc", n_tc, tc_gates(ws, M, D, rows, True)), ("exact", n_ex, simt_gates(ws_s, M, D, rows)[:8])):
        pp = p.double().cpu().requires_grad_(True)
        n64, = torch.autograd.grad(logit_gated(W, pp, [torch.from_numpy(m).double() for m in gates]).sum(), pp)
        errs[name] = relmax(n[:, 0].cpu().numpy(), -n64.numpy())
        errs["flip_" + name] = flip_depth(gates, cache, True)
    print("gradient D=%d: against float64 with the engine's gates, engine='tc' %.2e, exact %.2e of the normals' maximum; deepest gate "
          "flip %.1e / %.1e of the layer's largest pre-activation" % (D, errs["tc"], errs["exact"], errs["flip_tc"], errs["flip_exact"]))
    assert errs["tc"] <= TOL and errs["exact"] <= TOL and errs["flip_tc"] <= FLIP_DEPTH and errs["flip_exact"] <= FLIP_DEPTH, errs
    assert not torch.equal(bits(n_tc), bits(n_ex))   # the engines differ in the last bits: the checks above can tell them apart
    # grad mode on and p requiring grad: the exact, differentiable path, whatever the engine
    pg = p.clone().requires_grad_(True)
    n1 = net.gradient(pg, 0, engine="tc")
    n0 = net.gradient(p.clone().requires_grad_(True), 0)
    assert n1.requires_grad and torch.equal(bits(n1.detach()), bits(n0.detach())) and torch.equal(bits(n1.detach()), bits(n_ex))
    # grad mode on, p a plain tensor: detached, so the tensor-core engine serves it
    n2 = net.gradient(p, 0, engine="tc")
    assert not n2.requires_grad and torch.equal(bits(n2), bits(n_tc))
    with torch.no_grad():
        assert net.gradient(p[:0], 0, engine="tc").shape == (0, 1, 3)


def _geometry_setup(cfg, net_seed=31):
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200.model import common as mc
    H, W, V = 24, 32, 4
    state = FC.start_state(cfg, V, net_seed, 95, geo=True)
    gold = dict(np.load(os.path.join(GOLDEN, "fullsize_phong.npz")))
    dev = torch.device("cuda")
    net = mdl.OfficialStaticNerf(cfg)
    net.load_state_dict({k: v.clone() for k, v in state["net"].items()})
    data = FC.small_scene(H, W, V=V)
    pixels = mc.arange_pixels((H, W), 1)[1].cuda()
    cam = data["img.camera_mat"].cuda(); smat = data["img.scale_mat"].cuda()
    pose = mdl.LearnPose(V, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.copy_(state["r"]); pose.t.copy_(state["t"])
        c2w = pose(int(gold["view"]))
    return net, pixels, cam, smat, c2w, gold, state


def _phong(net, cfg, pixels, cam, smat, c2w, fe, ne):
    import nope_nerf_b200.model as mdl
    rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), field_engine=fe, normal_engine=ne)
    assert rend.normal_engine == ne
    o = rend(pixels, None, cam, torch.inverse(c2w).unsqueeze(0), smat, "phong_renderer", it=0)
    return o["rgb"].detach().reshape(-1, 3).cpu(), o["rgb_surf"].detach().reshape(-1, 3).cpu()


def _criterion(ref, got):
    (rgb_ref, surf_ref), (rgb, surf) = ref, got
    bad = ((rgb_ref - rgb).abs().max(1).values > 2.0 / 255) | ((surf_ref - surf).abs().max(1).values > 2.0 / 255)
    return dict(frac_bad=float(bad.float().mean()), med_rgb=float((rgb_ref - rgb).abs().median()), med_surf=float((surf_ref - surf).abs().median()))


def test_geometry_view_normals_on_tensor_cores():
    """Renderer(field_engine='tc', normal_engine='tc') against the stored reference frame, by the criterion of
    test_gpu_field_tc.py::test_geometry_view_on_tensor_cores (<= 1 % of pixels off by more than 2/255, medians < 1e-4)"""
    cfg = FC.default_cfg()
    net, pixels, cam, smat, c2w, gold, state = _geometry_setup(cfg)
    assert abs(FC.state_digest(state) - float(gold["digest"])) <= 1e-9 * max(1.0, abs(float(gold["digest"])))
    got = _phong(net, cfg, pixels, cam, smat, c2w, "tc", "tc")
    e = _criterion((torch.as_tensor(gold["rgb"]), torch.as_tensor(gold["rgb_surf"])), got)
    print("phong_renderer field_engine=tc normal_engine=tc vs stored frame: %s" % e)
    assert e["frac_bad"] <= 0.01 and e["med_rgb"] < 1e-4 and e["med_surf"] < 1e-4, e
    assert float((got[1].abs().sum(1) > 0).float().mean()) > 0.02   # the scene has a visible surface


@pytest.mark.parametrize("D", [64, 128])
def test_geometry_view_normals_against_exact_engine(D):
    """at the narrower widths, against the exact engine's frame (field_engine=None) by the same criterion"""
    cfg = FC.default_cfg(); cfg["model"]["hidden_dim"] = D
    for seed in range(31, 41):   # the first seeded geometry field of width D whose surface the camera sees
        net, pixels, cam, smat, c2w, _, _ = _geometry_setup(cfg, seed)
        ex = _phong(net, cfg, pixels, cam, smat, c2w, None, None)
        if float((ex[1].abs().sum(1) > 0).float().mean()) > 0.02:
            break
    got = _phong(net, cfg, pixels, cam, smat, c2w, "tc", "tc")
    e = _criterion(ex, got)
    print("phong_renderer D=%d tc/tc vs exact engine: %s" % (D, e))
    assert e["frac_bad"] <= 0.01 and e["med_rgb"] < 1e-4 and e["med_surf"] < 1e-4, e
    assert float((ex[1].abs().sum(1) > 0).float().mean()) > 0.02   # the scene has a visible surface


def test_camera_rays_depend_on_the_chunk():
    """why rendering.GEOMETRY_CHUNK stays at the reference's 1024 pixels on every engine: every field query of the geometry view is
    independent of the chunk on the tensor-core engine, but the camera rays are not.  Renderer._rays_world's batched matmul T @ ph rounds
    differently with the number of pixels in the call, so a pixel's ray (and with it the frame's bits) changes with the chunk size."""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200.model.common import arange_pixels
    from nope_nerf_b200.model.rendering import GEOMETRY_CHUNK
    cfg = FC.default_cfg()
    net, _, cam, smat, c2w, _, _ = _geometry_setup(cfg)
    rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), field_engine="tc", normal_engine="tc")
    _, pixels = arange_pixels(resolution=(60, 80), device="cuda")   # 4800 pixels: one call against 1024-pixel chunks
    wm = torch.linalg.inv(c2w.detach().reshape(4, 4)).unsqueeze(0)
    cam = cam.reshape(1, 4, 4)
    with torch.no_grad():
        cw, rv = rend._rays_world(pixels, cam, wm, smat)
        parts = [rend._rays_world(px, cam, wm, smat) for px in torch.split(pixels, GEOMETRY_CHUNK, dim=1)]
    rv_chunked = torch.cat([q[1] for q in parts], dim=1)
    assert torch.allclose(rv, rv_chunked, rtol=0, atol=1e-6)
    assert not torch.equal(rv, rv_chunked), "the camera rays no longer depend on the chunk: GEOMETRY_CHUNK could be raised"

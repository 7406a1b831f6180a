"""GPU: explicit-point field queries on the tensor-core engine (nnb_field_fwd with NNB_ENGINE_TC, tc_points_fwd in csrc/nnb_tc.cu).

The kernel is the render path's split-fp16 forward fed with points instead of rays; what is new, and checked here, is the per-row view
direction (two more K-steps of the rgb hidden layer instead of a per-ray bias), the occupancy-only mode (NNB_OCC_ONLY), the row-bounded
float4 output, the argument checks, and the Python surface (field_query / OfficialStaticNerf.forward / Renderer(field_engine=)).

Reference: oracle/nerf_oracle.py's field in float64 at the fp32 points, directions and weights.  Bound: 1e-4 of the tensor's maximum
on rgb and on the fourth channel (DESIGN.md §2).  Largest measured over all cases below (NVIDIA H100 80GB HBM3, 700 W power limit):
6.3e-7 against float64 (the raw logit at D = 128; rgb 1.7e-7) and 7.7e-7 against the exact engine; run with -s to print them.
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
# one row, the 128-row tile's edges, more than one wave of 132 CTAs (132 * 128 = 16 896), many tiles per CTA
SIZES = (1, 127, 128, 129, 16901, 200003)
ORACLE_ROWS = 4096   # float64 rows checked at the sizes above it: a seeded draw plus the first row, the last, and the last tile's edges


def _lib():
    from nope_nerf_b200 import _lib as L, ops
    return L, ops


def field_call(flat, D, p, d, flags, engine, ws=None, out=None, ws_bytes=None):
    """one nnb_field_fwd call; returns (rc, out).  ws / out default to fresh buffers of the documented sizes."""
    L, ops = _lib()
    M = p.shape[0]
    if ws is None:
        ws = torch.empty(L.lib.nnb_workspace_bytes_dim(M, 1, flags, engine, D), dtype=torch.uint8, device="cuda")
    if out is None:
        out = torch.full((M, 4), float("nan"), device="cuda")
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p); a.dirs = L.ptr(d); a.N = M; a.S = 1; a.flags = flags; a.engine = engine; a.hidden_dim = D
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel() if ws_bytes is None else ws_bytes
    rc = L.lib.nnb_field_fwd(C.byref(a), L.ptr(out), ops._stream())
    torch.cuda.synchronize()
    return rc, out


def make_inputs(D, M, seed, with_dirs=True):
    rng = np.random.default_rng(seed)
    P = O.init_params(seed=7 + D, D=D)
    p = rng.uniform(-1.5, 1.5, (M, 3)).astype(np.float32)
    d = rng.normal(size=(M, 3)); d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    flat = torch.from_numpy(O.flatten_params(P)).cuda()
    return P, p, (d if with_dirs else None), flat


def oracle64(P, p, d, act):
    """(rgb (M,3), fourth channel (M,)) in float64 at the fp32 inputs"""
    P64 = {k: np.asarray(v, np.float64) for k, v in P.items()}
    dd = np.ones_like(p, dtype=np.float64) if d is None else d.astype(np.float64)
    rgb, a, cache = O.mlp_forward(P64, p.astype(np.float64), dd, dist_alpha=(act == "sigma"), occ_activation="softplus")
    return rgb, (cache["s"] if act == "logit" else a)


def act_flags(act):
    L, _ = _lib()
    return L.SOFTPLUS | {"alpha": 0, "sigma": L.DIST_ALPHA, "logit": L.RAW_DENSITY}[act]


def relmax(x, ref):
    return float(np.abs(np.asarray(x, np.float64) - ref).max() / max(np.abs(ref).max(), 1e-30))


@pytest.mark.parametrize("with_dirs", [True, False], ids=["dirs", "ones"])
@pytest.mark.parametrize("act", ["alpha", "sigma", "logit"])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_against_float64_and_exact_engine(D, act, with_dirs):
    L, _ = _lib()
    worst = dict(rgb64=0.0, a64=0.0, rgb_simt=0.0, a_simt=0.0)
    for M in SIZES:
        P, p, d, flat = make_inputs(D, M, seed=1000 + M, with_dirs=with_dirs)
        pc = torch.from_numpy(p).cuda(); dc = None if d is None else torch.from_numpy(d).cuda()
        rc, out = field_call(flat, D, pc, dc, act_flags(act), L.ENGINE_TC)
        assert rc == 0, L.lib.nnb_last_error()
        rc, ref = field_call(flat, D, pc, dc, act_flags(act), L.ENGINE_SIMT)
        assert rc == 0, L.lib.nnb_last_error()
        out, ref = out.cpu().numpy(), ref.cpu().numpy()
        assert np.isfinite(out).all()
        rows = np.arange(M)
        if M > ORACLE_ROWS:
            last_tile = (M - 1) // 128 * 128
            rows = np.unique(np.concatenate([np.random.default_rng(M).choice(M, ORACLE_ROWS, replace=False),
                                             [0, last_tile - 1, last_tile, M - 1]]))
        rgb64, a64 = oracle64(P, p[rows], None if d is None else d[rows], act)
        e = dict(rgb64=relmax(out[rows, :3], rgb64), a64=relmax(out[rows, 3], a64),
                 rgb_simt=relmax(out[:, :3], ref[:, :3].astype(np.float64)), a_simt=relmax(out[:, 3], ref[:, 3].astype(np.float64)))
        assert max(e.values()) <= TOL, (D, act, with_dirs, M, e)
        worst = {k: max(worst[k], e[k]) for k in worst}
    print("field_tc D=%d %s %s: vs float64 rgb %.2e a %.2e; vs exact engine rgb %.2e a %.2e"
          % (D, act, "dirs" if with_dirs else "ones", worst["rgb64"], worst["a64"], worst["rgb_simt"], worst["a_simt"]))


@pytest.mark.parametrize("D", [64, 128, 256])
def test_direction_is_per_row_permutation_is_bitwise(D):
    """every row has its own direction; a row's MMA sequence does not depend on where it sits, so permuting the rows permutes the
    output bit for bit.  A row that read a neighbour's direction or bias would break that.  M has a ragged last tile."""
    L, _ = _lib()
    M = 3 * 128 + 77
    P, p, d, flat = make_inputs(D, M, seed=5)
    perm = torch.from_numpy(np.random.default_rng(6).permutation(M)).cuda()
    pc, dc = torch.from_numpy(p).cuda(), torch.from_numpy(d).cuda()
    rc, out = field_call(flat, D, pc, dc, L.SOFTPLUS, L.ENGINE_TC)
    assert rc == 0, L.lib.nnb_last_error()
    rc, out_p = field_call(flat, D, pc[perm].contiguous(), dc[perm].contiguous(), L.SOFTPLUS, L.ENGINE_TC)
    assert rc == 0, L.lib.nnb_last_error()
    assert torch.equal(out[perm].view(torch.int32), out_p.view(torch.int32))
    # and the direction matters: the same points with one shared direction give another colour on most rows
    rc, out_1 = field_call(flat, D, pc, dc[:1].expand(M, 3).contiguous(), L.SOFTPLUS, L.ENGINE_TC)
    assert rc == 0
    assert torch.equal(out_1[0].view(torch.int32), out[0].view(torch.int32))
    assert float((out_1[:, :3] != out[:, :3]).any(dim=1).float().mean()) > 0.9
    assert torch.equal(out_1[:, 3].view(torch.int32), out[:, 3].view(torch.int32))   # the density does not see the direction


@pytest.mark.parametrize("act", ["alpha", "sigma", "logit"])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_occupancy_only_matches_full_query_bitwise(D, act):
    L, _ = _lib()
    for M in (1, 129, 16901):
        P, p, d, flat = make_inputs(D, M, seed=20 + M)
        pc, dc = torch.from_numpy(p).cuda(), torch.from_numpy(d).cuda()
        rc, full = field_call(flat, D, pc, dc, act_flags(act), L.ENGINE_TC)
        assert rc == 0, L.lib.nnb_last_error()
        rc, occ = field_call(flat, D, pc, None, act_flags(act) | L.OCC_ONLY, L.ENGINE_TC)
        assert rc == 0, L.lib.nnb_last_error()
        assert torch.equal(occ[:, 3].view(torch.int32), full[:, 3].view(torch.int32))
        assert torch.equal(occ[:, :3], torch.zeros_like(occ[:, :3]))


@pytest.mark.parametrize("occ", [False, True], ids=["full", "occ_only"])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_nothing_out_of_bounds_nothing_uninitialised(D, occ):
    """rows of out past M keep their sentinel; a workspace full of NaN bytes changes nothing (every byte the kernel reads was written
    by the call)"""
    L, _ = _lib()
    M, PAD, SENT = 2 * 128 + 5, 300, -12345.5
    P, p, d, flat = make_inputs(D, M, seed=31)
    pc, dc = torch.from_numpy(p).cuda(), torch.from_numpy(d).cuda()
    flags = L.SOFTPLUS | (L.OCC_ONLY if occ else 0)
    rc, clean = field_call(flat, D, pc, dc, flags, L.ENGINE_TC)
    assert rc == 0, L.lib.nnb_last_error()
    nbytes = L.lib.nnb_workspace_bytes_dim(M, 1, flags, L.ENGINE_TC, D)
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")
    buf = torch.full((M + PAD, 4), SENT, device="cuda")
    rc, _ = field_call(flat, D, pc, dc, flags, L.ENGINE_TC, ws=ws, out=buf)
    assert rc == 0, L.lib.nnb_last_error()
    assert torch.isfinite(buf[:M]).all()
    assert torch.equal(buf[:M].view(torch.int32), clean.view(torch.int32))
    assert torch.equal(buf[M:], torch.full((PAD, 4), SENT, device="cuda"))


def test_error_paths():
    L, _ = _lib()
    D, M = 64, 100
    P, p, d, flat = make_inputs(D, M, seed=41)
    pc = torch.from_numpy(p).cuda()
    err = lambda: L.lib.nnb_last_error().decode()
    nan_out = lambda o: bool(torch.isnan(o).all())   # a rejected call launches nothing
    rc, o = field_call(flat, D, pc, None, L.SOFTPLUS | L.STASH, L.ENGINE_TC)
    assert rc == -6 and "NNB_STASH" in err() and "SIMT" in err() and nan_out(o), (rc, err())
    rc, o = field_call(flat, D, pc, None, L.SOFTPLUS | L.OCC_ONLY, L.ENGINE_SIMT)
    assert rc == -6 and "NNB_OCC_ONLY" in err() and nan_out(o), (rc, err())
    need = L.lib.nnb_workspace_bytes_dim(M, 1, L.SOFTPLUS, L.ENGINE_TC, D)
    ws = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    rc, o = field_call(flat, D, pc, None, L.SOFTPLUS, L.ENGINE_TC, ws=ws, ws_bytes=need - 1)
    assert rc == -5 and "too small" in err() and str(need) in err() and nan_out(o), (rc, err())
    rc, o = field_call(flat, D, pc, None, L.SOFTPLUS, L.ENGINE_TC, ws=ws[16:], ws_bytes=need)
    assert rc == -5 and "aligned" in err() and nan_out(o), (rc, err())
    rc, o = field_call(flat, 96, pc, None, L.SOFTPLUS, L.ENGINE_TC, ws=ws)
    assert rc == -8 and "hidden_dim" in err() and nan_out(o), (rc, err())
    rc, o = field_call(flat, D, pc, None, L.SOFTPLUS, L.ENGINE_TC, ws=ws)   # and the same buffers are fine when the arguments are
    assert rc == 0 and bool(torch.isfinite(o).all()), (rc, err())


def test_removed_flag_bits_are_rejected():
    """the flag bits removed in version 105 (512, 1024, 4096, 8192) are rejected (rc -7) by every entry point that takes rendering
    flags, on every engine it serves.  The buffers are real, zeroed and sized for the same call without the bit, which succeeds
    first: a call that did not check the bit would run on valid memory."""
    L, ops = _lib()
    D, N, S, H, W = 64, 4, 32, 8, 8
    z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device="cuda")
    weights, g_weights = z(L.num_params(D)), z(L.num_params(D))
    c2w, cam, g_c2w = torch.eye(4, device="cuda"), torch.diag(torch.tensor([1.0, 1.0, -1.0, 1.0])).cuda(), z(4, 4)
    ray_idx, depth, g_rgb = z(N, dtype=torch.int64), z(N) + 1.0, z(N, 3)
    rgb, depth_pred, depth_gt, mask = z(N, 3), z(N), z(N), z(N, dtype=torch.uint8)
    pts, quad = z(N, 3), [z(N, 4) for _ in range(4)]   # quad: out_rgba / g_rgba / u, g_pts, g_dirs
    need = max(L.lib.nnb_workspace_bytes_dim(n, s, f, e, D) for n, s in ((N, S), (N, 1)) for e in (L.ENGINE_SIMT, L.ENGINE_TC)
               for f in (L.STASH, L.STASH | L.HVP))
    ws = z(need, dtype=torch.uint8)
    st = ops._stream()
    err = lambda: L.lib.nnb_last_error().decode()

    def render_args(flags, engine, fields=False):
        a = L.RenderArgs()
        a.weights, a.c2w, a.cam, a.ray_idx, a.depth = L.ptr(weights), L.ptr(c2w), L.ptr(cam), L.ptr(ray_idx), L.ptr(depth)
        a.N, a.S, a.H, a.W, a.near_, a.far_, a.flags, a.engine, a.hidden_dim = N, 1 if fields else S, H, W, 0.1, 4.0, flags, engine, D
        a.rgb, a.depth_pred, a.depth_gt, a.mask = L.ptr(rgb), L.ptr(depth_pred), L.ptr(depth_gt), L.ptr(mask)
        a.pts = L.ptr(pts) if fields else None
        a.workspace, a.workspace_bytes = L.ptr(ws), ws.numel()
        return a

    def render_bwd(flags, engine):
        b = L.RenderBwdArgs()
        b.fwd = render_args(flags, engine)
        b.g_rgb, b.g_weights, b.g_c2w = L.ptr(g_rgb), L.ptr(g_weights), L.ptr(g_c2w)
        return L.lib.nnb_render_bwd(C.byref(b), st)

    out, u, g_pts, g_dirs = (L.ptr(t) for t in quad)
    calls = []   # (name, valid flags, call(flags))
    for e in (L.ENGINE_SIMT, L.ENGINE_TC):
        calls += [("nnb_render_fwd/%d" % e, L.STASH, lambda f, e=e: L.lib.nnb_render_fwd(C.byref(render_args(f, e)), st)),
                  ("nnb_render_bwd/%d" % e, L.STASH, lambda f, e=e: render_bwd(f, e)),
                  ("nnb_debug_wgrad/%d" % e, L.STASH, lambda f, e=e: L.lib.nnb_debug_wgrad(C.byref(render_args(f, e)), L.ptr(g_weights), st)),
                  ("nnb_field_fwd/%d" % e, L.SOFTPLUS, lambda f, e=e: L.lib.nnb_field_fwd(C.byref(render_args(f, e, True)), out, st))]
    calls += [("nnb_field_bwd", L.STASH, lambda f: L.lib.nnb_field_bwd(C.byref(render_args(f, L.ENGINE_SIMT, True)), u, g_pts, g_dirs,
                                                                      L.ptr(g_weights), st)),
              ("nnb_field_hvp", L.STASH | L.HVP, lambda f: L.lib.nnb_field_hvp(C.byref(render_args(f, L.ENGINE_SIMT, True)), u, g_pts,
                                                                             L.ptr(g_weights), st))]
    for name, flags, call in calls:
        rc = call(flags)
        torch.cuda.synchronize()
        assert rc == 0, (name, rc, err())
        for bit in (512, 1024, 4096, 8192):
            rc = call(flags | bit)
            assert rc == -7 and "not defined" in err(), (name, bit, rc, err())
    torch.cuda.synchronize()


def _net(D=256, seed=3):
    import nope_nerf_b200.model as mdl
    cfg = FC.default_cfg(); cfg["model"]["hidden_dim"] = D
    torch.manual_seed(seed)
    return mdl.OfficialStaticNerf(cfg).cuda(), cfg


@pytest.mark.parametrize("D", [64, 256])
def test_python_surface(D):
    L, _ = _lib()
    net, cfg = _net(D)
    M = 1000
    g = torch.Generator().manual_seed(9)
    p = (torch.rand(M, 3, generator=g) * 3 - 1.5).cuda(); d = torch.nn.functional.normalize(torch.randn(M, 3, generator=g), dim=1).cuda()
    flags = (L.DIST_ALPHA if net.dist_alpha else 0) | (L.SOFTPLUS if net.occ_activation == "softplus" else 0)
    flat = net.flat_weights()
    bits = lambda t: t.contiguous().view(torch.int32)
    # engine='tc' without a gradient is the library call on the tensor-core engine
    with torch.no_grad():
        rgb, a = net(p, d, return_addocc=True, engine="tc")
        occ = net(p, only_occupancy=True, engine=L.ENGINE_TC)
        _, s = net.infer_occ(p, engine="tc")
    rc, c_out = field_call(flat, D, p, d, flags, L.ENGINE_TC)
    assert rc == 0
    assert rgb.shape == (M, 3) and a.shape == (M, 1) and occ.shape == (M, 1) and s.shape == (M, 1)
    assert torch.equal(bits(rgb), bits(c_out[:, :3])) and torch.equal(bits(a[:, 0]), bits(c_out[:, 3]))
    assert torch.equal(bits(occ), bits(a))
    rc, c_raw = field_call(flat, D, p, None, flags | L.RAW_DENSITY | L.OCC_ONLY, L.ENGINE_TC)
    assert rc == 0 and torch.equal(bits(s[:, 0]), bits(c_raw[:, 3]))
    # frozen parameters and plain inputs: no gradient is needed with grad mode on either
    for q in net.parameters(): q.requires_grad_(False)
    rgb_f = net(p, d, engine="tc")
    assert not rgb_f.requires_grad and torch.equal(bits(rgb_f), bits(rgb))
    for q in net.parameters(): q.requires_grad_(True)
    # no engine argument: the exact engine, bit for bit
    rc, c_simt = field_call(flat, D, p, d, flags, L.ENGINE_SIMT)
    assert rc == 0
    with torch.no_grad():
        rgb0, a0 = net(p, d, return_addocc=True)
    assert torch.equal(bits(rgb0), bits(c_simt[:, :3])) and torch.equal(bits(a0[:, 0]), bits(c_simt[:, 3]))
    assert not torch.equal(bits(rgb0), bits(rgb))   # the engines differ in the last bits: the checks above can tell them apart
    # a call that needs a gradient runs on the exact engine, whatever engine it names: same outputs, same gradients, bit for bit
    grads = []
    for engine in (None, "tc"):
        net.zero_grad(set_to_none=True)
        pg = p.clone().requires_grad_(True); dg = d.clone().requires_grad_(True)
        r_, a_ = net(pg, dg, return_addocc=True, engine=engine)
        assert r_.requires_grad and torch.equal(bits(r_.detach()), bits(c_simt[:, :3]))
        (r_.sum() + 2.0 * a_.sum()).backward()
        grads.append([pg.grad.clone(), dg.grad.clone()] + [q.grad.clone() for q in net.parameters()])
    assert all(torch.equal(bits(x), bits(y)) for x, y in zip(*grads))
    # no point: empty tensors, no library call
    with torch.no_grad():
        r_e, a_e = net(p[:0], d[:0], return_addocc=True, engine="tc")
    assert r_e.shape == (0, 3) and a_e.shape == (0, 1)
    with pytest.raises(ValueError):
        net(p, d, engine="tensor")


def test_geometry_view_on_tensor_cores():
    """Renderer(field_engine='tc') through phong_renderer (512-step ray marching, 8 secant steps, surface colour on the tensor-core
    engine; normals on gradient()) against the stored reference result, by the criterion of the exact engine's test: a pixel whose
    occupancy sits at the threshold may resolve to another march step, so at most 1 % of the pixels may differ by more than 2 / 255."""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200.model import common as mc
    cfg = FC.default_cfg()
    H, W, V = 24, 32, 4
    state = FC.start_state(cfg, V, 31, 95, geo=True)
    gold = dict(np.load(os.path.join(GOLDEN, "fullsize_phong.npz")))
    assert abs(FC.state_digest(state) - float(gold["digest"])) <= 1e-9 * max(1.0, abs(float(gold["digest"])))
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
    outs = {}
    for name, fe in (("exact", None), ("tc", "tc")):
        rend = mdl.Renderer(net, cfg["rendering"], device=dev, field_engine=fe)
        assert rend.field_engine == fe
        o = rend(pixels, None, cam, torch.inverse(c2w).unsqueeze(0), smat, "phong_renderer", it=0)
        outs[name] = (o["rgb"].detach().reshape(-1, 3).cpu(), o["rgb_surf"].detach().reshape(-1, 3).cpu())
    rgb_ref, surf_ref = torch.as_tensor(gold["rgb"]), torch.as_tensor(gold["rgb_surf"])
    for name, (rgb, surf) in outs.items():
        bad = ((rgb_ref - rgb).abs().max(1).values > 2.0 / 255) | ((surf_ref - surf).abs().max(1).values > 2.0 / 255)
        e = dict(frac_bad=float(bad.float().mean()), med_rgb=float((rgb_ref - rgb).abs().median()), med_surf=float((surf_ref - surf).abs().median()))
        print("phong_renderer field_engine=%s: %s" % (name, e))
        assert e["frac_bad"] <= 0.01 and e["med_rgb"] < 1e-4 and e["med_surf"] < 1e-4, (name, e)
    assert float((surf_ref.abs().sum(1) > 0).float().mean()) > 0.02   # the scene has a visible surface

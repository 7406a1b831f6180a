"""GPU: the fused ray march and the one-call geometry frame on the exact-fp32 engine (simt_march / simt_secant / simt_mlp_fwd_n /
simt_mlp_dgrad_n in csrc/nnb_simt.cu, nnb_ray_march_engine and nnb_geometry_frame_engine with NNB_ENGINE_SIMT; field.ray_march(engine='simt'),
field.geometry_frame(engine='simt'), Renderer(fused_march=True), Renderer(geometry_frame=True, geometry_frame_engine='simt')).

A point's exact-engine result does not depend on the tile or row that evaluates it, so every stage is checked bit for bit against the
default (exact) engine's own calls: the torch march Renderer._ray_marching_torch(engine=None), OfficialStaticNerf.gradient(p, it) and
OfficialStaticNerf.forward(p, -dir).  The fields and rays are those of test_gpu_ray_march.py and test_gpu_geometry_frame.py.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import _fullsize_cases as FC
from test_gpu_ray_march import geo_net, make_rays, expected, TAU, _raw_call
from test_gpu_geometry_frame import scene, T_of, pixels_of, frame, same, _mods, N_STEPS
from test_gpu_field_vjp import _criterion, _phong

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _release_workspaces():
    """the library's workspace pool keeps every size it has handed out; drop the ones this module added (a 1080p frame among them), so
    that the memory is free for the modules that run after it"""
    ops = _mods()[2]
    before = {k: len(v) for k, v in ops._pool.free.items()}
    yield
    for k in list(ops._pool.free):
        del ops._pool.free[k][before.get(k, 0):]
    torch.cuda.empty_cache()


def exact_values(net, ray0, dirs, far, n_steps):
    frac = torch.linspace(0, 1, steps=n_steps, device="cuda").view(1, n_steps)
    t = 0. * (1. - frac) + far.view(-1, 1) * frac
    p = ray0.unsqueeze(1) + dirs.unsqueeze(1) * t.unsqueeze(-1)
    with torch.no_grad():
        val = net(p.reshape(1, -1, 3), only_occupancy=True).reshape(-1, n_steps) - TAU
    return val.cpu().numpy(), t.cpu().numpy()


def torch_march(D, ray0, dirs, far, n_steps, n_secant):
    net, rend, cfg, _ = geo_net(D)
    rend._sphere_far = lambda cam_loc, d, r: far.view(1, -1)
    try:
        with torch.no_grad():
            return rend._ray_marching_torch(ray0[None], dirs[None], net, n_steps, n_secant, [0., 2.4], 3500000, 1.0, None)[0]
    finally:
        del rend._sphere_far


def exact_march(D, ray0, dirs, far, n_steps, n_secant):
    field = _mods()[3]
    frac = torch.linspace(0, 1, steps=n_steps, device="cuda")
    out = field.ray_march(geo_net(D)[0], ray0, dirs, far, frac, 0.0, n_secant, TAU, want_bracket=True, engine="simt")
    torch.cuda.synchronize()
    return out


def check(D, ray0, dirs, far, n_steps, n_secant):
    net = geo_net(D)[0]
    depth, first, bracket, counts = exact_march(D, ray0, dirs, far, n_steps, n_secant)
    ref = torch_march(D, ray0, dirs, far, n_steps, n_secant)
    assert torch.equal(depth.view(torch.int32), ref.view(torch.int32)), (D, n_steps, n_secant, int((depth != ref).sum()))
    val, t = exact_values(net, ray0, dirs, far, n_steps)
    e_first, hit, v0neg, br = expected(val, t)
    assert np.array_equal(first.cpu().numpy(), e_first)
    b = bracket.cpu().numpy()
    assert np.array_equal(b[hit].view(np.int32), br[hit].astype(np.float32).view(np.int32))
    assert not b[~hit].any()
    return depth, first, counts


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("n_steps,n_secant", [(2, 8), (129, 0), (512, 8)])
def test_march_is_the_torch_march_bit_for_bit(D, n_steps, n_secant):
    ray0, dirs, far = make_rays(D, 4096 + 37, seed=D + n_steps)
    depth, first, counts = check(D, ray0, dirs, far, n_steps, n_secant)
    d = depth.cpu()
    n_hit, n_occ, n_inf = int((torch.isfinite(d) & (d != 0)).sum()), int((d == 0).sum()), int(torch.isinf(d).sum())
    f = first.cpu()
    print("D=%d n_steps=%d: hit %d occupied %d miss %d, later-round hits %d, counts %s" %
          (D, n_steps, n_hit, n_occ, n_inf, int((f >= 127).sum()), counts.tolist()))
    if n_steps == 512:
        assert n_hit > 0 and n_occ > 0 and n_inf > 0 and int((f >= 127).sum()) > 0


@pytest.mark.parametrize("flags", ["relu", "dist_alpha", "relu_dist_alpha"])
def test_march_heads(flags):
    net = geo_net(64)[0]
    keep = (net.occ_activation, net.dist_alpha)
    try:
        net.occ_activation = "relu" if "relu" in flags else "softplus"
        net.dist_alpha = "dist_alpha" in flags
        ray0, dirs, far = make_rays(64, 4096, seed=7)
        check(64, ray0, dirs, far, 512, 8)
    finally:
        net.occ_activation, net.dist_alpha = keep


def test_march_sizes():
    ray0, dirs, far = make_rays(128, 4000, seed=3)
    for n in (1, 63, 65, 1001):
        check(128, ray0[-n:].contiguous(), dirs[-n:].contiguous(), far[-n:].contiguous(), 512, 8)
    depth, first, bracket, counts = exact_march(128, ray0[:0], dirs[:0], far[:0], 512, 8)
    assert depth.shape == (0,) and int(counts.sum()) == 0


def _engine_call(L, ops, net, engine, N=8, n_steps=16, hidden_dim=None, ws_bytes=None):
    """nnb_ray_march_engine on a small batch of rays, with a workspace of ws_bytes (default: the engine's size)"""
    t = dict(ray0=torch.zeros(N, 3, device="cuda"), dirs=torch.ones(N, 3, device="cuda"), far=torch.ones(N, device="cuda"),
             frac=torch.linspace(0, 1, n_steps, device="cuda"), depth=torch.full((N,), -7.0, device="cuda"))
    need = L.lib.nnb_ray_march_workspace_bytes_engine(N, n_steps, net.hidden_dim, L.ENGINE_SIMT)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    a = L.RayMarchArgs()
    a.weights = L.ptr(net.flat_weights()); a.ray0 = L.ptr(t["ray0"]); a.ray_dir = L.ptr(t["dirs"]); a.far_ = L.ptr(t["far"])
    a.frac = L.ptr(t["frac"]); a.N = N; a.n_steps = n_steps; a.n_secant = 2; a.hidden_dim = net.hidden_dim if hidden_dim is None else hidden_dim
    a.near_ = 0.0; a.tau = TAU; a.flags = L.SOFTPLUS; a.engine = engine
    a.depth = L.ptr(t["depth"]); a.workspace = L.ptr(ws); a.workspace_bytes = need if ws_bytes is None else ws_bytes
    rc = L.lib.nnb_ray_march_engine(C.byref(a), ops._stream())
    torch.cuda.synchronize()
    return rc, t["depth"], need


def test_march_argument_checks():
    L, ops = _mods()[1:3]
    net = geo_net(64)[0]
    rc, depth, need = _engine_call(L, ops, net, L.ENGINE_SIMT)
    assert rc == 0 and not (depth == -7.0).any()
    for kw in (dict(engine=2), dict(engine=L.ENGINE_SIMT, hidden_dim=96), dict(engine=L.ENGINE_SIMT, ws_bytes=need - 1)):
        rc, depth, _ = _engine_call(L, ops, net, **kw)
        assert rc < 0 and (depth == -7.0).all(), kw
    # the tensor-core call keeps rejecting the exact engine, whatever its workspace
    rc, depth, _ = _raw_call(L, ops, net, engine=L.ENGINE_SIMT)
    assert rc == -4 and (depth == -7.0).all()


# ---- the frame ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 128, 256])
def test_frame_stages_bit_for_bit(D):
    field = _mods()[3]
    net, cfg, cam, smat, c2w = scene(D)
    T, px = T_of(cam, c2w, smat), pixels_of(60, 80)
    rgb, surf, it = frame(net, T, px, engine="simt")
    _, _, it_tc = frame(net, T, px)
    for k in ("ray0", "ray_dir", "far"):
        assert same(it[k], it_tc[k]), k
    ray0, rd, far, depth, grad = it["ray0"], it["ray_dir"], it["far"], it["depth"], it["grad"]
    frac = torch.linspace(0, 1, N_STEPS, device="cuda")
    with torch.no_grad():
        assert same(depth, field.ray_march(net, ray0, rd, far, frac, 0.0, 8, 0.5, engine="simt"))
        obj = torch.isfinite(depth) & (depth != 0)
        assert int(obj.sum()) > 0
        p = ray0 + rd * depth.unsqueeze(-1)
        assert same(grad[obj], net.gradient(p[obj], 0)[:, 0])
        assert same(surf[obj], net(p[obj], -rd[obj]))
        # geo_shade's arithmetic from the grad it wrote, each operation rounded on its own in the documented order
        g = grad[obj]; c = T.reshape(4, 4)[:3, 3]
        dot = lambda u, v: (u[..., 0] * v[..., 0] + u[..., 1] * v[..., 1]) + u[..., 2] * v[..., 2]
        n = g / torch.sqrt(dot(g, g)).unsqueeze(-1); l = c / torch.sqrt(dot(c, c))
        s = (0.3 + dot(n, l.expand_as(n)).clamp_min(0) * 0.7).clamp_max(1.0)
        assert same(rgb[obj], s.unsqueeze(-1).expand(-1, 3).contiguous())
    assert bool((rgb[~obj] == 1).all()) and bool((surf[~obj] == 0).all()) and bool((grad[~obj] == 0).all())
    print("D=%d: %d of %d pixels on the surface" % (D, int(obj.sum()), obj.numel()))


def test_frame_is_independent_of_the_split():
    net, cfg, cam, smat, c2w = scene(128)
    T, px = T_of(cam, c2w, smat), pixels_of(60, 80).reshape(-1, 2)
    whole = frame(net, T, px, engine="simt")[:2]
    parts = [frame(net, T, px[a:b], engine="simt")[:2] for a, b in ((0, 1234), (1234, 1300), (1300, px.shape[0]))]
    for k in range(2):
        assert same(whole[k], torch.cat([q[k] for q in parts]))
    perm = torch.randperm(px.shape[0], generator=torch.Generator().manual_seed(1)).cuda()
    pp = frame(net, T, px[perm], engine="simt")[:2]
    again = frame(net, T, px, engine="simt")[:2]
    for k in range(2):
        assert same(pp[k], whole[k][perm]) and same(again[k], whole[k])


def test_1080p_row_band_alone():
    net, cfg, cam, smat, c2w = scene(256)
    T = T_of(cam, c2w, smat)
    px = pixels_of(1080, 1920).reshape(1080, 1920, 2)
    band = px[500:540].reshape(-1, 2)
    full = frame(net, T, px.reshape(-1, 2), engine="simt")[:2]
    alone = frame(net, T, band, engine="simt")[:2]
    for k in range(2):
        assert same(full[k].reshape(1080, 1920, 3)[500:540].reshape(-1, 3), alone[k])


@pytest.mark.parametrize("D", [64, 256])
def test_frame_against_the_chunked_default(D):
    """Renderer(geometry_frame=True, geometry_frame_engine='simt') against the chunked exact phong_renderer: they differ only through the
    chunked path's batched-matmul rays; gated as test_gpu_geometry_frame.py gates the tensor-core frame"""
    mdl = _mods()[0]
    net, cfg, cam, smat, c2w = scene(D)
    pixels = pixels_of(24, 32)
    ex = _phong(net, cfg, pixels, cam, smat, c2w, None, None)
    rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), geometry_frame=True, geometry_frame_engine="simt")
    o = rend(pixels, None, cam, torch.inverse(c2w).unsqueeze(0), smat, "phong_renderer", it=0)
    e = _criterion(ex, (o["rgb"].reshape(-1, 3).cpu(), o["rgb_surf"].reshape(-1, 3).cpu()))
    print("exact frame D=%d vs chunked exact phong_renderer: %s" % (D, e))
    assert e["frac_bad"] <= 0.01 and e["med_rgb"] < 1e-4 and e["med_surf"] < 1e-4, e


def test_fused_march_renderer_gives_the_default_bits():
    mdl = _mods()[0]
    net, cfg, cam, smat, c2w = scene(128)
    pixels = pixels_of(24, 32)
    outs = []
    for kw in (dict(), dict(fused_march=True)):
        rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), **kw)
        torch.manual_seed(5)
        o = rend(pixels, None, cam, torch.inverse(c2w).unsqueeze(0), smat, "phong_renderer", it=0)
        outs.append((o["rgb"], o["rgb_surf"], torch.rand(1, device="cuda")))
    for a, b in zip(*outs):
        assert same(a, b)


def test_render_geometry_caller():
    """Extract_Images.render_geometry with the exact frame: one library frame, the image within the gate of the chunked exact path"""
    mdl = _mods()[0]
    from nope_nerf_b200.model.extracting_images import Extract_Images
    net, cfg, cam, smat, c2w = scene(64)
    imgs = []
    for kw in (dict(), dict(geometry_frame=True, geometry_frame_engine="simt")):
        rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), **kw)
        ex = Extract_Images(rend, dict(cfg, extract_images={"resolution": (24, 32)}), device=torch.device("cuda"))
        imgs.append(np.asarray(ex.render_geometry(c2w, cam.reshape(1, 4, 4), smat.reshape(1, 4, 4), 24, 32, it=0)).astype(np.float32))
    bad = (np.abs(imgs[0] - imgs[1]).max(-1) > 2).mean()
    print("render_geometry: share of pixels off by more than 2/255: %.4f" % bad)
    assert bad <= 0.01


def _direct(net, T, px, word, engine):
    L, ops, field = _mods()[1:4]
    N = px.shape[0]
    frac = torch.linspace(0, 1, N_STEPS, device="cuda")
    need = L.lib.nnb_geometry_frame_workspace_bytes_engine(N, N_STEPS, net.hidden_dim, engine)
    ws = torch.empty(need // 4 + 64, dtype=torch.int32, device="cuda").fill_(word)
    rgb = torch.empty(N, 3, device="cuda"); surf = torch.empty(N, 3, device="cuda")
    a = L.GeometryArgs()
    keep = [net.flat_weights(), T.reshape(16).contiguous(), px.contiguous(), frac]
    a.weights, a.T, a.pixels, a.frac = [L.ptr(t) for t in keep]
    a.N = N; a.n_steps = N_STEPS; a.n_secant = 8; a.hidden_dim = net.hidden_dim; a.near_ = 0.0; a.tau = 0.5
    a.radius = float(FC.default_cfg()["rendering"]["radius"]); a.flags = field._field_flags(net); a.engine = engine
    a.rgb = L.ptr(rgb); a.rgb_surf = L.ptr(surf); a.workspace = L.ptr(ws); a.workspace_bytes = need
    rc = L.lib.nnb_geometry_frame_engine(C.byref(a), ops._stream())
    torch.cuda.synchronize()
    return rc, rgb, surf, need


@pytest.mark.parametrize("D", [64, 256])
def test_poisoned_workspace_and_checks(D):
    L = _mods()[1]
    net, cfg, cam, smat, c2w = scene(D)
    T, px = T_of(cam, c2w, smat), pixels_of(24, 32).reshape(-1, 2)
    outs = [_direct(net, T, px, w, L.ENGINE_SIMT) for w in (0, 0x7fc00000, 0x7f000000)]
    assert all(o[0] == 0 for o in outs)
    for o in outs[1:]:
        assert same(o[1], outs[0][1]) and same(o[2], outs[0][2])
    ref = frame(net, T, px, engine="simt")[:2]
    assert same(outs[0][1], ref[0]) and same(outs[0][2], ref[1])
    # undersized, bad flags and unknown engines are rejected before anything runs
    need = outs[0][3]
    a_rc = _direct_rc(net, T, px, L.ENGINE_SIMT, need - 1, 0)
    assert a_rc == -5
    assert _direct_rc(net, T, px, L.ENGINE_SIMT, need, L.NDC) == -6
    assert _direct_rc(net, T, px, 3, need, 0) == -4


def _direct_rc(net, T, px, engine, nbytes, flags):
    L, ops = _mods()[1:3]
    N = px.shape[0]
    frac = torch.linspace(0, 1, N_STEPS, device="cuda")
    ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device="cuda")
    rgb = torch.empty(N, 3, device="cuda"); surf = torch.empty(N, 3, device="cuda")
    a = L.GeometryArgs()
    keep = [net.flat_weights(), T.reshape(16).contiguous(), px.contiguous(), frac]
    a.weights, a.T, a.pixels, a.frac = [L.ptr(t) for t in keep]
    a.N = N; a.n_steps = N_STEPS; a.n_secant = 8; a.hidden_dim = net.hidden_dim; a.near_ = 0.0; a.tau = 0.5; a.radius = 4.0
    a.flags = flags; a.engine = engine; a.rgb = L.ptr(rgb); a.rgb_surf = L.ptr(surf); a.workspace = L.ptr(ws); a.workspace_bytes = nbytes
    rc = L.lib.nnb_geometry_frame_engine(C.byref(a), ops._stream())
    torch.cuda.synchronize()
    return rc

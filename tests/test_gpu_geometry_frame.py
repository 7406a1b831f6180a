"""GPU: the geometry view of any set of pixels in one tensor-core call (nnb_geometry_frame: geo_rays / geo_compact / geo_shade and the
device-count forms of tc_points_fwd, tc_points_vjp_fwd and tc_points_vjp in csrc/nnb_tc.cu; field.geometry_frame;
Renderer.phong_frame and Renderer(geometry_frame=True) through Extract_Images.render_geometry and Trainer.render_visdata).

The march, the normals and the surface colour are the existing tensor-core kernels, so the call's stages are checked bit for bit against
field.ray_march, OfficialStaticNerf.gradient(engine='tc') and OfficialStaticNerf.forward(engine='tc') run on the call's own rays.  Its
own arithmetic (rays, far sphere depth, shading) is checked against float64 from the call's inputs and intermediates.  The scenes and
fields are those of test_gpu_field_vjp.py (_geometry_setup).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import _fullsize_cases as FC
from test_gpu_field_vjp import _criterion, _geometry_setup, _phong

pytestmark = pytest.mark.gpu

N_STEPS = 512
EPS = 2.0 ** -23   # ulp of 1.0 in float32


def _mods():
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import _lib as L, ops, field
    from nope_nerf_b200.model import common as mc
    return mdl, L, ops, field, mc


def bits(t):
    return t.contiguous().view(torch.int32)


def same(a, b):
    return torch.equal(bits(a), bits(b))


_scenes = {}


def scene(D):
    """(net, cfg, cam, smat, c2w): D = 256 the stored frame's field and view; 64 / 128 the first seeded field of that width whose surface
    the camera sees (the seed search of test_geometry_view_normals_against_exact_engine)"""
    if D not in _scenes:
        cfg = FC.default_cfg(); cfg["model"]["hidden_dim"] = D
        for seed in ([31] if D == 256 else range(31, 41)):
            net, pixels, cam, smat, c2w, _, _ = _geometry_setup(cfg, seed)
            net = net.cuda()
            rgb, surf = frame(net, T_of(cam, c2w, smat), pixels)[:2]
            if float((surf.abs().sum(1) > 0).float().mean()) > 0.02:
                break
        _scenes[D] = (net, cfg, cam, smat, c2w)
    return _scenes[D]


def T_of(cam, c2w, smat):
    mdl = _mods()[0]
    return mdl.Renderer._ray_transform(cam.reshape(1, 4, 4), torch.inverse(c2w).reshape(1, 4, 4), smat.reshape(1, 4, 4), torch.device("cuda"))


def pixels_of(H, W):
    return _mods()[4].arange_pixels((H, W), 1)[1].cuda()


def frame(net, T, pixels, radius=None, **kw):
    field = _mods()[3]
    frac = torch.linspace(0, 1, N_STEPS, device="cuda")
    r = FC.default_cfg()["rendering"]["radius"] if radius is None else radius
    with torch.no_grad():
        out = field.geometry_frame(net, T, pixels, frac, r, want_intermediates=True, **kw)
    torch.cuda.synchronize()
    return out


def _all(out):
    rgb, surf, it = out
    return dict(rgb=rgb, rgb_surf=surf, **it)


# ---- 1. against the stored reference frame, and the exact engine's frame --------------------------------------------------------------
def test_phong_frame_against_stored_frame():
    """Renderer(geometry_frame=True) on the fullsize_phong.npz scene, by the criterion of test_geometry_view_normals_on_tensor_cores"""
    mdl = _mods()[0]
    cfg = FC.default_cfg()
    net, pixels, cam, smat, c2w, gold, state = _geometry_setup(cfg)
    assert abs(FC.state_digest(state) - float(gold["digest"])) <= 1e-9 * max(1.0, abs(float(gold["digest"])))
    rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), geometry_frame=True)
    o = rend(pixels, None, cam, torch.inverse(c2w).unsqueeze(0), smat, "phong_renderer", it=0)
    assert o["normal"] is None and o["rgb"].shape == (1, pixels.shape[1], 3) and o["rgb_surf"].shape == (1, pixels.shape[1], 3)
    got = (o["rgb"].reshape(-1, 3).cpu(), o["rgb_surf"].reshape(-1, 3).cpu())
    e = _criterion((torch.as_tensor(gold["rgb"]), torch.as_tensor(gold["rgb_surf"])), got)
    print("phong_frame D=256 vs stored frame: %s" % e)
    assert e["frac_bad"] <= 0.01 and e["med_rgb"] < 1e-4 and e["med_surf"] < 1e-4, e
    assert float((got[1].abs().sum(1) > 0).float().mean()) > 0.02


@pytest.mark.parametrize("D", [64, 128])
def test_phong_frame_against_exact_engine(D):
    mdl = _mods()[0]
    net, cfg, cam, smat, c2w = scene(D)
    pixels = pixels_of(24, 32)
    ex = _phong(net, cfg, pixels, cam, smat, c2w, None, None)
    rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), geometry_frame=True)
    o = rend.phong_frame(pixels, cam, torch.inverse(c2w).unsqueeze(0), smat, 0)
    e = _criterion(ex, (o["rgb"].reshape(-1, 3).cpu(), o["rgb_surf"].reshape(-1, 3).cpu()))
    print("phong_frame D=%d vs exact engine: %s" % (D, e))
    assert e["frac_bad"] <= 0.01 and e["med_rgb"] < 1e-4 and e["med_surf"] < 1e-4, e
    assert float((ex[1].abs().sum(1) > 0).float().mean()) > 0.02


# ---- 2. stage bits ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 128, 256])
def test_stages_are_the_existing_kernels_bit_for_bit(D):
    field = _mods()[3]
    net, cfg, cam, smat, c2w = scene(D)
    rgb, surf, it = frame(net, T_of(cam, c2w, smat), pixels_of(60, 80))
    ray0, rd, far, depth, grad = it["ray0"], it["ray_dir"], it["far"], it["depth"], it["grad"]
    frac = torch.linspace(0, 1, N_STEPS, device="cuda")
    with torch.no_grad():
        assert same(depth, field.ray_march(net, ray0, rd, far, frac, 0.0, 8, 0.5))
        obj = torch.isfinite(depth) & (depth != 0)
        p = ray0 + rd * depth.unsqueeze(-1)
        assert int(obj.sum()) > 0   # misses: the edge-case tests below
        assert same(grad[obj], net.gradient(p[obj], 0, engine="tc")[:, 0])
        assert same(surf[obj], net(p[obj], -rd[obj], engine="tc"))
    assert bool((rgb[~obj] == 1).all()) and bool((surf[~obj] == 0).all()) and bool((grad[~obj] == 0).all())
    print("D=%d: %d of %d pixels on the surface" % (D, int(obj.sum()), obj.numel()))


# ---- 3. against float64 ---------------------------------------------------------------------------------------------------------------
def test_rays_far_and_shading_against_float64():
    mdl = _mods()[0]
    net, cfg, cam, smat, c2w = scene(256)
    pixels = pixels_of(60, 80)
    T = T_of(cam, c2w, smat)
    rgb, surf, it = frame(net, T, pixels)
    T64 = T.reshape(4, 4).double().cpu()
    px = pixels.reshape(-1, 2).double().cpu()
    ph = torch.cat([px, torch.ones(px.shape[0], 2, dtype=torch.float64)], 1)
    pw64 = ph @ T64.t()
    cw64 = T64[:3, 3]
    d64 = pw64[:, :3] - cw64
    dir64 = d64 / d64.norm(dim=1, keepdim=True)
    assert torch.equal(it["ray0"].cpu(), T.reshape(4, 4)[:3, 3].cpu().expand(px.shape[0], 3))
    # a few ulp of the largest term of each component (pw and cw cancel in d = pw - cw), relative to |d|
    scale = torch.maximum(pw64[:, :3].abs(), cw64.abs()).amax(1, keepdim=True) / d64.norm(dim=1, keepdim=True) + 1.0
    ulps = float(((it["ray_dir"].double().cpu() - dir64).abs() / (EPS * scale)).max())
    # far from the call's own rays
    rd = it["ray_dir"].double().cpu()
    r = float(cfg["rendering"]["radius"])
    dot = rd @ cw64
    under = dot ** 2 - (cw64 @ cw64 - r * r)
    far64 = torch.where(under > 0, under.clamp_min(0).sqrt() - dot, torch.zeros_like(dot)).clamp_min(0)
    far = it["far"].double().cpu()
    clear = under > 1e-2 * r * r                               # not near-tangent
    far_rel = float(((far - far64).abs() / far64.clamp_min(1e-30))[clear & (far64 > 0)].max())
    assert bool((far[under < -1e-2 * r * r] == 0).all())
    # shading of the returned gradient on the object rays
    depth = it["depth"].cpu()
    obj = torch.isfinite(depth) & (depth != 0)
    g = it["grad"].double().cpu()[obj]
    n = g / g.norm(dim=1, keepdim=True)
    light = cw64 / cw64.norm()
    s64 = (float(np.float32(0.3)) + float(np.float32(0.7)) * (n @ light).clamp_min(0)).clamp_max(1.0)
    shade = float((rgb.double().cpu()[obj] - s64.unsqueeze(1)).abs().max())
    # against the chunked path's rays on the whole frame
    with torch.no_grad():
        cw_r, rv_r = mdl.Renderer._rays_world(pixels, cam.reshape(1, 4, 4), torch.inverse(c2w).reshape(1, 4, 4), smat.reshape(1, 4, 4))
    vs_torch = max(float((it["ray_dir"] - rv_r[0]).abs().max()), float((it["ray0"] - cw_r[0]).abs().max()))
    print("rays %.2f ulp, far %.2e relative, shading %.2e, rays vs _rays_world %.2e, %d object rays" % (ulps, far_rel, shade, vs_torch, int(obj.sum())))
    assert ulps <= 4 and far_rel <= 1e-6 and shade <= 1e-6 and vs_torch <= 1e-6 and int(obj.sum()) > 0


# ---- 4. pixel independence -------------------------------------------------------------------------------------------------------------
def test_pixels_are_independent_of_the_call():
    net, cfg, cam, smat, c2w = scene(256)
    T = T_of(cam, c2w, smat)
    pixels = pixels_of(60, 80)
    N = pixels.shape[1]
    whole = _all(frame(net, T, pixels))
    again = _all(frame(net, T, pixels))
    cuts = (0, 37, 2900, N)
    parts = [_all(frame(net, T, pixels[:, a:b])) for a, b in zip(cuts[:-1], cuts[1:])]
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(5)).cuda()
    permuted = _all(frame(net, T, pixels[:, perm]))
    inv = torch.empty_like(perm); inv[perm] = torch.arange(N, device="cuda")
    for k, v in whole.items():
        assert same(v, again[k]), k
        assert same(v, torch.cat([q[k] for q in parts])), k
        assert same(v, permuted[k][inv]), k


# ---- 5. edge cases ------------------------------------------------------------------------------------------------------------------
def _shifted_net(D, bias):
    mdl = _mods()[0]
    net, cfg, _, _, _ = scene(D)
    other = mdl.OfficialStaticNerf(cfg)
    other.load_state_dict({k: v.clone() for k, v in net.state_dict().items()})
    with torch.no_grad():
        other.fc_density.bias.fill_(bias)
    return other.cuda()


@pytest.mark.parametrize("bias,expect", [(-1e4, "inf"), (1e4, "zero")])
def test_no_surface_and_camera_inside(bias, expect):
    """a field with no surface (occupancy 0 everywhere: every depth is inf), and a camera inside the occupied region (every depth 0):
    every pixel 1 / 0"""
    _, _, cam, smat, c2w = scene(256)
    rgb, surf, it = frame(_shifted_net(256, bias), T_of(cam, c2w, smat), pixels_of(24, 32))
    d = it["depth"]
    assert bool(torch.isinf(d).all()) if expect == "inf" else bool((d == 0).all())
    assert bool((rgb == 1).all()) and bool((surf == 0).all())


def test_rays_that_miss_the_sphere():
    net, cfg, cam, smat, c2w = scene(256)
    T = T_of(cam, c2w, smat)
    cw = T.reshape(4, 4)[:3, 3]
    rgb, surf, it = frame(net, T, pixels_of(24, 32), radius=0.05 * float(cw.norm()))
    rd = it["ray_dir"].double()
    dot = rd @ cw.double()
    under = dot ** 2 - (cw.double() @ cw.double() - (0.05 * float(cw.norm())) ** 2)
    miss = under < -1e-3 * float(cw.double() @ cw.double())
    assert 0 < int(miss.sum())
    assert bool((it["far"][miss] == 0).all()) and bool((rgb[miss] == 1).all()) and bool((surf[miss] == 0).all())


def test_small_and_empty_calls():
    mdl, L, ops, field, _ = _mods()
    net, cfg, cam, smat, c2w = scene(256)
    T = T_of(cam, c2w, smat)
    pixels = pixels_of(24, 32)
    whole = _all(frame(net, T, pixels))
    hit = int(torch.nonzero(torch.isfinite(whole["depth"]) & (whole["depth"] != 0))[0])
    for a, b in ((hit, hit + 1), (0, 1), (100, 229)):   # N = 1 (an object ray, then the corner), N = 129
        part = _all(frame(net, T, pixels[:, a:b]))
        for k, v in whole.items():
            assert same(v[a:b], part[k]), (a, b, k)
    rgb, surf, it = frame(net, T, pixels[:, :0])
    assert rgb.shape == (0, 3) and surf.shape == (0, 3) and it["depth"].shape == (0,)
    a = L.GeometryArgs(); a.N = 0; a.n_steps = N_STEPS; a.engine = L.ENGINE_TC; a.hidden_dim = 256
    assert L.lib.nnb_geometry_frame(C.byref(a), ops._stream()) == 0   # nothing to launch, nothing read


# ---- 6. workspace poison ------------------------------------------------------------------------------------------------------------
def _direct(net, T, pixels, word):
    _, L, ops, _, _ = _mods()
    N = pixels.shape[1]
    frac = torch.linspace(0, 1, N_STEPS, device="cuda")
    nbytes = L.lib.nnb_geometry_frame_workspace_bytes(N, N_STEPS, net.hidden_dim)
    ws = torch.empty((nbytes + 255) // 256 * 256, dtype=torch.uint8, device="cuda")
    ws.view(torch.int32).fill_(word)
    nan = lambda *s: torch.full(s, float("nan"), device="cuda")
    out = dict(rgb=nan(N, 3), rgb_surf=nan(N, 3), ray0=nan(N, 3), ray_dir=nan(N, 3), far_=nan(N), depth=nan(N), grad=nan(N, 4))
    px = pixels.reshape(-1, 2).contiguous(); Tc = T.reshape(16).contiguous()
    a = L.GeometryArgs()
    a.weights = L.ptr(net.flat_weights()); a.T = L.ptr(Tc); a.pixels = L.ptr(px); a.frac = L.ptr(frac)
    a.N = N; a.n_steps = N_STEPS; a.n_secant = 8; a.hidden_dim = net.hidden_dim; a.near_ = 0.0; a.tau = 0.5
    a.radius = float(FC.default_cfg()["rendering"]["radius"]); a.flags = 0; a.engine = L.ENGINE_TC
    for k, v in out.items():
        setattr(a, k, L.ptr(v))
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    assert L.lib.nnb_geometry_frame(C.byref(a), ops._stream()) == 0, L.lib.nnb_last_error()
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


@pytest.mark.parametrize("D", [64, 256])
def test_poisoned_workspace(D):
    net, cfg, cam, smat, c2w = scene(D)
    T = T_of(cam, c2w, smat)
    pixels = pixels_of(24, 32)
    runs = {f: _direct(net, T, pixels, w) for f, w in {"zeros": 0, "nan": -1, "big": 0x7E7E7E7E}.items()}
    for k, v in runs["zeros"].items():
        for f, o in runs.items():
            assert same(v, o[k]), (D, k, f)
    assert bool(torch.isfinite(runs["zeros"]["rgb"]).all())


# ---- 7. a 1080p frame ----------------------------------------------------------------------------------------------------------------
def test_1080p_frame_rows_alone():
    _, L, _, _, _ = _mods()
    net, cfg, _, smat, c2w = scene(256)
    H, W = 1080, 1920
    cam = FC.small_scene(H, W)["img.camera_mat"].cuda()
    T = T_of(cam, c2w, smat)
    pixels = pixels_of(H, W)
    whole = _all(frame(net, T, pixels))
    rows = _all(frame(net, T, pixels[:, 531 * W:549 * W]))
    for k, v in whole.items():
        assert same(v[531 * W:549 * W], rows[k]), k
    assert L.lib.nnb_geometry_frame_workspace_bytes(H * W, N_STEPS, 256) <= 945541632   # the header's figure
    print("1080p frame: %d object rays" % int((torch.isfinite(whole["depth"]) & (whole["depth"] != 0)).sum()))


# ---- 8. routing through the callers -------------------------------------------------------------------------------------------------
def _trainer(net, cfg, V, state, **kw):
    mdl = _mods()[0]
    dev = torch.device("cuda")
    rend = mdl.Renderer(net, cfg["rendering"], device=dev, **kw)
    model = mdl.get_model(rend, cfg, device=dev)
    pose = mdl.LearnPose(V, True, True, cfg).to(dev)
    with torch.no_grad():
        pose.r.copy_(state["r"]); pose.t.copy_(state["t"])
    tr = cfg["training"]
    trainer = mdl.Trainer(model, torch.optim.Adam(model.parameters(), lr=tr["learning_rate"]), tr, device=dev,
                          optimizer_pose=torch.optim.Adam(pose.parameters(), lr=tr["pose_lr"]), pose_param_net=pose)
    return trainer, rend, pose


def _count(rend, name):
    calls = []
    real = getattr(rend, name)
    setattr(rend, name, lambda *a, **k: calls.append(a[0].shape[1]) or real(*a, **k))
    return calls


def test_callers_make_one_call_per_frame():
    mdl = _mods()[0]
    cfg = FC.default_cfg(); assert cfg["training"]["vis_geo"] is True
    net, pixels, cam, smat, c2w, gold, state = _geometry_setup(cfg)
    H, W, V = 24, 32, 4
    data = FC.small_scene(H, W, V=V); data["img.idx"] = torch.tensor([int(gold["view"])])
    trainer, rend, pose = _trainer(net, cfg, V, state, geometry_frame=True)
    with torch.no_grad():
        c2w = pose(int(gold["view"]))
        ref = rend.phong_frame(pixels, cam.reshape(1, 4, 4), torch.inverse(c2w).unsqueeze(0), smat, 0)["rgb"]
    ref8 = (ref.reshape(H, W, 3).cpu().numpy() * 255).astype(np.uint8)
    calls = _count(rend, "phong_frame")
    torch.manual_seed(3); img = trainer.render_visdata(data, (H, W), 0, None); st = torch.get_rng_state()
    torch.manual_seed(3); torch.randint(512, 513, (1,))
    assert calls == [H * W] and np.array_equal(img, ref8) and torch.equal(st, torch.get_rng_state())
    ex = mdl.Extract_Images(rend, {"extract_images": {"resolution": [H, W]}}, device=torch.device("cuda"))
    del calls[:]
    geo = ex.render_geometry(c2w, cam, smat, H, W, it=0)
    assert calls == [H * W] and np.array_equal(geo, ref8)


def test_callers_without_the_option_are_unchanged():
    """default renderer: GEOMETRY_CHUNK-pixel phong_renderer calls, one randint each, as before the option existed"""
    mdl = _mods()[0]
    from nope_nerf_b200.model.rendering import GEOMETRY_CHUNK
    cfg = FC.default_cfg()
    net, _, cam, smat, c2w, gold, state = _geometry_setup(cfg)
    H, W, V = 40, 60, 4   # 2400 pixels: three calls
    pixels = pixels_of(H, W)
    data = FC.small_scene(H, W, V=V); data["img.idx"] = torch.tensor([int(gold["view"])])
    data["img.camera_mat"] = cam.cpu()
    trainer, rend, pose = _trainer(net, cfg, V, state)
    assert rend.geometry_frame is False
    with torch.no_grad():
        c2w = pose(int(gold["view"]))
        torch.manual_seed(3)
        ref = torch.cat([rend.phong_renderer(px, cam.reshape(1, 4, 4), torch.inverse(c2w).unsqueeze(0), smat, 0)["rgb"]
                         for px in torch.split(pixels, GEOMETRY_CHUNK, dim=1)], dim=1)
    st_ref = torch.get_rng_state()
    ref8 = (ref.reshape(H, W, 3).cpu().numpy() * 255).astype(np.uint8)
    calls = _count(rend, "phong_renderer")
    torch.manual_seed(3); img = trainer.render_visdata(data, (H, W), 0, None)
    assert calls == [1024, 1024, 352] and np.array_equal(img, ref8) and torch.equal(torch.get_rng_state(), st_ref)
    ex = mdl.Extract_Images(rend, {"extract_images": {"resolution": [H, W]}}, device=torch.device("cuda"))
    del calls[:]
    torch.manual_seed(3); geo = ex.render_geometry(c2w, cam, smat, H, W, it=0)
    assert calls == [1024, 1024, 352] and np.array_equal(geo, ref8) and torch.equal(torch.get_rng_state(), st_ref)

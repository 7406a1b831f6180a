"""GPU: the fused ray march of the geometry view (nnb_ray_march: tc_march / tc_secant / march_finish in csrc/nnb_tc.cu; field.ray_march;
Renderer.ray_marching with field_engine='tc').

On the tensor-core engine a point's occupancy does not depend on the tile or row that evaluates it, and the fused kernels form depths,
points, products and secant iterates with the roundings of the torch code.  So the reference is exact: Renderer._ray_marching_torch
(the torch march over explicit-point queries) with engine='tc' for the depth, and the numpy restatement of its bracket search
(tests/_ray_march_ref.py, pinned against the torch march in tests/test_ray_march_ref.py) for `first` and `bracket`; everything is compared
with torch.equal.  The float64 oracle checks, independently of that, that a returned root is a root.
"""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
import _fullsize_cases as FC
import _ray_march_ref as R

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TAU = 0.5
N_ALL = 20000        # more than one wave of one-ray tiles (132 CTAs) and of 128-ray secant tiles
SIZES = (1, 127, 1024, N_ALL)


def _mods():
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import _lib as L, ops, field
    return mdl, L, ops, field


_nets = {}


def geo_net(D):
    """D = 256: the geometry field of test_geometry_view_on_tensor_cores (a visible surface).  64 / 128: a seeded field of that width made
    the same way (density head scaled by 10: the occupancy crosses tau = 0.5 where the logit crosses 0), with the density bias set so
    that the logit's median over the scene is 0: about half the space is occupied and rays start, cross and miss in numbers"""
    if D not in _nets:
        mdl = _mods()[0]
        cfg = FC.default_cfg()
        cfg["model"]["hidden_dim"] = D
        state = FC.start_state(cfg, 4, 31 if D == 256 else 100 + D, 95, geo=True)
        net = mdl.OfficialStaticNerf(cfg)
        net.load_state_dict({k: v.clone() for k, v in state["net"].items()})
        net = net.cuda().eval()
        for q in net.parameters():
            q.requires_grad_(False)
        if D != 256:
            p = (torch.randn(4096, 3, generator=torch.Generator().manual_seed(D)) * 0.8).cuda()
            with torch.no_grad():
                net.fc_density.bias -= _mods()[3].field_query(net, p, None, raw_density=True)[1].median()
        _nets[D] = (net, mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), field_engine="tc"), cfg, state)
    return _nets[D]


def sphere_far(o, d, r):
    """far intersection of each ray with |x| = r, 0 where it misses (per-ray origins)"""
    dot = (o * d).sum(-1)
    under = dot ** 2 - ((o * o).sum(-1) - r * r)
    return torch.where(under > 0, torch.sqrt(under.clamp_min(0)) - dot, torch.zeros_like(dot)).clamp_min(0.0)


def make_rays(D, n, seed):
    """camera rays of a small view of the scene (Renderer._rays_world) followed by hand-made rays: origins in and around the unit ball,
    seeded directions.  The last quarter of the rays is cut short (far * 1e-4): these fields vary so fast that a ray of full length
    always crosses, and a short ray that starts in free space is the one that finds nothing and runs through every round.
    Returns ray0, dirs (n, 3) and far (n,)"""
    net, rend, cfg, state = geo_net(D)
    mdl = _mods()[0]
    from nope_nerf_b200.model import common as mc
    g = torch.Generator().manual_seed(seed)
    H, W = 48, 64
    data = FC.small_scene(H, W, V=4)
    pixels = mc.arange_pixels((H, W), 1)[1].cuda()
    pose = mdl.LearnPose(4, True, True, cfg).cuda()
    with torch.no_grad():
        pose.r.copy_(state["r"]); pose.t.copy_(state["t"])
        c2w = pose(1)
        cw, rv = rend._rays_world(pixels, data["img.camera_mat"].cuda(), torch.inverse(c2w).unsqueeze(0), data["img.scale_mat"].cuda())
    cw, rv = cw[0], rv[0]
    m = n - cw.shape[0]
    assert m > 0
    o = (torch.randn(m, 3, generator=g) * 0.4).cuda()
    d = torch.randn(m, 3, generator=g).cuda()
    d = d / d.norm(2, -1, keepdim=True)
    ray0 = torch.cat([cw, o]).contiguous(); dirs = torch.cat([rv, d]).contiguous()
    far = sphere_far(ray0, dirs, float(cfg["rendering"]["radius"]))
    far[n - n // 4:] *= 1e-4
    return ray0, dirs, far.contiguous()


def old_march(D, ray0, dirs, far, n_steps, n_secant):
    """Renderer._ray_marching_torch on the tensor-core engine with the given per-ray far depths"""
    net, rend, cfg, _ = geo_net(D)
    rend._sphere_far = lambda cam_loc, d, r: far.view(1, -1)
    try:
        with torch.no_grad():
            return rend._ray_marching_torch(ray0[None], dirs[None], net, n_steps, n_secant, [0., 2.4], 3500000, 1.0, "tc")[0]
    finally:
        del rend._sphere_far


def values(D, ray0, dirs, far, n_steps):
    """val (n, n_steps) = occupancy - tau on the tensor-core engine at the torch march's points, and their depths t"""
    net = geo_net(D)[0]
    frac = torch.linspace(0, 1, steps=n_steps, device="cuda").view(1, n_steps)
    t = 0. * (1. - frac) + far.view(-1, 1) * frac
    p = ray0.unsqueeze(1) + dirs.unsqueeze(1) * t.unsqueeze(-1)
    with torch.no_grad():
        val = net(p.reshape(1, -1, 3), only_occupancy=True, engine="tc").reshape(-1, n_steps) - TAU
    return val.cpu().numpy(), t.cpu().numpy()


def fused(D, ray0, dirs, far, n_steps, n_secant):
    field = _mods()[3]
    frac = torch.linspace(0, 1, steps=n_steps, device="cuda")
    out = field.ray_march(geo_net(D)[0], ray0, dirs, far, frac, 0.0, n_secant, TAU, want_bracket=True)
    torch.cuda.synchronize()
    return out


def expected(val, t):
    """first as the library reports it (-1 also where the first sample is occupied), hit, v0neg, bracket"""
    first, hit, v0neg, br = R.first_and_bracket(val, t)
    return np.where(v0neg, first, -1).astype(np.int32), hit, v0neg, br


def check_batch(D, ray0, dirs, far, n_steps, n_secant, val=None, t=None):
    depth, first, bracket, counts = fused(D, ray0, dirs, far, n_steps, n_secant)
    ref = old_march(D, ray0, dirs, far, n_steps, n_secant)
    assert torch.equal(depth, ref), (D, ray0.shape[0], n_steps, n_secant, int((depth != ref).sum()))
    if val is None:
        val, t = values(D, ray0, dirs, far, n_steps)
    e_first, hit, v0neg, br = expected(val, t)
    assert np.array_equal(first.cpu().numpy(), e_first)
    assert np.array_equal(bracket.cpu().numpy()[hit].view(np.uint32), br[hit].view(np.uint32))
    d = depth.cpu().numpy()
    assert np.array_equal(np.isinf(d), v0neg & ~hit) and (d[~v0neg] == 0).all() and np.isfinite(d[hit]).all()
    assert int(counts[0]) == int(hit.sum())
    return depth, first, bracket, counts, (e_first, hit, v0neg, br)


@pytest.mark.parametrize("n_steps", [2, 127, 128, 129, 512, 513])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_bit_equal_to_unfused_march(D, n_steps):
    ray0, dirs, far = make_rays(D, N_ALL, seed=D + n_steps)
    val, t = values(D, ray0, dirs, far, n_steps)
    for n in SIZES:
        for n_secant in (0, 1, 8):
            *_, (e_first, hit, v0neg, _) = check_batch(D, ray0[:n], dirs[:n], far[:n], n_steps, n_secant, val[:n], t[:n])
    # the full batch has every outcome
    print("D %d, %d steps: %d hits, %d occupied at the start, %d without a hit" % (D, n_steps, hit.sum(), (~v0neg).sum(), (v0neg & ~hit).sum()))
    assert hit.sum() > 0 and (~v0neg).sum() > 0 and (n_steps == 2 or (v0neg & ~hit).sum() > 0)


def test_planted_edge_cases():
    D, n_steps = 256, 512
    ray0, dirs, far = make_rays(D, 6000, seed=3)
    depth, first, bracket, counts, (e_first, hit, v0neg, br) = check_batch(D, ray0, dirs, far, n_steps, 8)
    h = torch.from_numpy(hit).cuda()
    assert h.sum() >= 64
    o, d, ts = ray0[h][:64], dirs[h][:64], depth[h][:64]
    free = torch.from_numpy(v0neg & (e_first < 0) & (far.cpu().numpy() > 0)).cuda()     # rays that cross nothing
    inside = torch.from_numpy(~v0neg).cuda()                                            # rays whose origin is occupied
    assert free.sum() >= 8 and inside.sum() >= 64
    groups = {
        "miss_free": (ray0[free][:8], dirs[free][:8], torch.zeros(8, device="cuda")),            # far = 0: every step is the origin
        "miss_occupied": (ray0[inside][:8], dirs[inside][:8], torch.zeros(8, device="cuda")),
        "occupied_start": (ray0[inside][:64], dirs[inside][:64], torch.full((64,), 3.0, device="cuda")),
        "no_crossing": (ray0[free][:8], dirs[free][:8], far[free][:8]),
        "block_edge": (o, d, ts * (n_steps - 1) / 127.5),                       # bracket = steps (127, 128)
        "last_pair": (o, d, ts * (n_steps - 1) / (n_steps - 1.5)),              # bracket = the last two steps
        "first_pair": (o, d, ts * (n_steps - 1) / 0.5),                         # bracket = steps (0, 1)
    }
    names = list(groups)
    sizes = [groups[k][0].shape[0] for k in names]
    r0 = torch.cat([groups[k][0] for k in names]).contiguous(); dd = torch.cat([groups[k][1] for k in names]).contiguous()
    ff = torch.cat([groups[k][2] for k in names]).contiguous()
    depth, first, bracket, counts, (e_first, hit, v0neg, br) = check_batch(D, r0, dd, ff, n_steps, 8)
    val, _ = values(D, r0, dd, ff, n_steps)
    sl = dict(zip(names, np.split(np.arange(r0.shape[0]), np.cumsum(sizes)[:-1])))
    dn, fn = depth.cpu().numpy(), first.cpu().numpy()
    assert np.isinf(dn[sl["miss_free"]]).all() and (fn[sl["miss_free"]] == -1).all()
    assert (dn[sl["miss_occupied"]] == 0).all()
    i = sl["occupied_start"]
    later = (val[i, 0] >= 0) & ((val[i, :-1] * val[i, 1:]) < 0).any(1)
    assert later.sum() >= 1 and (dn[i][later] == 0).all()
    assert np.isinf(dn[sl["no_crossing"]]).all() and int(counts[-2]) >= len(sl["no_crossing"])   # they run through every round
    # (a finer step grid can find a crossing the 512-step march stepped over, so not every planted ray keeps its bracket)
    n_edge, n_last, n_first = [int((fn[sl[k]] == i).sum()) for k, i in (("block_edge", 127), ("last_pair", n_steps - 2), ("first_pair", 0))]
    print("planted brackets kept: block edge %d, last pair %d, first pair %d of 64" % (n_edge, n_last, n_first))
    assert n_edge >= 1 and hit[sl["block_edge"]][fn[sl["block_edge"]] == 127].all()
    assert n_last >= 1 and n_first >= 1


def test_root_is_a_root():
    """float64 oracle field at the returned depth and at the ends of the returned bracket"""
    D, n_steps = 256, 512
    net = geo_net(D)[0]
    ray0, dirs, far = make_rays(D, 6000, seed=9)
    depth, first, bracket, _ = fused(D, ray0, dirs, far, n_steps, 8)
    h = torch.isfinite(depth) & (depth > 0)
    assert h.sum() > 200
    o, d = ray0[h].cpu().numpy().astype(np.float64), dirs[h].cpu().numpy().astype(np.float64)
    dep, br = depth[h].cpu().numpy().astype(np.float64), bracket[h].cpu().numpy().astype(np.float64)
    P = {k: np.asarray(v, np.float64) for k, v in O.unflatten_params(net.flat_weights().cpu().numpy(), D).items()}
    occ = lambda tt: O.mlp_forward(P, o + tt[:, None] * d, np.ones_like(o), dist_alpha=net.dist_alpha, occ_activation=net.occ_activation)[1]
    f_low, f_high, f_root = occ(br[:, 0]) - TAU, occ(br[:, 1]) - TAU, occ(dep) - TAU
    assert np.abs(f_low - br[:, 2]).max() < 1e-5 and np.abs(f_high - br[:, 3]).max() < 1e-5      # the engine's values are the field's
    assert ((br[:, 0] <= dep) & (dep <= br[:, 1])).all()
    near_tau = (np.abs(f_low) < 1e-5) | (np.abs(f_high) < 1e-5)      # the engine's error could flip these signs
    assert near_tau.mean() < 0.05, near_tau.mean()
    assert (f_low[~near_tau] < 0).all() and (f_high[~near_tau] >= 0).all()
    assert (np.abs(f_root) <= np.maximum(np.abs(br[:, 2]), np.abs(br[:, 3])) + 1e-5).all()
    print("root: %d hits, median |occ(depth) - tau| %.2e, median bracket %.2e" % (h.sum(), np.median(np.abs(f_root)), np.median(np.abs(br[:, 2:]).max(1))))
    assert np.median(np.abs(f_root)) < 0.1 * np.median(np.abs(br[:, 2:]).max(1))     # eight secant steps do refine


@pytest.mark.parametrize("D", [64, 256])
def test_early_exit_counts(D):
    """round k (k >= 1) takes exactly the rays that block 0 .. k - 1 left undecided"""
    n_steps = 513
    ray0, dirs, far = make_rays(D, N_ALL, seed=21)
    val, t = values(D, ray0, dirs, far, n_steps)
    _, _, _, counts, (e_first, hit, v0neg, _) = check_batch(D, ray0, dirs, far, n_steps, 1, val, t)
    rounds = (n_steps + 127) // 128
    assert counts.numel() == rounds + 1
    want = [int((v0neg & ((e_first < 0) | (e_first + 1 >= 128 * k))).sum()) for k in range(1, rounds)]
    assert counts[1:rounds].tolist() == want, (counts.tolist(), want)
    assert want[0] < N_ALL and all(a >= b for a, b in zip(want, want[1:]))
    assert int(counts[rounds]) == 0      # the last round appends nothing


def _phong(rend, H=24, W=32, V=4):
    mdl = _mods()[0]
    from nope_nerf_b200.model import common as mc
    _, _, cfg, state = geo_net(256)
    gold = dict(np.load(os.path.join(GOLDEN, "fullsize_phong.npz")))
    data = FC.small_scene(H, W, V=V)
    pixels = mc.arange_pixels((H, W), 1)[1].cuda()
    pose = mdl.LearnPose(V, True, True, cfg).cuda()
    with torch.no_grad():
        pose.r.copy_(state["r"]); pose.t.copy_(state["t"])
        c2w = pose(int(gold["view"]))
    o = rend(pixels, None, data["img.camera_mat"].cuda(), torch.inverse(c2w).unsqueeze(0), data["img.scale_mat"].cuda(), "phong_renderer", it=0)
    return o["rgb"].detach().reshape(-1, 3), o["rgb_surf"].detach().reshape(-1, 3), gold


def _old_path_renderer(net, cfg, field_engine):
    """a Renderer whose ray_marching is the torch march on field_engine"""
    mdl = _mods()[0]

    class OldPath(mdl.Renderer):
        def ray_marching(self, ray0, ray_direction, model, c=None, tau=0.5, n_steps=[128, 129], n_secant_steps=8, depth_range=[0., 2.4],
                         max_points=3500000, rad=1.0):
            n = int(torch.randint(n_steps[0], n_steps[1], (1,)).item())
            return self._ray_marching_torch(ray0, ray_direction, model, n, n_secant_steps, depth_range, max_points, rad, self.field_engine)

    return OldPath(net, cfg["rendering"], device=torch.device("cuda"), field_engine=field_engine)


# sha256 of the float32 bytes of (rgb, rgb_surf) of the 24 x 32 golden view with field_engine=None, recorded from the build before the
# fused march existed (NVIDIA H100 80GB HBM3)
EXACT_PHONG_SHA256 = "7ed911f762dfedfbb5f28dbe7ca7a8d33ba201b0b931cdec41aa980f7992cfe0"


def test_renderer_level():
    mdl = _mods()[0]
    net, _, cfg, _ = geo_net(256)
    new = mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda"), field_engine="tc")
    torch.manual_seed(1); rgb, surf, gold = _phong(new); s_new = torch.get_rng_state()
    torch.manual_seed(1); rgb_o, surf_o, _ = _phong(_old_path_renderer(net, cfg, "tc")); s_old = torch.get_rng_state()
    assert torch.equal(rgb, rgb_o) and torch.equal(surf, surf_o)
    assert torch.equal(s_new, s_old)        # one randint per march, as before
    rgb_ref, surf_ref = torch.as_tensor(gold["rgb"]).cuda(), torch.as_tensor(gold["rgb_surf"]).cuda()
    bad = ((rgb_ref - rgb).abs().max(1).values > 2.0 / 255) | ((surf_ref - surf).abs().max(1).values > 2.0 / 255)
    assert float(bad.float().mean()) <= 0.01
    assert float((surf.abs().sum(1) > 0).float().mean()) > 0.02
    # the exact engine's path is the code it was
    rgb_e, surf_e, _ = _phong(mdl.Renderer(net, cfg["rendering"], device=torch.device("cuda")))
    rgb_eo, surf_eo, _ = _phong(_old_path_renderer(net, cfg, None))
    assert torch.equal(rgb_e, rgb_eo) and torch.equal(surf_e, surf_eo)
    digest = hashlib.sha256(rgb_e.cpu().numpy().tobytes() + surf_e.cpu().numpy().tobytes()).hexdigest()
    print("field_engine=None phong sha256", digest)
    assert digest == EXACT_PHONG_SHA256


def _raw_call(L, ops, net, N=8, n_steps=16, n_secant=2, engine=None, hidden_dim=None, far=True, ws_bytes=None):
    flat = net.flat_weights()
    t = dict(ray0=torch.zeros(max(N, 1), 3, device="cuda"), dirs=torch.ones(max(N, 1), 3, device="cuda"), far=torch.ones(max(N, 1), device="cuda"),
             frac=torch.linspace(0, 1, max(n_steps, 2), device="cuda"), depth=torch.full((max(N, 1),), -7.0, device="cuda"))
    hd = net.hidden_dim if hidden_dim is None else hidden_dim
    need = L.lib.nnb_ray_march_workspace_bytes(max(N, 1), max(n_steps, 2), net.hidden_dim)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    a = L.RayMarchArgs()
    a.weights = L.ptr(flat); a.ray0 = L.ptr(t["ray0"]); a.ray_dir = L.ptr(t["dirs"]); a.far_ = L.ptr(t["far"]) if far else None
    a.frac = L.ptr(t["frac"]); a.N = N; a.n_steps = n_steps; a.n_secant = n_secant; a.hidden_dim = hd
    a.near_ = 0.0; a.tau = TAU; a.flags = L.SOFTPLUS; a.engine = L.ENGINE_TC if engine is None else engine
    a.depth = L.ptr(t["depth"]); a.workspace = L.ptr(ws); a.workspace_bytes = need if ws_bytes is None else ws_bytes
    rc = L.lib.nnb_ray_march(C.byref(a), ops._stream())
    torch.cuda.synchronize()
    return rc, t["depth"], need


def test_argument_checks():
    _, L, ops, _ = _mods()
    net = geo_net(64)[0]
    assert L.lib.nnb_version() >= 104
    rc, depth, need = _raw_call(L, ops, net)
    assert rc == 0 and need > 0 and not (depth == -7.0).any()
    for kw in (dict(engine=L.ENGINE_SIMT), dict(hidden_dim=96), dict(n_steps=1), dict(n_secant=-1), dict(ws_bytes=need - 1), dict(far=False), dict(N=-1)):
        rc, depth, _ = _raw_call(L, ops, net, **kw)
        assert rc < 0 and L.lib.nnb_last_error().decode() != "", kw
        assert (depth == -7.0).all(), kw
    rc, depth, _ = _raw_call(L, ops, net, N=0)
    assert rc == 0 and (depth == -7.0).all()
    assert L.lib.nnb_ray_march_workspace_bytes(0, 16, 64) == 0 and L.lib.nnb_ray_march_workspace_bytes(8, 1, 64) == 0
    assert L.lib.nnb_ray_march_workspace_bytes(8, 16, 96) == 0

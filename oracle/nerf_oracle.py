"""CPU oracle for the NoPe-NeRF render + pose-optimisation hot path.

TEST INFRASTRUCTURE ONLY.  This module is a numpy restatement of the reference's
algorithm (ActiveVisionLab/nope-nerf @ 47c861f6).  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` leg may import it; the product path (``nope_nerf_b200``) never does
and fails loudly when its CUDA library is missing.

Parity status: PINNED.  The reference ships no tests or golden vectors
(SURVEY.md section 4), so the oracle is pinned against outputs of the reference
itself: ``tools/make_golden.py`` imports the unmodified reference from
a reference checkout, runs it (torch CPU, fp32, autograd)
on seeded inputs and commits inputs/outputs/gradients under ``tests/golden/``;
``tests/test_oracle_golden.py`` checks this restatement against those fixtures.

Every function cites the reference file:line it follows.  All functions take a
``dtype`` (np.float32 reproduces the reference arithmetic, np.float64 gives a
"truth" used to budget rounding error).  Forward functions return caches and the
matching ``*_bwd`` functions are hand-derived adjoints (the reference relies on
torch autograd; SURVEY.md appendix A.5/A.6 states the closed forms).
"""
import math
import numpy as np

EPSILON = 1e-6  # model/rendering.py:9

# Order of the 24 parameter tensors == OfficialStaticNerf.parameters() order
# (model/official_nerf.py:20-37); this is also the layout of the flat fp32
# weight / gradient buffer of the CUDA library (include/nope_nerf_b200.h).
PARAM_NAMES = []
for _blk in ("layers0", "layers1"):
    for _i in (0, 2, 4, 6):
        PARAM_NAMES += ["%s.%d.weight" % (_blk, _i), "%s.%d.bias" % (_blk, _i)]
PARAM_NAMES += ["fc_density.weight", "fc_density.bias", "fc_feature.weight", "fc_feature.bias",
                "rgb_layers.0.weight", "rgb_layers.0.bias", "fc_rgb.weight", "fc_rgb.bias"]


def param_shapes(D=256, pos_levels=10, dir_levels=4):
    """Shapes in PARAM_NAMES order (model/official_nerf.py:9-37)."""
    pin, din = (2 * pos_levels + 1) * 3, (2 * dir_levels + 1) * 3
    sh = {}
    ins0 = [pin, D, D, D]
    ins1 = [D + pin, D, D, D]
    for j, i in enumerate((0, 2, 4, 6)):
        sh["layers0.%d.weight" % i] = (D, ins0[j]); sh["layers0.%d.bias" % i] = (D,)
        sh["layers1.%d.weight" % i] = (D, ins1[j]); sh["layers1.%d.bias" % i] = (D,)
    sh["fc_density.weight"] = (1, D); sh["fc_density.bias"] = (1,)
    sh["fc_feature.weight"] = (D, D); sh["fc_feature.bias"] = (D,)
    sh["rgb_layers.0.weight"] = (D // 2, D + din); sh["rgb_layers.0.bias"] = (D // 2,)
    sh["fc_rgb.weight"] = (3, D // 2); sh["fc_rgb.bias"] = (3,)
    return [(n, sh[n]) for n in PARAM_NAMES]


def init_params(seed=42, D=256, white_bkgd=False, dtype=np.float32, hf_damp=False):
    """nn.Linear default init U(-1/sqrt(in), 1/sqrt(in)) + the bias overrides of
    model/official_nerf.py:39-44.  (Distribution-equivalent to torch's init, not
    stream-identical; parity tests pass explicit weights.)

    hf_damp: test aid for WELL-CONDITIONED parity cases.  The columns of the two layers that read the positional encoding are
    scaled by 2^-l for frequency level l, so the ~1e-4 noise that sin/cos(2^9 p) of fp32-rounded points puts on the first
    pre-activations drops to the GEMM rounding level and hidden-unit ReLU gates no longer switch between evaluation orders
    (tests/test_oracle_golden.py::test_render_gate_matched_and_kxy): every fp32 implementation then agrees on the GRADIENTS to
    ~1e-5, and the 1e-4 parity gate can be applied to them without an envelope term."""
    rng = np.random.default_rng(seed)
    P = {}
    for n, s in param_shapes(D):
        fan_in = s[1] if len(s) == 2 else dict(param_shapes(D))[n.replace("bias", "weight")][1]
        b = 1.0 / math.sqrt(fan_in)
        P[n] = rng.uniform(-b, b, size=s).astype(dtype)
    P["fc_density.bias"][:] = 0.1
    P["fc_rgb.bias"][:] = 0.8 if white_bkgd else 0.02
    if hf_damp:
        damp = np.ones(63, dtype)
        for l in range(10):
            damp[3 + 6 * l:9 + 6 * l] = 2.0 ** (-l)
        P["layers0.0.weight"] *= damp[None, :]
        P["layers1.0.weight"][:, D:] *= damp[None, :]
    return P


def flatten_params(P, dtype=np.float32):
    return np.concatenate([np.asarray(P[n], dtype=dtype).reshape(-1) for n in PARAM_NAMES])


def unflatten_params(flat, D=256):
    P, o = {}, 0
    for n, s in param_shapes(D):
        k = int(np.prod(s)); P[n] = flat[o:o + k].reshape(s); o += k
    assert o == flat.size
    return P


# ----------------------------------------------------------------------------
# Field: positional encoding + 8x256 MLP (model/official_nerf.py:60-119)
# ----------------------------------------------------------------------------
def encode_position(x, levels):
    """model/official_nerf.py:99-119, inc_input=True: [x, sin(2^0 x), cos(2^0 x), ...]."""
    out = [x]
    for i in range(levels):
        t = x.dtype.type(2.0 ** i) * x
        out.append(np.sin(t)); out.append(np.cos(t))
    return np.concatenate(out, axis=-1)


def encode_position_bwd(x, levels, g):
    """Adjoint of encode_position (SURVEY.md A.6)."""
    gx = g[..., 0:3].copy()
    for i in range(levels):
        f = x.dtype.type(2.0 ** i)
        t = f * x
        gs = g[..., 3 + 6 * i: 6 + 6 * i]; gc = g[..., 6 + 6 * i: 9 + 6 * i]
        gx += f * (np.cos(t) * gs - np.sin(t) * gc)
    return gx


def _softplus(s):
    # F.softplus beta=1, threshold=20 (model/official_nerf.py:77-78)
    return np.where(s > 20, s, np.log1p(np.exp(np.minimum(s, 20))))


def _sigmoid(s):
    return 1.0 / (1.0 + np.exp(-s))


def mlp_forward(P, pts, dirs, dist_alpha=False, occ_activation="softplus"):
    """OfficialStaticNerf.forward(p, ray_d, return_addocc=True)
    (model/official_nerf.py:60-96).  Returns rgb (M,3), a (M,) [alpha if not
    dist_alpha else sigma] and a cache for mlp_backward."""
    e = encode_position(pts, 10)                                   # :61
    h = e
    X, Y = [], []                                                  # layer inputs / pre-activations
    for i in (0, 2, 4, 6):                                         # :62 layers0
        X.append(h); y = h @ P["layers0.%d.weight" % i].T + P["layers0.%d.bias" % i]
        Y.append(y); h = np.maximum(y, 0)
    h = np.concatenate([h, e], axis=-1)                            # :63
    for i in (0, 2, 4, 6):                                         # :64 layers1
        X.append(h); y = h @ P["layers1.%d.weight" % i].T + P["layers1.%d.bias" % i]
        Y.append(y); h = np.maximum(y, 0)
    s = (h @ P["fc_density.weight"].T + P["fc_density.bias"])[:, 0]  # :66
    sigma = _softplus(s) if occ_activation == "softplus" else np.maximum(s, 0)   # :77-80
    a = sigma if dist_alpha else 1 - np.exp(-sigma)                # :82-83
    de = encode_position(dirs, 4)                                  # :87
    feat = h @ P["fc_feature.weight"].T + P["fc_feature.bias"]     # :88
    xr = np.concatenate([feat, de], axis=-1)                       # :89
    yr = xr @ P["rgb_layers.0.weight"].T + P["rgb_layers.0.bias"]  # :90
    hr = np.maximum(yr, 0)
    yc = hr @ P["fc_rgb.weight"].T + P["fc_rgb.bias"]              # :91
    rgb = _sigmoid(yc)                                             # :92
    cache = dict(pts=pts, dirs=dirs, X=X, Y=Y, h8=h, s=s, sigma=sigma, xr=xr, yr=yr, hr=hr, rgb=rgb,
                 dist_alpha=dist_alpha, occ=occ_activation)
    return rgb, a, cache


def mlp_backward(P, cache, g_rgb, g_a):
    """Adjoint of mlp_forward: returns (grads dict, g_pts (M,3), g_dirs (M,3))."""
    G = {}
    s, sigma = cache["s"], cache["sigma"]
    rgb = cache["rgb"]
    # colour head
    g_yc = g_rgb * rgb * (1 - rgb)
    G["fc_rgb.weight"] = g_yc.T @ cache["hr"]; G["fc_rgb.bias"] = g_yc.sum(0)
    g_hr = g_yc @ P["fc_rgb.weight"]
    g_yr = g_hr * (cache["yr"] > 0)
    G["rgb_layers.0.weight"] = g_yr.T @ cache["xr"]; G["rgb_layers.0.bias"] = g_yr.sum(0)
    g_xr = g_yr @ P["rgb_layers.0.weight"]
    D = P["fc_feature.weight"].shape[0]
    g_feat, g_de = g_xr[:, :D], g_xr[:, D:]
    g_dirs = encode_position_bwd(cache["dirs"], 4, g_de)
    G["fc_feature.weight"] = g_feat.T @ cache["h8"]; G["fc_feature.bias"] = g_feat.sum(0)
    g_h = g_feat @ P["fc_feature.weight"]
    # density head
    ds = _sigmoid(s) if cache["occ"] == "softplus" else (s > 0).astype(s.dtype)
    if cache["occ"] == "softplus":
        ds = np.where(s > 20, np.ones_like(s), ds)
    g_sigma = g_a if cache["dist_alpha"] else g_a * np.exp(-sigma)
    g_s = (g_sigma * ds)[:, None]
    G["fc_density.weight"] = g_s.T @ cache["h8"]; G["fc_density.bias"] = g_s.sum(0)
    g_h = g_h + g_s @ P["fc_density.weight"]
    # trunk
    X, Y = cache["X"], cache["Y"]
    g_e = None
    for li, (blk, i) in reversed(list(enumerate([("layers0", 0), ("layers0", 2), ("layers0", 4), ("layers0", 6),
                                                 ("layers1", 0), ("layers1", 2), ("layers1", 4), ("layers1", 6)]))):
        g_y = g_h * (Y[li] > 0)
        W = P["%s.%d.weight" % (blk, i)]
        G["%s.%d.weight" % (blk, i)] = g_y.T @ X[li]; G["%s.%d.bias" % (blk, i)] = g_y.sum(0)
        g_x = g_y @ W
        if li == 4:                     # skip concat [h, enc]
            g_h, g_e = g_x[:, :D], g_x[:, D:]
        else:
            g_h = g_x
    g_e = g_e + g_h                     # layer 0 input is enc itself
    g_pts = encode_position_bwd(cache["pts"], 10, g_e)
    return G, g_pts, g_dirs


# ----------------------------------------------------------------------------
# Poses (model/poses.py:23-31, model/common.py:277-330)
# ----------------------------------------------------------------------------
def vec2skew(v):
    """model/common.py:277-287"""
    z = v.dtype.type(0)
    return np.array([[z, -v[2], v[1]], [v[2], z, -v[0]], [-v[1], v[0], z]], dtype=v.dtype)


def exp_so3(r):
    """model/common.py:290-299 (Rodrigues with norm_r = |r| + 1e-15)."""
    K = vec2skew(r)
    n = np.sqrt((r * r).sum()).astype(r.dtype) + r.dtype.type(1e-15)
    return np.eye(3, dtype=r.dtype) + (np.sin(n) / n) * K + ((1 - np.cos(n)) / n ** 2) * (K @ K)


def exp_so3_bwd(r, gR):
    """Adjoint of exp_so3 following what autograd does (norm sub-gradient 0 at r=0)."""
    dt = r.dtype
    K = vec2skew(r)
    n0 = np.sqrt((r * r).sum()).astype(dt)
    n = n0 + dt.type(1e-15)
    A = np.sin(n) / n; B = (1 - np.cos(n)) / n ** 2
    K2 = K @ K
    gA = (gR * K).sum(); gB = (gR * K2).sum()
    gK = A * gR + B * (gR @ K.T + K.T @ gR)
    gr = np.array([gK[2, 1] - gK[1, 2], gK[0, 2] - gK[2, 0], gK[1, 0] - gK[0, 1]], dtype=dt)
    if n0 > 0:                          # autograd: d|r|/dr = r/|r|, sub-gradient 0 at r = 0
        dA = (np.cos(n) * n - np.sin(n)) / n ** 2
        dB = (np.sin(n) * n ** 2 - (1 - np.cos(n)) * 2 * n) / n ** 4
        gn = gA * dA + gB * dB
        gr = gr + gn * r / n0
    return gr


def make_c2w(r, t, init_c2w=None):
    """LearnPose.forward (model/poses.py:23-31) + make_c2w/convert3x4_4x4 (common.py:301-330)."""
    c = np.eye(4, dtype=r.dtype)
    c[:3, :3] = exp_so3(r); c[:3, 3] = t
    if init_c2w is not None:
        c = c @ init_c2w.astype(r.dtype)
    return c


def make_c2w_bwd(r, t, init_c2w, g_c2w):
    """g_c2w (4,4) -> (g_r, g_t)."""
    g = g_c2w if init_c2w is None else g_c2w @ init_c2w.astype(r.dtype).T
    return exp_so3_bwd(r, g[:3, :3]), g[:3, 3].copy()


# ----------------------------------------------------------------------------
# Pixels / prior depth (model/common.py:13-39, model/network.py:19-33)
# ----------------------------------------------------------------------------
def pixels_from_idx(ray_idx, H, W, dtype=np.float32):
    """arange_pixels (model/common.py:13-39) evaluated at ray_idx (row-major)."""
    row = (ray_idx // W).astype(dtype); col = (ray_idx % W).astype(dtype)
    two, one = dtype(2.0), dtype(1.0)
    x = two * col / dtype(W - 1) - one
    y = two * row / dtype(H - 1) - one
    return np.stack([x, y], -1)


def gather_prior_depth(dpt, ray_idx, H, W):
    """nope_nerf.forward: F.interpolate(depth,(H,W),'nearest')[ray_idx]
    (model/network.py:22-24).  Legacy 'nearest': src = floor(dst * in/out) with the
    scale computed in float32 (ATen nearest_idx)."""
    h_d, w_d = dpt.shape[-2:]
    row = ray_idx // W; col = ray_idx % W
    sr = np.minimum(np.floor(row.astype(np.float32) * np.float32(h_d / H)).astype(np.int64), h_d - 1)
    sc = np.minimum(np.floor(col.astype(np.float32) * np.float32(w_d / W)).astype(np.int64), w_d - 1)
    return dpt.reshape(h_d, w_d)[sr, sc], sr * w_d + sc


# ----------------------------------------------------------------------------
# Renderer.nope_nerf (model/rendering.py:36-167)
# ----------------------------------------------------------------------------
DEFAULT_CFG = dict(num_points=128, depth_range=(0.01, 10.0), dist_alpha=False, sample_option="uniform",
                   use_ray_dir=True, normalise_ray=True, white_background=False,
                   occ_activation="softplus")


def linspace01(S, dtype):
    """torch.linspace(0,1,S) in the working dtype (symmetric evaluation, ATen RangeFactories)."""
    step = dtype(1.0) / dtype(S - 1)
    i = np.arange(S)
    lo = (dtype(0.0) + step * i.astype(dtype)).astype(dtype)
    hi = (dtype(1.0) - step * (S - 1 - i).astype(dtype)).astype(dtype)
    return np.where(i < S // 2, lo, hi).astype(dtype)


def render_forward(P, pixels, depth, c2w, kx, ky, cfg, noise=None, eval_=False):
    """Renderer.nope_nerf (model/rendering.py:36-167) for one camera.

    pixels (N,2) in [-1,1]; depth (N,) prior depth already distorted; c2w (4,4)
    (the reference receives world_mat = inverse(c2w) and inverts it again,
    model/training.py:238, model/common.py:139-141); camera_mat = diag(kx,ky,-1,1)
    (dataloading/dataset.py:101-104), scale_mat = I.  ``noise`` (N,S) in [0,1) is
    the torch.rand draw of sample_uniform (:189) or None for add_noise=False.
    """
    dt = pixels.dtype.type
    N = pixels.shape[0]
    S = cfg["num_points"]
    R = c2w[:3, :3].astype(dt); t = c2w[:3, 3].astype(dt)
    normalise = cfg["normalise_ray"]; ndc = cfg["sample_option"] == "ndc"
    dc = np.stack([pixels[:, 0] / dt(kx), pixels[:, 1] / dt(ky), -np.ones(N, dtype=dt)], -1)   # common.py:139-152
    dtil = dc @ R.T                                                     # ray_vector :66
    nrm = np.sqrt((dtil * dtil).sum(-1))                                # :67
    d = dtil / nrm[:, None] if normalise else dtil                      # :68-69
    gdepth = np.abs(depth)
    g = gdepth * nrm if normalise else gdepth                           # d_i_gt :57-60, :70-71
    mask = np.isfinite(g) & (g != 0)                                    # :73-87
    o = np.broadcast_to(t, (N, 3))
    u = linspace01(S, dt)                                               # :95
    if ndc:                                                             # sample_ndc :168-180, common.py:632-675
        tau = -(dt(1.0) + o[:, 2]) / d[:, 2]
        o2 = o + tau[:, None] * d
        ox, oy = o2[:, 0] / o2[:, 2], o2[:, 1] / o2[:, 2]
        O = np.stack([-dt(kx) * ox, -dt(ky) * oy, dt(1.0) + dt(2.0) / o2[:, 2]], -1)
        Dn = np.stack([-dt(kx) * (d[:, 0] / d[:, 2] - ox), -dt(ky) * (d[:, 1] / d[:, 2] - oy), dt(1.0) - O[:, 2]], -1)
        z = np.broadcast_to(u, (N, S)).copy()                           # depth_range literal [0,1]; no jitter
        pts = O[:, None, :] + Dn[:, None, :] * z[:, :, None]
        geo = dict(o2=o2, tau=tau, O=O, Dn=Dn)
    else:                                                               # sample_uniform :182-197
        near, far = dt(cfg["depth_range"][0]), dt(cfg["depth_range"][1])
        z1 = near * (dt(1.0) - u) + far * u
        z = np.broadcast_to(z1, (N, S)).copy()
        if noise is not None:
            mid = dt(0.5) * (z[:, 1:] + z[:, :-1])
            hi = np.concatenate([mid, z[:, -1:]], -1); lo = np.concatenate([z[:, :1], mid], -1)
            z = lo + (hi - lo) * noise.astype(dt)
        pts = o[:, None, :] + d[:, None, :] * z[:, :, None]
        geo = {}
    vd = -d if cfg["use_ray_dir"] else np.ones_like(d)                  # :103-104,:194-195
    dirs = np.broadcast_to(vd[:, None, :], (N, S, 3)).reshape(-1, 3)
    rgb_s, a_s, mcache = mlp_forward(P, pts.reshape(-1, 3).astype(dt), dirs.astype(dt),
                                     dist_alpha=cfg["dist_alpha"], occ_activation=cfg["occ_activation"])
    rgb_s = rgb_s.reshape(N, S, 3); a_s = a_s.reshape(N, S)
    if cfg["dist_alpha"]:                                               # :122-128
        delta = np.concatenate([z[:, 1:] - z[:, :-1], np.full((N, 1), 1e10, dtype=dt)], -1)
        alpha = 1 - np.exp(-a_s * delta)
        alpha[:, -1] = 1
    else:
        delta = None
        alpha = a_s
    om = dt(1.0) - alpha + dt(EPSILON)
    T = np.cumprod(np.concatenate([np.ones((N, 1), dtype=dt), om], -1), -1)[:, :-1]   # :130
    w = alpha * T
    C = (w[:, :, None] * rgb_s).sum(1)                                  # :131
    Dist = (w * z).sum(1)                                               # :132
    if cfg["white_background"]:                                         # :145-147
        C = C + (dt(1.0) - w.sum(1))[:, None]
    Dist_out, g_out = Dist, g
    if eval_ and normalise:                                             # :150-154
        Dist_out = Dist / nrm; g_out = g / nrm
    if ndc:                                                             # :157-158
        with np.errstate(divide="ignore"):
            g_out = dt(1.0) - dt(1.0) / g_out
    cache = dict(N=N, S=S, R=R, dc=dc, dtil=dtil, nrm=nrm, d=d, depth=depth, gdepth=gdepth, g=g, z=z, alpha=alpha,
                 delta=delta, a_s=a_s, T=T, w=w, rgb_s=rgb_s, om=om, Dist=Dist, mcache=mcache, geo=geo,
                 cfg=cfg, eval_=eval_, kx=kx, ky=ky, o=o, pixels=pixels)
    out = dict(rgb=C, depth_pred_full=Dist_out, depth_gt_full=g_out, mask=mask, z_vals=z, alpha=alpha,
               depth_pred=Dist_out[mask], depth_gt=g_out[mask])
    return out, cache


def render_backward(P, cache, g_rgb, g_depth_pred_full, g_depth_gt_full):
    """Adjoint of render_forward.  g_* are dense (N,...) cotangents (zero for masked-out
    rays).  Returns dict: params (dict), c2w (4,4), depth (N,), kxy (2,)."""
    cfg = cache["cfg"]; N, S = cache["N"], cache["S"]
    dt = cache["z"].dtype.type
    normalise = cfg["normalise_ray"]; ndc = cfg["sample_option"] == "ndc"
    nrm, d, dtil, dc, R = cache["nrm"], cache["d"], cache["dtil"], cache["dc"], cache["R"]
    z, w, T, alpha, om, rgb_s = cache["z"], cache["w"], cache["T"], cache["alpha"], cache["om"], cache["rgb_s"]
    g_nrm = np.zeros(N, dtype=z.dtype)
    g_Dist = g_depth_pred_full.astype(z.dtype)
    g_g = g_depth_gt_full.astype(z.dtype)
    gcur = cache["g"]
    if cache["eval_"] and normalise:
        gcur = cache["g"] / nrm
    if ndc:
        g_g = g_g / (gcur * gcur)
    if cache["eval_"] and normalise:
        g_nrm = g_nrm - g_Dist * cache["Dist"] / (nrm * nrm)
        g_Dist = g_Dist / nrm
        g_nrm = g_nrm - g_g * cache["g"] / (nrm * nrm)
        g_g = g_g / nrm
    if normalise:
        g_gdepth = g_g * nrm; g_nrm = g_nrm + g_g * cache["gdepth"]
    else:
        g_gdepth = g_g
    g_depth = g_gdepth * np.sign(cache["depth"])
    # compositing (SURVEY.md A.5)
    g_w = (g_rgb[:, None, :] * rgb_s).sum(-1) + g_Dist[:, None] * z
    if cfg["white_background"]:
        g_w = g_w - g_rgb.sum(-1)[:, None]
    g_c = w[:, :, None] * g_rgb[:, None, :]
    wg = w * g_w
    suffix = np.cumsum(wg[:, ::-1], axis=1)[:, ::-1] - wg               # sum_{k>i} w_k gw_k
    g_alpha = T * g_w - suffix / om
    if cfg["dist_alpha"]:
        g_a = g_alpha * cache["delta"] * np.exp(-cache["a_s"] * cache["delta"])
        g_a[:, -1] = 0
    else:
        g_a = g_alpha
    G, g_pts, g_dirs = mlp_backward(P, cache["mcache"], g_c.reshape(-1, 3), g_a.reshape(-1))
    g_pts = g_pts.reshape(N, S, 3); g_dirs = g_dirs.reshape(N, S, 3)
    g_kx = dt(0); g_ky = dt(0)
    if ndc:
        geo = cache["geo"]; o = cache["o"]; kx, ky = dt(cache["kx"]), dt(cache["ky"])
        g_O = g_pts.sum(1); g_Dn = (g_pts * z[:, :, None]).sum(1)
        o2, tau, O = geo["o2"], geo["tau"], geo["O"]
        ox, oy = o2[:, 0] / o2[:, 2], o2[:, 1] / o2[:, 2]
        # Dn = (-kx (dx/dz - ox), -ky (dy/dz - oy), 1 - Oz)
        g_Oz = g_O[:, 2] - g_Dn[:, 2]
        g_ox = -kx * g_O[:, 0] + kx * g_Dn[:, 0]
        g_oy = -ky * g_O[:, 1] + ky * g_Dn[:, 1]
        g_d = np.zeros_like(d)
        g_d[:, 0] = -kx * g_Dn[:, 0] / d[:, 2]
        g_d[:, 1] = -ky * g_Dn[:, 1] / d[:, 2]
        g_d[:, 2] = (kx * g_Dn[:, 0] * d[:, 0] + ky * g_Dn[:, 1] * d[:, 1]) / (d[:, 2] ** 2)
        g_kx = (-(ox) * g_O[:, 0] - (d[:, 0] / d[:, 2] - ox) * g_Dn[:, 0]).sum()
        g_ky = (-(oy) * g_O[:, 1] - (d[:, 1] / d[:, 2] - oy) * g_Dn[:, 1]).sum()
        g_o2 = np.zeros_like(o2)
        g_o2[:, 0] = g_ox / o2[:, 2]; g_o2[:, 1] = g_oy / o2[:, 2]
        g_o2[:, 2] = -(g_ox * ox + g_oy * oy) / o2[:, 2] - dt(2.0) * g_Oz / (o2[:, 2] ** 2)
        g_o = g_o2.copy()
        g_tau = (g_o2 * d).sum(-1)
        g_d = g_d + g_o2 * tau[:, None]
        # tau = -(1 + oz)/dz
        g_o[:, 2] += -g_tau / d[:, 2]
        g_d[:, 2] += g_tau * (dt(1.0) + o[:, 2]) / (d[:, 2] ** 2)
    else:
        g_o = g_pts.sum(1)
        g_d = (g_pts * z[:, :, None]).sum(1)
    if cfg["use_ray_dir"]:
        g_d = g_d - g_dirs.sum(1)
    if normalise:
        g_dtil = (g_d - d * (d * g_d).sum(-1, keepdims=True)) / nrm[:, None]
    else:
        g_dtil = g_d
    g_dtil = g_dtil + (g_nrm / nrm)[:, None] * dtil
    g_c2w = np.zeros((4, 4), dtype=z.dtype)
    g_c2w[:3, :3] = g_dtil.T @ dc
    g_c2w[:3, 3] = g_o.sum(0)
    g_dc = g_dtil @ R
    pix = cache["pixels"]
    g_kx = g_kx + (g_dc[:, 0] * (-pix[:, 0] / dt(cache["kx"]) ** 2)).sum()
    g_ky = g_ky + (g_dc[:, 1] * (-pix[:, 1] / dt(cache["ky"]) ** 2)).sum()
    return dict(params=G, c2w=g_c2w, depth=g_depth, kxy=np.array([g_kx, g_ky], dtype=z.dtype))


# ----------------------------------------------------------------------------
# Losses (model/losses.py:27-64,158-218)
# ----------------------------------------------------------------------------
def loss_rgb_depth(rgb, rgb_gt, depth_pred, depth_gt, mask, w_rgb, w_depth, rgb_loss_type="l1"):
    """Loss.forward restricted to the photometric + depth-L1 terms.
    Returns (loss_dict, g_rgb (N,3), g_depth_pred (N,), g_depth_gt (N,)) where the
    cotangents are d loss / d (dense outputs)."""
    dt = rgb.dtype.type
    N = rgb.shape[0]
    diff = rgb - rgb_gt
    if rgb_loss_type == "l1":                                           # losses.py:27-32
        l_rgb = np.abs(diff).sum() / dt(N); g_rgb = np.sign(diff) / dt(N)
    else:
        l_rgb = (diff * diff).sum() / dt(N); g_rgb = dt(2.0) * diff / dt(N)
    nm = int(mask.sum())
    dd = (depth_pred - depth_gt)[mask]
    l_depth = np.abs(dd).sum() / dt(max(nm, 1))                         # losses.py:59-61
    g_dp = np.zeros(N, dtype=rgb.dtype); g_dp[mask] = np.sign(dd) / dt(max(nm, 1))
    l2_mean = (diff * diff).mean()                                      # losses.py:192
    loss = dt(w_rgb) * l_rgb + dt(w_depth) * l_depth                    # losses.py:196-202
    d = dict(loss=loss, loss_rgb=l_rgb, loss_depth=l_depth, l2_mean=l2_mean)
    return d, (dt(w_rgb) * g_rgb).astype(rgb.dtype), dt(w_depth) * g_dp, -dt(w_depth) * g_dp


def chamfer(X, Y, chunk=2048):
    """Loss.get_pc_loss 'dense' (model/losses.py:114-148): symmetric mean nearest-neighbour
    L2 distance with argmin ties -> first index.  Returns (loss, gX, gY, idx_xy, idx_yx)."""
    def nn_idx(A, B):
        idx = np.empty(A.shape[0], dtype=np.int64)
        for s in range(0, A.shape[0], chunk):
            diff = A[s:s + chunk, None, :] - B[None, :, :]
            dist = np.sqrt((diff * diff).sum(-1))
            idx[s:s + chunk] = np.argmin(dist, axis=1)
        return idx
    gX = np.zeros_like(X); gY = np.zeros_like(Y)
    ixy = nn_idx(X, Y); v = X - Y[ixy]; n = np.sqrt((v * v).sum(-1))
    l1 = n.mean()
    with np.errstate(invalid="ignore", divide="ignore"):
        gv = np.where(n[:, None] > 0, v / n[:, None], 0) / X.shape[0]
    gX += gv; np.add.at(gY, ixy, -gv)
    iyx = nn_idx(Y, X); v = Y - X[iyx]; n = np.sqrt((v * v).sum(-1))
    l2 = n.mean()
    with np.errstate(invalid="ignore", divide="ignore"):
        gv = np.where(n[:, None] > 0, v / n[:, None], 0) / Y.shape[0]
    gY += gv; np.add.at(gX, iyx, -gv)
    return l1 + l2, gX, gY, ixy, iyx


# ----------------------------------------------------------------------------
# Reference-image stage of Trainer.compute_loss (model/training.py:280-365): point-cloud (chamfer)
# and warped-RGB terms between the current view and one reference view
# ----------------------------------------------------------------------------
REF_CFG = dict(nearest_limit=0.01, pc_ratio=4, scale_pcs=True, detach_rgbs_scale=False)   # configs/default.yaml training.*


def nearest_resize(d, res):
    """F.interpolate(d, res, mode='nearest') (training.py:318-319): src = floor(dst * in/out), scale in float32."""
    hd, wd = d.shape; h, w = res
    sr = np.minimum(np.floor(np.arange(h, dtype=np.float32) * np.float32(hd / h)).astype(np.int64), hd - 1)
    sc = np.minimum(np.floor(np.arange(w, dtype=np.float32) * np.float32(wd / w)).astype(np.int64), wd - 1)
    return d[sr][:, sc], sr, sc


def bilinear_resize(img, res):
    """F.interpolate(img, res, mode='bilinear') with align_corners=False, no antialiasing (training.py:326-327); img (C,H,W)."""
    C, H, W = img.shape; h, w = res; dt = img.dtype.type
    def axis(n_out, n_in):
        src = np.maximum((np.arange(n_out, dtype=img.dtype) + dt(0.5)) * dt(n_in / n_out) - dt(0.5), dt(0))
        i0 = np.minimum(np.floor(src).astype(np.int64), n_in - 1); i1 = np.minimum(i0 + 1, n_in - 1)
        return i0, i1, (src - i0.astype(img.dtype)).astype(img.dtype)
    y0, y1, ly = axis(h, H); x0, x1, lx = axis(w, W)
    top = img[:, y0][:, :, x0] * (1 - lx) + img[:, y0][:, :, x1] * lx
    bot = img[:, y1][:, :, x0] * (1 - lx) + img[:, y1][:, :, x1] * lx
    return top * (1 - ly)[None, :, None] + bot * ly[None, :, None]


def grid_sample_bilinear(img, xy, g_out=None):
    """F.grid_sample(img, xy, mode='bilinear', padding_mode='zeros', align_corners=True) for img (C,h,w), xy (P,2) in [-1,1]
    (get_tensor_values, model/common.py:75-109).  Returns values (P,C); with g_out (P,C) also d loss / d xy (P,2)."""
    C, h, w = img.shape; dt = img.dtype.type
    fx = (xy[:, 0] + dt(1)) * dt(0.5) * dt(w - 1); fy = (xy[:, 1] + dt(1)) * dt(0.5) * dt(h - 1)
    x0 = np.floor(fx); y0 = np.floor(fy)
    lx = fx - x0; ly = fy - y0
    x0 = x0.astype(np.int64); y0 = y0.astype(np.int64)
    def tap(yy, xx):
        ok = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
        v = img[:, np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].T            # (P,C)
        return np.where(ok[:, None], v, dt(0))
    v00, v01, v10, v11 = tap(y0, x0), tap(y0, x0 + 1), tap(y0 + 1, x0), tap(y0 + 1, x0 + 1)
    lx_, ly_ = lx[:, None], ly[:, None]
    out = v00 * (1 - lx_) * (1 - ly_) + v01 * lx_ * (1 - ly_) + v10 * (1 - lx_) * ly_ + v11 * lx_ * ly_
    if g_out is None:
        return out
    d_fx = ((v01 - v00) * (1 - ly_) + (v11 - v10) * ly_)
    d_fy = ((v10 - v00) * (1 - lx_) + (v11 - v01) * lx_)
    g_xy = np.stack([(g_out * d_fx).sum(1) * dt(0.5) * dt(w - 1), (g_out * d_fy).sum(1) * dt(0.5) * dt(h - 1)], -1)
    return out, g_xy


def ref_stage(img, ref_img, d_in_raw, d_ref_raw, c2w, c2w_ref, scale_in, shift_in, scale_ref, shift_ref, is_last, kx, ky,
              w_pc=1.0, w_rgb_s=1.0, cfg=REF_CFG):
    """Forward and adjoint of the reference-image stage (training.py:280-365) with the defaults `detach_ref_img: True`,
    `shift_first: False`, `match_method: dense`, `with_ssim: False`.

    img, ref_img (3,H,W); d_in_raw, d_ref_raw (h_d,w_d) raw DPT maps; c2w, c2w_ref (4,4); scale/shift: effective
    distortion of the two views; is_last: current view is the last camera (roles of the views swap, training.py:296-313).
    Returns (dict(loss_pc, loss_rgb_s), dict(c2w (4,4), scale, shift) = gradients of w_pc*loss_pc + w_rgb_s*loss_rgb_s w.r.t.
    the CURRENT view's pose matrix and effective distortion; the reference view is detached)."""
    dt = img.dtype.type
    nl = dt(cfg["nearest_limit"])
    hd, wd = d_in_raw.shape
    res = (int(hd / cfg["pc_ratio"]), int(wd / cfg["pc_ratio"]))
    P = res[0] * res[1]
    # pixel grid of the low-resolution maps (arange_pixels, common.py:13-39) and the two depth maps
    ys, xs = np.meshgrid(np.arange(res[0]), np.arange(res[1]), indexing="ij")
    px = (dt(2) * xs.reshape(-1).astype(img.dtype) / dt(res[1] - 1) - dt(1)); py = (dt(2) * ys.reshape(-1).astype(img.dtype) / dt(res[0] - 1) - dt(1))
    raw_in, _, _ = nearest_resize(d_in_raw, res); raw_ref, _, _ = nearest_resize(d_ref_raw, res)
    raw_in = raw_in.reshape(-1).astype(img.dtype); raw_ref = raw_ref.reshape(-1).astype(img.dtype)
    shift_first = bool(cfg.get("shift_first", False))
    if shift_first:                                                                               # training.py:241-245, 283-287
        din = (raw_in + dt(shift_in)) * dt(scale_in); dref = (raw_ref + dt(shift_ref)) * dt(scale_ref)
    else:
        din = raw_in * dt(scale_in) + dt(shift_in); dref = raw_ref * dt(scale_ref) + dt(shift_ref)
    live_in = din >= nl                                                                           # d[d < nl] = nl (training.py:320-321)
    din_c = np.where(live_in, din, nl); dref_c = np.where(dref >= nl, dref, nl)
    bp = lambda d: np.stack([px * d / dt(kx), py * d / dt(ky), -d], -1)                           # transform_to_world, identity pose
    if not is_last:
        d1, d2 = din_c, dref_c; img1, img2 = img, ref_img
        M = np.linalg.inv(c2w_ref) @ c2w                                                          # ref_Rt @ inverse(world_mat)
        s2 = dt(scale_ref)
    else:
        d1, d2 = dref_c, din_c; img1, img2 = ref_img, img
        inv_c2w = np.linalg.inv(c2w)
        M = inv_c2w @ c2w_ref                                                                     # world_mat @ inverse(ref_Rt)
        s2 = dt(scale_in)
    M = M.astype(img.dtype)
    R, t = M[:3, :3], M[:3, 3]
    pc1, pc2 = bp(d1), bp(d2)
    g_pc1 = np.zeros_like(pc1); g_pc2 = np.zeros_like(pc2); gR = np.zeros((3, 3), img.dtype); gt = np.zeros(3, img.dtype)
    g_s2 = dt(0)
    g_kxy = np.zeros(2, img.dtype)                   # d/d(kx, ky): LearnFocal reaches this stage through camera_mat (training.py:247-252)
    losses = dict(loss_pc=dt(0), loss_rgb_s=dt(0))
    # ---- warped-RGB term (training.py:325-341, losses.py:150-157,77-85) ----
    if w_rgb_s != 0.0:
        i1, i2 = bilinear_resize(img1, res), bilinear_resize(img2, res)
        rgb1 = grid_sample_bilinear(i1, np.stack([px, py], -1))
        Xr = pc1 @ R.T + t
        bad = (-Xr[:, 2] < nl)
        Xr_c = np.where(bad[:, None], nl, Xr)                                                     # behind-camera fix-up (:334-335)
        z = -Xr_c[:, 2]
        xy = np.stack([dt(kx) * Xr_c[:, 0] / z, dt(ky) * Xr_c[:, 1] / z], -1)                     # project_to_cam (common.py:436-457)
        valid = np.abs(xy).max(-1) <= 1
        nv = int(valid.sum()) * 3
        diff = rgb1 - grid_sample_bilinear(i2, xy)
        ad = np.clip(np.abs(diff), 0, 1)
        losses["loss_rgb_s"] = ad[valid].sum() / dt(max(nv, 1)) if nv > 0 else dt(0)
        if nv > 0:
            g_proj = np.where(valid[:, None] & (np.abs(diff) < 1), -np.sign(diff), dt(0)) * dt(w_rgb_s) / dt(nv)
            _, g_xy = grid_sample_bilinear(i2, xy, g_proj)
            gX = np.stack([g_xy[:, 0] * dt(kx) / z, g_xy[:, 1] * dt(ky) / z,
                           (g_xy[:, 0] * dt(kx) * Xr_c[:, 0] + g_xy[:, 1] * dt(ky) * Xr_c[:, 1]) / (z * z)], -1)
            gX = np.where(bad[:, None], dt(0), gX)
            g_kxy += np.array([(g_xy[:, 0] * Xr_c[:, 0] / z).sum(), (g_xy[:, 1] * Xr_c[:, 1] / z).sum()], img.dtype)   # xy = (kx X, ky Y) / z
            gR += gX.T @ pc1; gt += gX.sum(0)
            if not cfg["detach_rgbs_scale"]:
                g_pc1 += gX @ R
    # ---- point-cloud term (training.py:355-362, losses.py:114-148) ----
    if w_pc != 0.0:
        X = pc1 @ R.T + t; Y = pc2
        if cfg["scale_pcs"]:
            Xs, Ys = X / s2, Y / s2
        else:
            Xs, Ys = X, Y
        l, gXs, gYs, _, _ = chamfer(Xs, Ys)
        losses["loss_pc"] = l
        gXs = gXs * dt(w_pc); gYs = gYs * dt(w_pc)
        if cfg["scale_pcs"]:
            g_s2 = -((gXs * Xs).sum() + (gYs * Ys).sum()) / s2
            gX, gY = gXs / s2, gYs / s2
        else:
            gX, gY = gXs, gYs
        gR += gX.T @ pc1; gt += gX.sum(0); g_pc1 += gX @ R; g_pc2 += gY
    # ---- back to the current view's pose and distortion ----
    gM = np.zeros((4, 4), img.dtype); gM[:3, :3] = gR; gM[:3, 3] = gt
    if not is_last:
        g_c2w = np.linalg.inv(c2w_ref).T.astype(img.dtype) @ gM
        g_d = g_pc1[:, 0] * px / dt(kx) + g_pc1[:, 1] * py / dt(ky) - g_pc1[:, 2]                 # d1 = current view's depth
        g_scale_extra = dt(0)                                                                     # scale2 = detached reference scale
    else:
        g_inv = gM @ c2w_ref.T.astype(img.dtype)
        g_c2w = -(inv_c2w.T.astype(img.dtype) @ g_inv @ inv_c2w.T.astype(img.dtype))
        g_d = g_pc2[:, 0] * px / dt(kx) + g_pc2[:, 1] * py / dt(ky) - g_pc2[:, 2]                 # d2 = current view's depth
        g_scale_extra = g_s2                                                                      # scale2 = current view's scale
    g_d = np.where(live_in, g_d, dt(0))
    # back-projection (x d / kx, y d / ky, -d): d pc[:,0] / d kx = -pc[:,0] / kx
    g_kxy += np.array([-((g_pc1[:, 0] * pc1[:, 0]).sum() + (g_pc2[:, 0] * pc2[:, 0]).sum()) / dt(kx),
                       -((g_pc1[:, 1] * pc1[:, 1]).sum() + (g_pc2[:, 1] * pc2[:, 1]).sum()) / dt(ky)], img.dtype)
    if shift_first:
        g_scale, g_shift = (g_d * (raw_in + dt(shift_in))).sum(), (g_d * dt(scale_in)).sum()
    else:
        g_scale, g_shift = (g_d * raw_in).sum(), g_d.sum()
    grads = dict(c2w=g_c2w, scale=g_scale + g_scale_extra, shift=g_shift, kxy=g_kxy)
    return losses, grads


# ----------------------------------------------------------------------------
# Adam (torch.optim.Adam defaults as used at train.py:58,99,117)
# ----------------------------------------------------------------------------
def adam_step(p, g, m, v, step, lr, b1=0.9, b2=0.999, eps=1e-8):
    m *= b1; m += (1 - b1) * g
    v *= b2; v += (1 - b2) * g * g
    bc1 = 1 - b1 ** step; bc2 = 1 - b2 ** step
    p -= (lr / bc1) * m / (np.sqrt(v) / math.sqrt(bc2) + eps)


# ----------------------------------------------------------------------------
# One optimisation step (model/training.py:67-97 + compute_loss:197-378, render terms)
# ----------------------------------------------------------------------------
def _distortion(state, cam_id, dt, cfg):
    """Learn_Distortion.forward (distortions.py:19-27): (scale_eff, shift, scale is a live parameter)"""
    V = state["r"].shape[0]
    scale = state["scales"][cam_id, 0]; shift = state["shifts"][cam_id, 0]
    scale_eff, live = scale, True
    if scale < 0.01:
        scale_eff, live = dt(0.01), False
    if cfg.get("fix_scaleN", True) and cam_id == V - 1:
        scale_eff, live = dt(1.0), False
    return scale_eff, shift, live


def train_step(state, img, dpt, ray_idx, noise, cam_id, kx, ky, cfg, w_rgb=1.0, w_depth=0.04,
               rgb_loss_type="l1", lrs=(1e-3, 5e-4, 5e-4), apply_update=True, ref=None, focal=None):
    """Trainer.train_step: render + rgb + depth losses, and with ref = dict(img (3,H,W), dpt (h_d,w_d), idx, w_pc, w_rgb_s)
    also the reference-image stage (point-cloud + warped-RGB terms, training.py:280-365).
    state: dict(P, r (V,3), t (V,3), scales (V,1), shifts (V,1), adam={...}, step).
    img (3,H,W); dpt (h_d,w_d).  Returns loss dict + grads."""
    P = state["P"]; dt = img.dtype.type
    H, W = img.shape[1:]
    V = state["r"].shape[0]
    if focal is not None:              # LearnFocal order 2 (intrinsics.py:59-70): camera_mat = diag(fx^2, -fy^2, -1, 1) (training.py:247-252)
        kx, ky = dt(state["focal"][0]) ** 2, -dt(state["focal"][1]) ** 2
    r, t = state["r"][cam_id], state["t"][cam_id]
    init = state.get("init_c2w")
    c2w = make_c2w(r, t, None if init is None else init[cam_id])        # training.py:237
    scale = state["scales"][cam_id, 0]; shift = state["shifts"][cam_id, 0]
    scale_eff, scale_live = scale, True                                  # distortions.py:19-27
    if scale < 0.01:
        scale_eff, scale_live = dt(0.01), False
    if cfg.get("fix_scaleN", True) and cam_id == V - 1:
        scale_eff, scale_live = dt(1.0), False
    raw, _ = gather_prior_depth(dpt, ray_idx, H, W)
    depth = raw * scale_eff + shift                                     # training.py:241-245
    pixels = pixels_from_idx(ray_idx, H, W, img.dtype.type)             # training.py:257-262
    rgb_gt = img.reshape(3, -1)[:, ray_idx].T
    out, cache = render_forward(P, pixels, depth.astype(img.dtype), c2w, kx, ky, cfg, noise=noise)
    ld, g_rgb, g_dp, g_dg = loss_rgb_depth(out["rgb"], rgb_gt, out["depth_pred_full"], out["depth_gt_full"],
                                           out["mask"], w_rgb, w_depth, rgb_loss_type)
    gr = render_backward(P, cache, g_rgb, g_dp, g_dg)
    g_c2w = gr["c2w"]
    g_kxy = gr["kxy"].copy()
    g_scale = (gr["depth"] * raw).sum() if scale_live else dt(0)
    g_shift = gr["depth"].sum()
    if ref is not None:
        ri = int(ref["idx"])
        c2w_ref = make_c2w(state["r"][ri], state["t"][ri], None if init is None else init[ri])
        s_ref, h_ref, _ = _distortion(state, ri, dt, cfg)
        w_pc, w_rgb_s = ref.get("w_pc", 1.0), ref.get("w_rgb_s", 1.0)
        rl, rg = ref_stage(img, ref["img"], dpt, ref["dpt"], c2w, c2w_ref, scale_eff, shift, s_ref, h_ref, cam_id == V - 1, kx, ky,
                           w_pc=w_pc, w_rgb_s=w_rgb_s)
        ld["loss_pc"] = rl["loss_pc"]; ld["loss_rgb_s"] = rl["loss_rgb_s"]
        ld["loss"] = ld["loss"] + dt(w_pc) * rl["loss_pc"] + dt(w_rgb_s) * rl["loss_rgb_s"]
        g_c2w = g_c2w + rg["c2w"]; g_kxy = g_kxy + rg["kxy"]
        g_scale = g_scale + (rg["scale"] if scale_live else dt(0)); g_shift = g_shift + rg["shift"]
    g_r, g_t = make_c2w_bwd(r, t, None if init is None else init[cam_id], g_c2w)
    grads = dict(P=gr["params"], r=g_r, t=g_t, scale=g_scale, shift=g_shift, c2w=g_c2w, kxy=g_kxy)
    if focal is not None:
        grads["focal"] = np.array([g_kxy[0] * 2 * state["focal"][0], -g_kxy[1] * 2 * state["focal"][1]], img.dtype)
        ld["focalx"] = kx / dt(focal["kx_gt"]); ld["focaly"] = -ky / dt(focal["ky_gt"])    # training.py:372-375
    if apply_update:
        state["step"] = state.get("step", 0) + 1
        ad = state.setdefault("adam", {})
        for n in PARAM_NAMES:
            m = ad.setdefault("m." + n, np.zeros_like(P[n])); v = ad.setdefault("v." + n, np.zeros_like(P[n]))
            adam_step(P[n], gr["params"][n].astype(P[n].dtype), m, v, state["step"], lrs[0])
        G_r = np.zeros_like(state["r"]); G_r[cam_id] = g_r
        G_t = np.zeros_like(state["t"]); G_t[cam_id] = g_t
        G_s = np.zeros_like(state["scales"]); G_s[cam_id, 0] = g_scale
        G_h = np.zeros_like(state["shifts"]); G_h[cam_id, 0] = g_shift
        for key, Gk, lr in (("r", G_r, lrs[1]), ("t", G_t, lrs[1]), ("scales", G_s, lrs[2]), ("shifts", G_h, lrs[2])):
            m = ad.setdefault("m." + key, np.zeros_like(state[key])); v = ad.setdefault("v." + key, np.zeros_like(state[key]))
            adam_step(state[key], Gk, m, v, state["step"], lr)
        if focal is not None:
            m = ad.setdefault("m.focal", np.zeros_like(state["focal"])); v = ad.setdefault("v.focal", np.zeros_like(state["focal"]))
            adam_step(state["focal"], grads["focal"].astype(state["focal"].dtype), m, v, state["step"], focal.get("lr", 1e-3))
    ld["scale"] = scale_eff; ld["shift"] = shift
    return ld, grads, out

"""Layer-local float64 checks of every MLP GEMM of both engines, on real data.

A seeded render forward (NNB_STASH) and backward (with weight gradients) runs on the GPU; then every GEMM is rebuilt in float64, on the
device, from the kernel's OWN inputs read back from the workspace stash, so ReLU gates that flip between fp32 evaluation orders cannot
enter:
- forward: h0 from enc[:, :63], h_l from h_{l-1} ([h3, enc] at layer 4), feat, hr from [feat, denc[:, :27]], and the colour,
  density-logit and a = density_act(logit) entries of the per-sample records (SampleRec, nnb_common.cuh);
- data gradient: dyc from gs and the records (head_ref: density_act_grad of every head, softplus or ReLU, alpha or dist_alpha's sigma,
  or the raw logit), dyr (gate: the kernel's hr > 0), dfeat, dy7 (with dsigma w_sigma), dy6..dy0 (gates from the kernel's h stash);
- weight gradient: every job's dW and db from the dy and h stash (the bf16 hi | lo conversion of values that span decades).

Each element's error is normalised by a scale from its own operands: u sqrt(sum_k (a_k b_k)^2) with u = 2^-24 (bias and added terms
included).  The forward of the tensor-core engine adds 2^-25 sqrt(sum_k (a_k^2 + b_k^2)) for the fp16 lo halves that are subnormal or
vanish.  The gradients add 2^-126 sqrt(sum_k (a_k^2 + b_k^2)) + 2^-126: samples far behind a surface carry gradients below the fp32
normal range (up to 9 % of the dy entries at 1024 x 128), which the kernels do not resolve (bf16 conversion, fp32 FMA); without this
term such an entry scores ~1e7 on both engines.  dyc is normalised by 8 u |value| + 2^-126, the colours by sigma'(logit) times the
logit's scale plus 4 u.

Largest normalised errors measured over all cases below on the unmodified kernels (NVIDIA H100 80GB HBM3, 700 W power limit), and the
gates (at most 4x those, and at most a tenth of the smallest wrong answer):
  tensor-core forward          13.9  (D = 256, 1024 x 128) -> 42
  tensor-core data gradient     468  (D = 128, 1024 x 128) -> 1870
  tensor-core weight gradient  1334  (D = 256, 1024 x 128) -> 3300
  SIMT forward                 47.8  (D = 256, 1024 x 128) -> 190
  SIMT data gradient           70.5  (D = 256, 1024 x 128) -> 280
  SIMT weight gradient          228  (D = 128, 301 x 17)   -> 680
The SIMT gates also serve the exact engine's explicit-point queries (test_gpu_field_local.py: 49.8, 51.0 and 139 there).  The SIMT
cases cover every width at 301 x 17 and 1024 x 128, and D = 64 / 128 at 64 x 2 and 64 x 15 (sample counts below the tensor-core
engine's 16, where the exact engine is the production engine).
Each gate has teeth: from the same stash, in float64, wrong answers must each exceed the gate at least 10x in every case and for every
layer or job: the lo half of the weight operand dropped (fp16 forward, bf16 data gradient) or of dY (weight gradient), one 16-wide K-step
omitted (forward, data gradient), the heaviest 32-sample chunk omitted (weight gradient), one bias (or dsigma w_sigma, or a bias chunk)
omitted, (data gradient) the layer's own ReLU gate instead of the one below, and the density head's alpha factor exp(-sigma) dropped
(alpha) or added (dist_alpha), and softplus' slope used for ReLU or ReLU's for softplus.  The margins are thin for the dropped lo
halves: the smallest wrong answers measured are 513 (tensor-core forward, 12x its gate), 3.76e4 (tensor-core weight gradient, 11x) and
3290 (SIMT forward of an explicit-point query, 17x); raising a gate, or a case with larger errors, can make these teeth assertions fail
without any kernel change.  The head's wrong answers score at least 1.89e6 in this module's cases.

Density heads (test_head_layer_local, both engines): softplus with dist_alpha at 1024 x 128 and 301 x 17, ReLU with alpha and with
dist_alpha at 301 x 17 (D = 256), ReLU with dist_alpha and softplus with alpha at D = 64.  fc_density is scaled and shifted from a first
run's logits so that the largest is 24 (alpha) or 200 (dist_alpha) and the upper quartile starts at 0: softplus logits above its
threshold 20, ReLU logits on both sides of 0, and samples whose alpha is within 1e-6 of 1, each branch held by at least 3 samples
(measured: at least 9).  These cases stay within the gates above (largest: tensor-core data gradient 454, weight gradient 880; SIMT 47.8,
61.9, 74.5).

The small-activation case (D = 256, 301 x 17) scales layer 0's weights, the encoding columns of layer 4 and every trunk bias by 2^-6:
ReLU layers are positively homogeneous, so every trunk activation is 2^-6 times that of the unscaled field.  The non-zero activations of
layers 1..6 then measured 9.5e-5 (5th percentile) .. 1.1e-3 (median) .. 0.026 (largest): below 2^-3, where the fp16 lo half is
subnormal.  The case passes the same gates (forward 2.6, data gradient 400, weight gradient 513), but the fp16 term is then as large as
the error of dropping the weights' lo half (11.6), so that wrong answer is not asserted there.  Against the plain fp32 scale (no fp16
term) the trunk layers score 3890 there against at most 211 on the unscaled fields: the split-fp16 forward is not fp32-accurate for
activations below ~2^-3 (DESIGN.md section 6); test_tc_small_activations_fp32_scale records that as an expected failure."""
import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
from test_gpu_relu_mask import _render, layout

U = 2.0 ** -24
SUB = 2.0 ** -25
TINY = 2.0 ** -126   # smallest normal fp32
GATES = dict(fwd=42.0, dgrad=1870.0, wgrad=3300.0)   # tensor-core engine, see the module docstring
SIMT_GATES = dict(fwd=190.0, dgrad=280.0, wgrad=680.0)   # exact engine, render and explicit-point cases, see the module docstring
FP32_TRUNK_GATE = 640.0   # forward trunk layers against the plain fp32 scale: 3x the 211 measured (D = 256, 1024 x 128)
SMALL_SCALE = 2.0 ** -6
TC_CASES = [(D, N, S) for D in (64, 128, 256) for (N, S) in ((1024, 128), (301, 17), (333, 16), (9, 1024))]
SIMT_CASES = [(D, N, S) for D in (64, 128, 256) for (N, S) in ((301, 17), (1024, 128))] + \
    [(D, 64, S) for D in (64, 128) for S in (2, 15)]   # sample counts below the tensor-core engine's 16
# density heads (occupancy activation, dist_alpha) other than the default (softplus, alpha), and that one with planted logits
HEAD_CASES = [("softplus", True, 256, 1024, 128), ("softplus", True, 256, 301, 17), ("relu", False, 256, 301, 17),
              ("relu", True, 256, 301, 17), ("relu", True, 64, 301, 17), ("softplus", False, 64, 301, 17)]
# the largest planted logit: near-opaque samples (alpha >= 1 - 1e-7 needs sigma >= 16.2, and with dist_alpha sigma delta >= 16.2 at
# sample spacings down to 0.08), and softplus logits above its threshold 20
HEAD_TARGET = {False: 24.0, True: 200.0}
TRUNK = [("layers0", 0), ("layers0", 2), ("layers0", 4), ("layers0", 6), ("layers1", 0), ("layers1", 2), ("layers1", 4), ("layers1", 6)]


# -------------------------------------------------------------------------------------------------------------------- read back
def _f32(ws, off, rows, cols):
    return ws[off:off + rows * cols * 4].view(torch.float32).view(rows, cols)


def run(engine, D, N, S, P, backward=True, flags=None):
    """forward (+ backward with weight gradients); returns (stash dict of float64 [M, cols] tensors, float64 weights dict, weight
    gradients dict or None); flags: the rendering flags (default: _render's)"""
    from nope_nerf_b200 import _lib as L
    call = _render(P, D, N, S, seed=11, engine=L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT, flags=flags)
    ws = call.ws
    lay = layout(N, S, D)
    G = None
    if backward:
        rng = np.random.default_rng(7)
        cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
        g_rgb = cu(rng.normal(0, 1, (N, 3)).astype(np.float32))
        g_dp = cu(rng.normal(0, 1, N).astype(np.float32)); g_dg = cu(rng.normal(0, 1, N).astype(np.float32))
        g_w = torch.zeros(L.num_params(D), device="cuda")
        g_c2w = torch.zeros(4, 4, device="cuda"); g_cam = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
        call.backward(g_rgb, g_dp, g_dg, g_w, g_c2w, g_cam, None, g_ss)   # hands the workspace back to the pool; ws stays alive
    torch.cuda.synchronize()
    Mp, DR = lay["Mpad"], D // 2
    st = {"h%d" % l: _f32(ws, lay["h"][l], Mp, D) for l in range(8)}
    st.update(feat=_f32(ws, lay["feat"], Mp, D), hr=_f32(ws, lay["hr"], Mp, DR), enc=_f32(ws, lay["enc"], Mp, 64)[:, :63],
              denc=_f32(ws, lay["denc"], Mp, 32)[:, :27], rec=_f32(ws, lay["rec"], Mp, 8))
    if backward:
        st.update({"dy%d" % l: _f32(ws, lay["dy"][l], Mp, D) for l in range(8)})
        st.update(dfeat=_f32(ws, lay["dfeat"], Mp, D), dyr=_f32(ws, lay["dyr"], Mp, DR), dyc=_f32(ws, lay["dyc"], Mp, 4),
                  gs=_f32(ws, lay["gs"], Mp, 4))
        G = {k: torch.from_numpy(v.astype(np.float64)).cuda() for k, v in O.unflatten_params(g_w.cpu().numpy(), D).items()}
    st = {k: v[:lay["M"]].double() for k, v in st.items()}   # copies, taken before the workspace can be reused
    st["flags"] = call.args.flags
    if not backward:
        call.release()
    W = {k: torch.from_numpy(np.asarray(v, np.float64)).cuda() for k, v in P.items()}
    return st, W, G


# ------------------------------------------------------------------------------------------------------------------ density head
def head_of(flags):
    """(occupancy activation, dist_alpha, raw logit) of a flag word"""
    from nope_nerf_b200 import _lib as L
    return ("softplus" if flags & L.SOFTPLUS else "relu"), bool(flags & L.DIST_ALPHA), bool(flags & L.RAW_DENSITY)


def head_ref(s, occ, dist, raw=False, ds_occ=None):
    """float64 density_act and density_act_grad (nnb_common.cuh) at the kernel's own logits s: (a, d a / d s).  softplus as torch's
    F.softplus (beta 1, threshold 20: s > 20 gives s and slope 1), ReLU with slope 0 at s <= 0; a = 1 - exp(-sigma) with slope
    exp(-sigma) sigma' (alpha), a = sigma (dist_alpha), or a = s (raw logit, slope 1).  ds_occ: the activation whose slope is used
    (a wrong answer when it is not occ)"""
    if raw:
        return s, torch.ones_like(s)
    sig = torch.where(s > 20, s, torch.log1p(torch.exp(s.clamp_max(20)))) if occ == "softplus" else s.clamp_min(0)
    if (ds_occ or occ) == "softplus":
        ds = torch.where(s > 20, torch.ones_like(s), torch.sigmoid(s))
    else:
        ds = (s > 0).to(s.dtype)
    if dist:
        return sig, ds
    e = torch.exp(-sig)
    return 1 - e, e * ds


def head_scale(s, occ, dist, raw=False):
    """error scale of the kernel's a = density_act(s) in fp32: softplus (expf, log1pf) within 4 ulp of sigma, then (alpha) expf within
    2 ulp of e = exp(-sigma) and the rounded 1 - e; plus the fp32 underflow term"""
    if raw:
        return torch.full_like(s, TINY)
    a, _ = head_ref(s, occ, dist)
    sig, _ = head_ref(s, occ, True)
    ssig = 4 * U * sig.abs() if occ == "softplus" else torch.zeros_like(s)
    if dist:
        return ssig + TINY
    e = torch.exp(-sig)
    return U * a.abs() + 2 * U * e + e * ssig + TINY


def plant_logits(engine, D, N, S, P, flags, target):
    """P with fc_density scaled and shifted (a first run's logits s = h7 . w + b) so that the largest logit is `target` and the upper
    quartile starts at 0: a quarter of the samples with positive logits, a few near `target`, the rest negative.  Returns a copy."""
    from nope_nerf_b200 import _lib as L
    lay = layout(N, S, D)
    probe = _render(P, D, N, S, seed=11, engine=L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT, flags=flags)
    M = N * S
    s0 = probe.ws[lay["rec"]:lay["rec"] + M * 32].view(torch.float32).view(M, 8)[:, 4].double()
    probe.release()
    m = s0 - float(P["fc_density.bias"][0])
    q = float(torch.quantile(m, 0.75))
    k = target / (float(m.max()) - q)
    P = dict(P)
    P["fc_density.weight"] = (P["fc_density.weight"] * np.float32(k)).astype(np.float32)
    P["fc_density.bias"] = np.full_like(P["fc_density.bias"], -k * q)
    return P


def head_branches(st):
    """samples in each branch of the density head of the run's flags: {branch: count}; the composited alpha of a sample is its rec.a
    (alpha) or 1 - exp(-sigma delta) (dist_alpha, the last sample of a ray excluded)"""
    occ, dist, _ = head_of(st["flags"])
    s, a, z = st["rec"][:, 4], st["rec"][:, 3], st["rec"][:, 5]
    out = {"s>20": int((s > 20).sum()), "s<=20": int((s <= 20).sum())} if occ == "softplus" else \
        {"s>0": int((s > 0).sum()), "s<=0": int((s <= 0).sum())}
    if dist:
        alpha = 1 - torch.exp(-a[:-1] * (z[1:] - z[:-1]))
        alpha = alpha[(z[1:] - z[:-1]) > 0]   # within a ray: z increases
    else:
        alpha = a
    out["alpha>=1-1e-6"] = int((alpha >= 1 - 1e-6).sum())
    return out


# ------------------------------------------------------------------------------------------------------------------ error model
def gemm_ref(A, B, bias=None, extra=None, fp16_abs=False, tiny=False):
    """y = A B^T (+ bias) (+ extra); and the per-element scale u sqrt(sum_k (a_k b_k)^2 + bias^2 + extra^2), plus the fp16 term
    (fp16_abs) or the fp32-underflow term (tiny)"""
    y = A @ B.T
    s2 = (A * A) @ (B * B).T
    if bias is not None:
        y = y + bias; s2 = s2 + bias * bias
    if extra is not None:
        y = y + extra; s2 = s2 + extra * extra
    scale = U * s2.sqrt()
    if fp16_abs or tiny:
        q = SUB if fp16_abs else TINY
        scale = scale + q * ((A * A).sum(1, keepdim=True) + (B * B).sum(1)[None, :]).sqrt()
    if tiny:
        scale = scale + TINY
    return y, scale


def nerr(got, ref, scale):
    """largest |got - ref| / scale (0 where both are exactly equal)"""
    d = (got - ref).abs()
    return float(torch.where(d == 0, torch.zeros_like(d), d / scale.clamp_min(1e-300)).max())


def fp16_hi(x):
    return x.float().half().double()


def bf16_hi(x):
    return x.float().bfloat16().double()


def drop_chunk(A):
    """A (samples x features) with the 32-sample chunk of largest sum |A| zeroed: the chunk whose loss matters most"""
    w = A.abs().sum(1)
    w = torch.cat([w, w.new_zeros((-w.numel()) % 32)]).view(-1, 32).sum(1)
    c = int(w.argmax())
    A = A.clone(); A[32 * c:32 * c + 32] = 0; return A


def drop_k(A, j):
    """A with the 16 columns of K-step j zeroed"""
    A = A.clone(); A[:, 16 * j:16 * j + 16] = 0; return A


# ---------------------------------------------------------------------------------------------------------------------- checks
def forward_errors(st, W, D, tc):
    """{'err': largest normalised error of the forward GEMMs and heads, 'err_fp32_trunk': that of the trunk layers without the fp16 term,
    'teeth': {kind: smallest over layers of the wrong answer's}}"""
    err, err32, teeth = 0.0, 0.0, {"lo": [], "kstep": [], "bias": []}
    for l, (blk, i) in enumerate(TRUNK):
        X = st["enc"] if l == 0 else (torch.cat([st["h3"], st["enc"]], 1) if l == 4 else st["h%d" % (l - 1)])
        Wl, b = W["%s.%d.weight" % (blk, i)], W["%s.%d.bias" % (blk, i)]
        y, sc = gemm_ref(X, Wl, b, fp16_abs=tc)
        got = st["h%d" % l]
        err = max(err, nerr(got, y.clamp_min(0), sc))
        err32 = max(err32, nerr(got, y.clamp_min(0), gemm_ref(X, Wl, b)[1]))
        teeth["lo"].append(nerr(got, (X @ fp16_hi(Wl).T + b).clamp_min(0), sc))
        teeth["kstep"].append(nerr(got, (drop_k(X, 1) @ Wl.T + b).clamp_min(0), sc))
        teeth["bias"].append(nerr(got, (X @ Wl.T).clamp_min(0), sc))
    Xf, Wf, bf = st["h7"], W["fc_feature.weight"], W["fc_feature.bias"]
    y, sc = gemm_ref(Xf, Wf, bf, fp16_abs=tc)
    err = max(err, nerr(st["feat"], y, sc))
    teeth["lo"].append(nerr(st["feat"], Xf @ fp16_hi(Wf).T + bf, sc))
    teeth["kstep"].append(nerr(st["feat"], drop_k(Xf, 1) @ Wf.T + bf, sc))
    teeth["bias"].append(nerr(st["feat"], Xf @ Wf.T, sc))
    Xr, Wr, br = torch.cat([st["feat"], st["denc"]], 1), W["rgb_layers.0.weight"], W["rgb_layers.0.bias"]
    y, sc = gemm_ref(Xr, Wr, br, fp16_abs=tc)
    err = max(err, nerr(st["hr"], y.clamp_min(0), sc))
    teeth["lo"].append(nerr(st["hr"], (Xr @ fp16_hi(Wr).T + br).clamp_min(0), sc))
    teeth["kstep"].append(nerr(st["hr"], (drop_k(Xr, 1) @ Wr.T + br).clamp_min(0), sc))
    teeth["bias"].append(nerr(st["hr"], (Xr @ Wr.T).clamp_min(0), sc))
    # heads (fp32 FMA in the epilogue): density logit and colours of the records {r, g, b, a, s, z, 0, 0}
    rec = st["rec"]
    s, sc = gemm_ref(st["h7"], W["fc_density.weight"], W["fc_density.bias"])
    err = max(err, nerr(rec[:, 4:5], s, sc))
    occ, dist, raw = head_of(st["flags"])   # the record's a = density_act(s) of the kernel's own logit
    err = max(err, nerr(rec[:, 3], head_ref(rec[:, 4], occ, dist, raw)[0], head_scale(rec[:, 4], occ, dist, raw)))
    yc, sc = gemm_ref(st["hr"], W["fc_rgb.weight"], W["fc_rgb.bias"])
    sg = torch.sigmoid(yc)
    err = max(err, nerr(rec[:, 0:3], sg, sg * (1 - sg) * sc + 4 * U * sg))
    return dict(err=err, err_fp32_trunk=err32, teeth={k: min(v) for k, v in teeth.items()})


def dgrad_errors(st, W, D):
    err, teeth = 0.0, {"lo": [], "kstep": [], "bias": [], "gate": []}
    rec, gs = st["rec"], st["gs"]
    # dyc: d/d(colour logits) = gs * c (1 - c), d/d density logit = gs_a * density_act_grad(s) (head_ref)
    c, s = rec[:, 0:3], rec[:, 4]
    occ, dist, raw = head_of(st["flags"])
    dyc = torch.cat([gs[:, :3] * c * (1 - c), (gs[:, 3] * head_ref(s, occ, dist, raw)[1])[:, None]], 1)
    sc = 8 * U * dyc.abs() + TINY
    err = max(err, nerr(st["dyc"], dyc, sc))
    if not raw:   # wrong heads: the alpha factor exp(-sigma) dropped (alpha) or added (dist_alpha); the other activation's slope
        got = st["dyc"][:, 3]
        teeth["head_factor"] = [nerr(got, gs[:, 3] * head_ref(s, occ, not dist)[1], sc[:, 3])]
        other = "relu" if occ == "softplus" else "softplus"
        teeth["head_slope"] = [nerr(got, gs[:, 3] * head_ref(s, occ, dist, ds_occ=other)[1], sc[:, 3])]
    # dyr = (dyc[:, :3] W_rgb) * (hr > 0)
    y, sc = gemm_ref(st["dyc"][:, :3], W["fc_rgb.weight"].T, tiny=True)
    err = max(err, nerr(st["dyr"], y * (st["hr"] > 0), sc))
    # dfeat = dyr W_rgbh[:, :D]
    Wr = W["rgb_layers.0.weight"][:, :D]
    y, sc = gemm_ref(st["dyr"], Wr.T, tiny=True)
    err = max(err, nerr(st["dfeat"], y, sc))
    teeth["lo"].append(nerr(st["dfeat"], st["dyr"] @ bf16_hi(Wr), sc))
    teeth["kstep"].append(nerr(st["dfeat"], drop_k(st["dyr"], 1) @ Wr, sc))
    # dy7 = (dfeat W_feat + dsigma w_sigma) * (h7 > 0): the added term plays the part of a bias
    Wf = W["fc_feature.weight"]
    add = st["dyc"][:, 3:4] * W["fc_density.weight"]
    y, sc = gemm_ref(st["dfeat"], Wf.T, extra=add, tiny=True)
    g7 = st["h7"] > 0
    err = max(err, nerr(st["dy7"], y * g7, sc))
    teeth["lo"].append(nerr(st["dy7"], (st["dfeat"] @ bf16_hi(Wf) + add) * g7, sc))
    teeth["kstep"].append(nerr(st["dy7"], (drop_k(st["dfeat"], 1) @ Wf + add) * g7, sc))
    teeth["bias"].append(nerr(st["dy7"], (st["dfeat"] @ Wf) * g7, sc))
    # dy_{l-1} = (dy_l W_l[:, :D]) * (h_{l-1} > 0)
    for l in range(7, 0, -1):
        blk, i = TRUNK[l]
        Wl = W["%s.%d.weight" % (blk, i)][:, :D]
        dy, got = st["dy%d" % l], st["dy%d" % (l - 1)]
        y, sc = gemm_ref(dy, Wl.T, tiny=True)
        gate = st["h%d" % (l - 1)] > 0
        err = max(err, nerr(got, y * gate, sc))
        teeth["lo"].append(nerr(got, (dy @ bf16_hi(Wl)) * gate, sc))
        teeth["kstep"].append(nerr(got, (drop_k(dy, 1) @ Wl) * gate, sc))
        teeth["gate"].append(nerr(got, y * (st["h%d" % l] > 0), sc))   # this layer's own gate instead of the one below
    return dict(err=err, teeth={k: min(v) for k, v in teeth.items()})


def wgrad_jobs(st, D):
    """(parameter, dY, X, column slice of the weight, bias parameter or None) of every weight-gradient job"""
    jobs = []
    for l, (blk, i) in enumerate(TRUNK):
        X = st["enc"] if l == 0 else st["h%d" % (l - 1)]
        jobs.append(("%s.%d.weight" % (blk, i), st["dy%d" % l], X, slice(0, X.shape[1]), "%s.%d.bias" % (blk, i)))
    jobs.append(("layers1.0.weight", st["dy4"], st["enc"], slice(D, D + 63), None))
    jobs.append(("fc_density.weight", st["dyc"][:, 3:4], st["h7"], slice(0, D), "fc_density.bias"))
    jobs.append(("fc_feature.weight", st["dfeat"], st["h7"], slice(0, D), "fc_feature.bias"))
    jobs.append(("rgb_layers.0.weight", st["dyr"], st["feat"], slice(0, D), "rgb_layers.0.bias"))
    jobs.append(("rgb_layers.0.weight", st["dyr"], st["denc"], slice(D, D + 27), None))
    jobs.append(("fc_rgb.weight", st["dyc"][:, :3], st["hr"], slice(0, D // 2), "fc_rgb.bias"))
    return jobs


def wgrad_errors(st, G, D):
    """every job's dW = dY^T X and db = sum dY over the samples; the wrong answers drop dY's bf16 lo half or one 32-sample chunk"""
    err, teeth = 0.0, {"lo": [], "chunk": [], "bias": []}
    for name, dY, X, cols, bname in wgrad_jobs(st, D):
        y, sc = gemm_ref(dY.T.contiguous(), X.T.contiguous(), tiny=True)
        got = G[name][:, cols]
        err = max(err, nerr(got, y, sc))
        teeth["lo"].append(nerr(got, bf16_hi(dY).T @ X, sc))
        teeth["chunk"].append(nerr(got, drop_chunk(dY).T @ X, sc))
        if bname:
            scb = U * (dY * dY).sum(0).sqrt() + TINY
            err = max(err, nerr(G[bname], dY.sum(0), scb))
            teeth["bias"].append(nerr(G[bname], drop_chunk(dY).sum(0), scb))
    return dict(err=err, teeth={k: min(v) for k, v in teeth.items()})


def small_params(D):
    """trunk activations scaled by SMALL_SCALE (see the module docstring)"""
    P = O.init_params(seed=5, D=D)
    P["layers0.0.weight"] *= SMALL_SCALE
    P["layers1.0.weight"][:, D:] *= SMALL_SCALE
    for blk, i in TRUNK:
        P["%s.%d.bias" % (blk, i)] *= SMALL_SCALE
    return P


def _check(key, out, gates, skip_teeth=()):
    for stage, gate in gates.items():
        r = out[stage]
        assert r["err"] <= gate, (key, stage, r["err"], gate)
        for kind, t in r["teeth"].items():
            if (stage, kind) not in skip_teeth:
                assert t >= 10 * gate, (key, stage, "wrong answer '%s' within 10x of the gate" % kind, t, gate)


def measure(engine, D, N, S, P, flags=None):
    st, W, G = run(engine, D, N, S, P, flags=flags)
    return dict(fwd=forward_errors(st, W, D, engine == "tc"), dgrad=dgrad_errors(st, W, D), wgrad=wgrad_errors(st, G, D)), st


def _report(key, out):
    print(key, {k: round(v["err"], 2) for k, v in out.items()},
          {(k, t): round(x, 1) for k, v in out.items() for t, x in v["teeth"].items()})


@pytest.mark.gpu
@pytest.mark.parametrize("D,N,S", TC_CASES)
def test_tc_layer_local(D, N, S):
    out, _ = measure("tc", D, N, S, O.init_params(seed=5, D=D))
    _report(("tc", D, N, S), out)
    _check(("tc", D, N, S), out, GATES)
    assert out["fwd"]["err_fp32_trunk"] <= FP32_TRUNK_GATE, out["fwd"]["err_fp32_trunk"]


@pytest.mark.gpu
@pytest.mark.parametrize("D,N,S", SIMT_CASES)
def test_simt_layer_local(D, N, S):
    out, _ = measure("simt", D, N, S, O.init_params(seed=5, D=D))
    _report(("simt", D, N, S), out)
    _check(("simt", D, N, S), out, SIMT_GATES)


def head_flags(occ, dist):
    from nope_nerf_b200 import ops
    cfg = dict(O.DEFAULT_CFG, dist_alpha=dist)
    return ops.flags_from_cfg(cfg, occ)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ("tc", "simt"))
@pytest.mark.parametrize("occ,dist,D,N,S", HEAD_CASES)
def test_head_layer_local(engine, occ, dist, D, N, S):
    """every density head, with its logits planted across the branches of density_act_grad"""
    flags = head_flags(occ, dist)
    P = plant_logits(engine, D, N, S, O.init_params(seed=5, D=D), flags, HEAD_TARGET[dist])
    out, st = measure(engine, D, N, S, P, flags)
    br = head_branches(st)
    _report((engine, occ, dist, D, N, S), out)
    print("  branches", br)
    assert min(br.values()) >= 3, br
    gates = GATES if engine == "tc" else SIMT_GATES
    _check((engine, occ, dist, D, N, S), out, gates)
    assert set(out["dgrad"]["teeth"]) >= {"head_factor", "head_slope"}


@pytest.mark.gpu
def test_tc_small_activations():
    D, N, S = 256, 301, 17
    out, st = measure("tc", D, N, S, small_params(D))
    nz = torch.cat([st["h%d" % l][st["h%d" % l] > 0] for l in range(1, 7)])
    p5, top = float(torch.quantile(nz.float(), 0.05)), float(nz.max())
    assert 2.0 ** -14 <= p5 and top <= 2.0 ** -3, (p5, top)
    _check(("tc-small", D, N, S), out, GATES, skip_teeth=(("fwd", "lo"),))


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="split-fp16 forward is not fp32-accurate for activations below ~2^-3 (DESIGN.md section 6)")
def test_tc_small_activations_fp32_scale():
    D, N, S = 256, 301, 17
    out, _ = measure("tc", D, N, S, small_params(D))
    assert out["fwd"]["err_fp32_trunk"] <= FP32_TRUNK_GATE, out["fwd"]["err_fp32_trunk"]


HEAD_LOGITS = np.concatenate([np.linspace(-30, 30, 241), [0.0, -0.0, 1e-30, -1e-30, 19.999, 20.0, np.nextafter(20.0, 21.0), 103.0,
                                                           200.0, -200.0]])


@pytest.mark.parametrize("occ", ("softplus", "relu"))
@pytest.mark.parametrize("dist", (False, True))
def test_head_ref_matches_autograd_and_oracle(occ, dist):
    """head_ref's value and slope equal float64 torch autograd of official_nerf.py's activations (F.softplus beta 1 threshold 20, or
    F.relu; then 1 - exp(-sigma) unless dist_alpha) and the density-head adjoint of oracle.nerf_oracle.mlp_backward, on logits that
    cover every branch (the threshold 20 and its neighbours, +-0, saturated and vanishing exp(-sigma))"""
    s = torch.tensor(HEAD_LOGITS, dtype=torch.float64)
    a, da = head_ref(s, occ, dist)
    x = s.clone().requires_grad_(True)
    sig = torch.nn.functional.softplus(x, beta=1, threshold=20) if occ == "softplus" else torch.nn.functional.relu(x)
    y = sig if dist else 1 - torch.exp(-sig)
    g, = torch.autograd.grad(y.sum(), x)
    torch.testing.assert_close(a, y.detach(), rtol=1e-15, atol=0)
    torch.testing.assert_close(da, g, rtol=1e-14, atol=0)
    # the oracle's head adjoint, one logit at a time: g_s = d a / d s for g_a = 1 is its fc_density.bias gradient
    D = 64
    P = {k: np.asarray(v, np.float64) for k, v in O.init_params(seed=5, D=D).items()}
    _, _, cache = O.mlp_forward(P, np.zeros((1, 3)), np.ones((1, 3)), dist_alpha=dist, occ_activation=occ)
    ref = []
    for sv in HEAD_LOGITS:
        sv = np.array([sv])
        c = dict(cache, s=sv, sigma=O._softplus(sv) if occ == "softplus" else np.maximum(sv, 0))
        G, _, _ = O.mlp_backward(P, c, np.zeros((1, 3)), np.ones(1))
        ref.append(G["fc_density.bias"][0])
    np.testing.assert_allclose(da.numpy(), np.array(ref), rtol=1e-14, atol=0)
    # the raw logit (NNB_RAW_DENSITY): a = s, slope 1
    a, da = head_ref(s, occ, dist, raw=True)
    assert torch.equal(a, s) and torch.equal(da, torch.ones_like(s))


def test_head_wrong_answers_differ():
    """each wrong head of dgrad_errors differs from head_ref on the logits the GPU cases plant (both sides of 0, above 20)"""
    s = torch.tensor(HEAD_LOGITS, dtype=torch.float64)
    for occ in ("softplus", "relu"):
        other = "relu" if occ == "softplus" else "softplus"
        for dist in (False, True):
            _, da = head_ref(s, occ, dist)
            assert (head_ref(s, occ, not dist)[1] != da).sum() >= 10, (occ, dist)
            assert (head_ref(s, occ, dist, ds_occ=other)[1] != da).sum() >= 10, (occ, dist)


@pytest.mark.gpu
def test_reference_matches_numpy():
    """the device float64 references equal numpy float64 on the CPU (one small case, forward and weight gradient)"""
    D, N, S = 64, 9, 16
    st, W, G = run("tc", D, N, S, O.init_params(seed=5, D=D))
    h = {k: v.cpu().numpy() for k, v in st.items() if torch.is_tensor(v)}
    Wn = {k: v.cpu().numpy() for k, v in W.items()}
    for l, (blk, i) in enumerate(TRUNK):
        X = h["enc"] if l == 0 else (np.concatenate([h["h3"], h["enc"]], 1) if l == 4 else h["h%d" % (l - 1)])
        ref = X @ Wn["%s.%d.weight" % (blk, i)].T + Wn["%s.%d.bias" % (blk, i)]
        Xd = st["enc"] if l == 0 else (torch.cat([st["h3"], st["enc"]], 1) if l == 4 else st["h%d" % (l - 1)])
        dev, _ = gemm_ref(Xd, W["%s.%d.weight" % (blk, i)], W["%s.%d.bias" % (blk, i)])
        assert np.all(np.abs(dev.cpu().numpy() - ref) <= 1e-12 * (np.abs(X) @ np.abs(Wn["%s.%d.weight" % (blk, i)]).T + 1)), l
    for name, dY, X, cols, _ in wgrad_jobs(st, D):
        dev, _ = gemm_ref(dY.T.contiguous(), X.T.contiguous())
        y, x = dY.cpu().numpy(), X.cpu().numpy()
        assert np.all(np.abs(dev.cpu().numpy() - y.T @ x) <= 1e-12 * (np.abs(y).T @ np.abs(x))), name

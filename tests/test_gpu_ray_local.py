"""Stage-local float64 checks of everything around the MLP: ray setup, sampling, encodings, compositing, the encoding adjoints, the ray
adjoint and its reduction, each from the kernel's OWN inputs.

A seeded render forward (NNB_STASH) and backward runs on the GPU; the workspace stash (records rec = {r, g, b, a, s, z}, the sample
points and encodings enc / denc, the compositing adjoint gs, dy0 / dy4 / dyr, the encoding adjoints gp / gv and the per-ray adjoint
rows rayred) and the outputs are copied to float64, and every stage is rebuilt in float64 from the fp32 values the kernel itself read:
  ray      setup_ray / sample_z / sample_point: the sample point p (enc[:, :3]), z (rec.z and z_vals), the view direction (denc[:, :3]);
  enc      the positional (10 octaves) and direction (4) encodings, sin / cos of the kernel's own p and view direction;
  cfwd     composite_fwd from rec alone: alpha, rgb, depth_pred, depth_gt (and mask, exactly);
  cbwd     composite_bwd: gs from rec and the seeds;
  encadj   gp = encode_bwd<10>(p, dy0 W0 + dy4 W4[:, D:D+63]) and gv = encode_bwd<4>(v, dyr W_rgbh[:, D:D+27]);
  raybwd   ray_bwd: every rayred row and g_depth from the kernel's gp, gv, rec.z, depth_pred and the seeds;
  reduce   ray_reduce: g_c2w, g_cam[0] / g_cam[5], g_scale_shift as sums of the kernel's rayred, added to a non-zero base.

Error model.  Each reference is written as the kernel's sequence of fp32 operations (warp scans as shuffle trees, the chunk carries,
lane-strided sums) on an Arith object: in float64 every rounding point v_k becomes v_k (1 + c_k eps_k), and the scale of an output y is
2^-24 sum_k c_k |dy / d eps_k| at eps = 0 (float64 autograd, one batched backward per output component; rows are independent), plus 2^-126
for underflow.  c_k = 1 for a rounded operation and 2 for sincosf / expf (their ulp bounds).  The encoding adjoints take the GEMM scale of
test_gpu_layer_local.gemm_ref(..., tiny=True) as an absolute error of their input, carried through encode_bwd by the same machinery.
The same code run in plain float32 is an emulation of the kernel; the host tests check that the emulation scores a few units on random and
planted inputs (so the model holds), that every wrong answer below scores at least 10x its gate on the same data, and that the float64
references equal the numpy oracle.  The normalised error is test_gpu_layer_local.nerr: |got - ref| / scale, over finite references;
where a reference is not finite the kernel must give the same non-finite pattern.

Largest normalised errors measured over all cases below on the unmodified kernels (NVIDIA H100 80GB HBM3, 700 W power limit), and the
gates (4x those):
  ray     0.86  (tc, 1024 x 128)  -> 3.5        enc     1.01  (tc, 1024 x 128)  -> 4.1
  cfwd    0.70  (tc, dist-white)  -> 2.8        cbwd    0.70  (tc, dist-white)  -> 2.8
  raybwd  0.94  (tc, eval-nonorm) -> 3.8        reduce  0.34  (tc, 9 x 1023)    -> 1.4
  encadj  73.8  (tc, 1024 x 128)  -> 295        encadj  1.88  (simt, 64 x 15)   -> 7.5
The emulation puts every stage below 1.5.  The tensor-core encoding adjoint is the exception, and it is expected: tc_dgrad runs the
encoding-gradient GEMMs on split-bf16 operands (hi + lo, 16 significant bits; DESIGN.md section 6), whose products carry ~2^-17 relative
error where gemm_ref's scale assumes fp32's 2^-24; the SIMT engine's fp32 GEMMs of the same stash score 1.9.  For the same reason the
wrong answer "W0's bf16 lo half dropped" scores only 700 .. 1300 on the tensor-core engine (12 .. 24x that engine's error in the same
case): there it must exceed the gate, on the SIMT engine 10x the gate.
Wrong answers (each must score at least 10x its gate in every case where it applies, from the same stash): the suffix of composite_bwd
taken as total - prefix in fp32; chunk c's transmittance carry taken from chunk c - 1 (S > 32); eps dropped from om (cases with
near-opaque samples); gsum dropped (white background); df != 0 at the dist_alpha last sample; the encoding argument reduced with the fp32
value of 2 pi; octave L - 1 dropped from encode_bwd; layer 4's encoding slice dropped and W0's bf16 lo half dropped (gp); the normalise
projection - d (d . g_d) dropped; the tau terms of the NDC chain dropped; g_nrm dropped (normalise); the first 32 rays dropped from the
reduction; the prior depth gathered with round-to-nearest instead of floor (cases with a depth map where that picks other cells).  Two
more must exceed the gate, but cannot reach 10x it: eps dropped from om in composite_fwd, and its chunk carry taken from chunk c - 1
(behind near-opaque samples, or with few absorbing samples, they move a ray's colour by ~1e-6 of itself).

Planted in the cases with a depth map: rays whose prior depth is exactly 0 after scale / shift (mask 0), rays whose prior depth is negative
(the sign in g_depth), and a fc_density.bias raised until the densest samples have alpha >= 1 - 1e-7; the transparent case lowers it until
every alpha is at most 2.5e-3."""
import math

import numpy as np
import pytest
import torch

from nope_nerf_b200 import _lib as L
from oracle import nerf_oracle as O
from test_gpu_layer_local import TINY, U, bf16_hi, gemm_ref, nerr
from test_gpu_relu_mask import layout

EPS32 = float(np.float32(O.EPSILON))
TWO_PI_F32 = float(np.float32(2 * math.pi))
STAGES = ("ray", "enc", "cfwd", "cbwd", "encadj", "raybwd", "reduce")
GATES = dict(ray=3.5, enc=4.1, cfwd=2.8, cbwd=2.8, encadj=295.0, raybwd=3.8, reduce=1.4)   # tensor-core engine, see the docstring
SIMT_GATES = dict(GATES, encadj=7.5)
EMU_GATE = 4.0   # largest normalised error of the float32 emulation on the host data (the model is a first-order bound)


# ------------------------------------------------------------------------------------------------------------------ arithmetic
class Arith:
    """the kernel's arithmetic, op by op: float64 with a perturbation eps_k at every fp32 rounding point (track=True), float64 without
    (the exact reference), or plain float32 (the emulation; every torch op on float32 tensors rounds as the kernel's op does)"""

    def __init__(self, f32=False, track=False):
        self.dt = torch.float32 if f32 else torch.float64
        self.track = track and not f32
        self.eps = []

    def t(self, x, dev):
        return torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).to(device=dev, dtype=self.dt)

    def r(self, v, c=1):
        """a rounded result (c = 1) or a libm result with a c-ulp bound"""
        if not self.track:
            return v
        e = torch.zeros(v.shape, dtype=v.dtype, device=v.device, requires_grad=True)
        self.eps.append(e)
        return v + c * v.detach() * e

    def err(self, v, scale):
        """an input that carries an absolute error bound `scale`"""
        if not self.track:
            return v
        e = torch.zeros(v.shape, dtype=v.dtype, device=v.device, requires_grad=True)
        self.eps.append(e)
        return v + (scale / U) * e

    def sin(self, x):
        return self.r(torch.sin(x), 2)

    def cos(self, x):
        return self.r(torch.cos(x), 2)

    def exp(self, x):
        return self.r(torch.exp(x), 2)


def scales(A, y, rows):
    """y [rows, K] built by A (track=True) -> [rows, K]: 2^-24 sum_k c_k |d y / d eps_k| + 2^-126, one batched backward per block of
    components (every eps is indexed by row first, and rows do not interact)"""
    y2 = y.reshape(rows, -1)
    K = y2.shape[1]
    out = torch.zeros(rows, K, dtype=torch.float64, device=y.device)
    eps = A.eps
    assert all(e.shape[:1] == (rows,) or e.shape[:2].numel() == rows for e in eps), "every rounding point must be indexed by row"
    B = max(1, min(K, 64, (1 << (23 if y.is_cuda else 21)) // max(1, y2.numel())))
    for j0 in range(0, K, B):
        j = torch.arange(j0, min(K, j0 + B), device=y.device)
        go = torch.zeros((len(j), rows, K), dtype=y2.dtype, device=y.device)
        go[torch.arange(len(j)), :, j] = 1.0
        gs = torch.autograd.grad(y2, eps, grad_outputs=go, is_grads_batched=True, retain_graph=True, allow_unused=True)
        for g in gs:
            if g is not None:
                out[:, j0:j0 + len(j)] += g.abs().reshape(len(j), rows, -1).sum(2).T
    return U * torch.nan_to_num(out, nan=math.inf) + TINY


def chunks(x, fill):
    """[rows, S] -> [rows, C, 32] (S padded to whole 32-sample chunks with `fill`)"""
    R, S = x.shape
    C = (S + 31) // 32
    return torch.cat([x, x.new_full((R, C * 32 - S), fill)], 1).view(R, C, 32)


def warp_sum(A, v):
    """butterfly sum over the last (32-lane) axis: every lane ends with the total; returns lane 0's"""
    lane = torch.arange(32, device=v.device)
    for o in (16, 8, 4, 2, 1):
        v = A.r(v + v[..., lane ^ o])
    return v[..., 0]


def lane_sum(A, x):
    """sum over the last axis of [rows, n] as a warp does: lane l adds elements l, l + 32, ... in order, then warp_sum"""
    c = chunks(x, 0.0)
    acc = c[:, 0]
    for k in range(1, c.shape[1]):
        acc = A.r(acc + c[:, k])
    return warp_sum(A, acc)


def incl_prod(A, v):
    """warp_incl_prod over the last axis (shuffle tree)"""
    lane = torch.arange(32, device=v.device)
    for o in (1, 2, 4, 8, 16):
        u = torch.cat([torch.ones_like(v[..., :o]), v[..., :-o]], -1)
        v = torch.where(lane >= o, A.r(v * u), v)
    return v


def incl_sum_rev(A, v):
    """warp_incl_sum_rev over the last axis (shuffle tree)"""
    lane = torch.arange(32, device=v.device)
    for o in (1, 2, 4, 8, 16):
        u = torch.cat([v[..., o:], torch.zeros_like(v[..., :o])], -1)
        v = torch.where(lane + o < 32, A.r(v + u), v)
    return v


# ----------------------------------------------------------------------------------------------------------------- references
def setup_ray(A, q, flags, bug=None):
    """setup_ray (nnb_common.cuh) on row-shaped inputs q (every entry already broadcast to the rows of the stage)"""
    r = A.r
    if "x" in q:
        x, y = q["x"], q["y"]
    else:   # arange_pixels at ray_idx: 2 col / (W - 1) - 1
        x = r(r(2.0 * q["col"] / (q["W"] - 1.0)) - 1.0)
        y = r(r(2.0 * q["row"] / (q["H"] - 1.0)) - 1.0)
    kx, ky, R, t = q["kx"], q["ky"], q["R"], q["t"]
    dc = [r(x / kx), r(y / ky), -torch.ones_like(x)]
    dt = [r(r(r(R[3 * i] * dc[0]) + r(R[3 * i + 1] * dc[1])) - R[3 * i + 2]) for i in range(3)]
    nrm = r(torch.sqrt(r(r(r(dt[0] * dt[0]) + r(dt[1] * dt[1])) + r(dt[2] * dt[2]))))
    norm = bool(flags & L.NORMALISE)
    d = [r(v / nrm) for v in dt] if norm else dt
    if "depth" in q:
        raw = depth = q["depth"]
    else:
        raw = q["raw_rint"] if bug == "rint" else q["raw"]
        sc, sf = q["scale"], q["shift"]
        depth = r(r(raw + sf) * sc) if flags & L.SHIFT_FIRST else r(r(raw * sc) + sf)
    g = r(depth.abs() * nrm) if norm else depth.abs()
    out = dict(x=x, y=y, kx=kx, ky=ky, R=R, t=t, dc=dc, dt=dt, nrm=nrm, d=d, raw=raw, depth=depth, g=g)
    if flags & L.NDC:
        tau = r(-r(1.0 + t[2]) / d[2])
        o2 = [r(t[i] + r(tau * d[i])) for i in range(3)]
        ox, oy = r(o2[0] / o2[2]), r(o2[1] / o2[2])
        Oo = [r(-kx * ox), r(-ky * oy), r(1.0 + r(2.0 / o2[2]))]
        Dn = [r(-kx * r(r(d[0] / d[2]) - ox)), r(-ky * r(r(d[1] / d[2]) - oy)), r(1.0 - Oo[2])]
        out.update(tau=tau, o2=o2, ox=ox, oy=oy, O=Oo, Dn=Dn)
    return out


def sample_z(A, i, S, near, far, noise, flags):
    """sample_z: i (float sample index), near / far / noise row-shaped"""
    r = A.r

    def lin01(j):
        step = r(torch.ones_like(j) / (S - 1))
        return torch.where(j < S // 2, r(step * j), r(1.0 - r(step * (S - 1 - j))))

    def zp(j):
        u = lin01(j)
        return u if flags & L.NDC else r(r(near * r(1.0 - u)) + r(far * u))
    z = zp(i)
    if noise is not None and not flags & L.NDC:
        lo = torch.where(i > 0, 0.5 * r(z + zp(i - 1)), z)
        hi = torch.where(i < S - 1, 0.5 * r(zp(i + 1) + z), z)
        z = r(lo + r(r(hi - lo) * noise))
    return z


def ray_stage(A, q, flags, S, noise):
    """per sample (rows [N, S]): (p [N, S, 3], z [N, S], view direction [N, S, 3], ray dict)"""
    ray = setup_ray(A, q, flags)
    i = torch.arange(S, device=ray["x"].device, dtype=A.dt).expand_as(ray["x"])
    z = sample_z(A, i, S, q["near"], q["far"], noise, flags)
    base, dirn = (ray["O"], ray["Dn"]) if flags & L.NDC else (ray["t"], ray["d"])
    p = torch.stack([A.r(base[c] + A.r(dirn[c] * z)) for c in range(3)], -1)
    v = torch.stack([-ray["d"][c] if flags & L.USE_DIR else torch.ones_like(z) for c in range(3)], -1)
    return p, z, v, ray


def encode_ref(x, levels, two_pi=None):
    """encode<L> of the kernel's own fp32 x [M, 3] (2^l x is exact): (value, scale); two_pi: the argument reduced with that value"""
    out, sc = [x], [x.new_zeros(x.shape)]
    for l in range(levels):
        a = (2.0 ** l) * x
        if two_pi is not None:
            a = a - torch.round(a / (2 * math.pi)) * two_pi
        s, c = torch.sin(a), torch.cos(a)
        out += [s, c]; sc += [2 * U * s.abs(), 2 * U * c.abs()]
    return torch.cat(out, 1), torch.cat(sc, 1) + TINY


def transmittance(A, alpha, bug=None):
    """om = 1 - alpha + eps, and T per sample with the chunk carries of composite_fwd / composite_bwd; alpha [N, S]"""
    r = A.r
    om = chunks(r(r(1.0 - alpha) + (0.0 if bug == "no_eps" else EPS32)), 1.0)
    a = om
    incl = incl_prod(A, om)
    excl = torch.cat([torch.ones_like(incl[..., :1]), incl[..., :-1]], -1)
    carries, carry = [], torch.ones_like(a[:, 0, 0])
    for c in range(a.shape[1]):
        carries.append(carry)
        carry = r(carry * incl[:, c, 31])
    if bug == "carry":
        carries = [carries[max(c - 1, 0)] for c in range(len(carries))]
    elif bug == "carry_one":
        carries = [torch.ones_like(carry)] * len(carries)
    T = torch.stack([r(carries[c][:, None] * excl[:, c]) for c in range(a.shape[1])], 1)
    return om, T


def alpha_of(A, rec, flags):
    a, z = rec["a"], rec["z"]
    if not flags & L.DIST_ALPHA:
        return a
    delta = A.r(z[:, 1:] - z[:, :-1])
    al = A.r(1.0 - A.exp(A.r(-a[:, :-1] * delta)))
    return torch.cat([al, torch.ones_like(a[:, -1:])], 1)


def composite_fwd_ref(A, rec, ray, flags, bug=None):
    """composite_fwd from the records: (alpha [N, S], rgb [N, 3], depth_pred [N], depth_gt [N])"""
    r = A.r
    N, S = rec["a"].shape
    alpha = alpha_of(A, rec, flags)
    om, T = transmittance(A, alpha, bug)
    w = r(chunks(alpha, 0.0) * T)
    sums = []
    for v in (rec["r"], rec["g"], rec["b"], rec["z"], None):
        x = w if v is None else r(w * chunks(v, 0.0))
        acc = x[:, 0]
        for c in range(1, x.shape[1]):
            acc = r(acc + x[:, c])
        sums.append(warp_sum(A, acc))
    C, Dist, acc = sums[:3], sums[3], sums[4]
    if flags & L.WHITE_BG:
        bg = r(1.0 - acc)
        C = [r(c + bg) for c in C]
    g = ray["g"]
    if flags & L.EVAL and flags & L.NORMALISE:
        Dist, g = r(Dist / ray["nrm"]), r(g / ray["nrm"])
    if flags & L.NDC:
        g = r(1.0 - r(1.0 / g))
    return alpha, torch.stack(C, 1), Dist, g


def composite_bwd_ref(A, rec, ray, seeds, flags, bug=None, want_suffix=False):
    """composite_bwd: gs [N, S, 4] (and with want_suffix the suffix carry after the first chunk, sum of w gw over the ray); bugs of the
    frame's reverse rounds: suffix_reset (the carry zeroed at every chunk), drop_late (chunks after the first dropped)"""
    r = A.r
    N, S = rec["a"].shape
    gC, gD = seeds["g_rgb"], seeds["g_dp"]
    if flags & L.EVAL and flags & L.NORMALISE:
        gD = r(gD / ray["nrm"])
    gsum = r(r(gC[:, 0] + gC[:, 1]) + gC[:, 2]) if flags & L.WHITE_BG and bug != "no_gsum" else torch.zeros_like(gD)
    alpha = alpha_of(A, rec, flags)
    om, T = transmittance(A, alpha, bug)
    w = r(chunks(alpha, 0.0) * T)
    ch = {k: chunks(rec[k], 0.0) for k in ("r", "g", "b", "z", "a")}
    e = lambda v: v[:, None, None]
    gw = r(r(e(gD) * ch["z"] + r(e(gC[:, 2]) * ch["b"] + r(e(gC[:, 1]) * ch["g"] + r(e(gC[:, 0]) * ch["r"])))) - e(gsum))
    valid = chunks(torch.ones_like(rec["a"]), 0.0) > 0
    if flags & L.DIST_ALPHA:
        z = rec["z"]
        delta = r(z[:, 1:] - z[:, :-1])
        df = r(delta * A.exp(r(-rec["a"][:, :-1] * delta)))
        df = chunks(torch.cat([df, torch.ones_like(z[:, -1:]) if bug == "df_last" else torch.zeros_like(z[:, -1:])], 1), 0.0)
    else:
        df = torch.ones_like(w)
    wg = torch.where(valid, r(w * gw), torch.zeros_like(w))
    if bug == "total_minus_prefix":   # fp32 total minus the inclusive prefix (the emulation's dtype carries the rounding)
        flat = wg.reshape(N, -1)
        suffix = (flat.sum(1, keepdim=True) - torch.cumsum(flat, 1)).view(wg.shape)
        carry_s = flat.sum(1)
    else:
        incl = incl_sum_rev(A, wg)
        excl = torch.cat([incl[..., 1:], torch.zeros_like(incl[..., :1])], -1)
        carry_s, suf = torch.zeros_like(gD), [None] * wg.shape[1]
        for c in range(wg.shape[1] - 1, -1, -1):
            if bug in ("suffix_reset", "drop_late"):
                carry_s = torch.zeros_like(gD)
            suf[c] = r(excl[:, c] + carry_s[:, None])
            carry_s = r(carry_s + incl[:, c, 0])
        suffix = torch.stack(suf, 1)
    g_alpha = r(r(T * gw) - r(suffix / om))
    gs = torch.stack([r(w * e(gC[:, k])) for k in range(3)] + [r(g_alpha * df)], -1)
    if bug == "drop_late":
        gs = torch.cat([gs[:, :1], torch.zeros_like(gs[:, 1:])], 1)
    gs = gs.reshape(N, -1, 4)[:, :S]
    return (gs, carry_s) if want_suffix else gs


def encode_bwd_ref(A, x, ge, levels, bug=None):
    """encode_bwd<L>: x [M, 3] (the kernel's fp32 point or view direction), ge [M, 6 L + 3] -> [M, 3]"""
    r = A.r
    gx = [ge[:, c] for c in range(3)]
    for l in range(levels - 1 if bug == "octave" else levels):
        f = 2.0 ** l
        for c in range(3):
            a = f * x[:, c]
            t = r(r(A.cos(a) * ge[:, 3 + 6 * l + c]) - r(A.sin(a) * ge[:, 6 + 6 * l + c]))
            gx[c] = r(gx[c] + f * t)
    return torch.stack(gx, 1)


def ray_bwd_ref(A, ray, gp, gv, z, depth_pred, seeds, flags, explicit_depth, bug=None):
    """ray_bwd: rows [N]; gp / gv [N, S, 3], z [N, S] -> (rayred [N, 16], g_depth [N])"""
    so = [lane_sum(A, gp[..., c]) for c in range(3)]
    sd = [lane_sum(A, A.r(z * gp[..., c])) for c in range(3)]
    sv = [lane_sum(A, gv[..., c]) for c in range(3)]
    return ray_adjoint_ref(A, ray, so, sd, sv, depth_pred, seeds, flags, explicit_depth, bug)


def ray_adjoint_ref(A, ray, so, sd, sv, depth_pred, seeds, flags, explicit_depth, bug=None):
    """ray_bwd's lane-0 block from its ray sums so = sum gp, sd = sum z gp, sv = sum gv (3 lists of [N]) -> (rayred [N, 16], g_depth)"""
    r = A.r
    norm = bool(flags & L.NORMALISE)
    ev = bool(flags & L.EVAL) and norm
    nrm, d, dt, dc, R = ray["nrm"], ray["d"], ray["dt"], ray["dc"], ray["R"]
    gDo, g_g = seeds["g_dp"], seeds["g_dg"]
    zero = torch.zeros_like(nrm)
    g_nrm = zero
    gcur = r(ray["g"] / nrm) if ev else ray["g"]
    if flags & L.NDC:
        g_g = r(g_g / r(gcur * gcur))
    if ev:
        Dist = r(depth_pred * nrm)
        g_nrm = r(g_nrm - r(r(gDo * Dist) / r(nrm * nrm)))
        g_nrm = r(g_nrm - r(r(g_g * ray["g"]) / r(nrm * nrm)))
        g_g = r(g_g / nrm)
    if norm:
        g_gdepth = r(g_g * nrm)
        g_nrm = r(g_nrm + r(g_g * ray["depth"].abs()))
    else:
        g_gdepth = g_g
    g_depth = g_gdepth * ray.get("depth_sign", torch.sign(ray["depth"].detach()))
    if bug == "no_gnrm":
        g_nrm = zero
    g_kx = g_ky = zero
    if flags & L.NDC:
        kx, ky, o2, ox, oy, tau, t = ray["kx"], ray["ky"], ray["o2"], ray["ox"], ray["oy"], ray["tau"], ray["t"]
        gO, gDn = so, sd
        g_Oz = r(gO[2] - gDn[2])
        g_ox = r(r(-kx * gO[0]) + r(kx * gDn[0]))
        g_oy = r(r(-ky * gO[1]) + r(ky * gDn[1]))
        d22 = r(d[2] * d[2])
        g_d = [r(r(-kx * gDn[0]) / d[2]), r(r(-ky * gDn[1]) / d[2]), r(r(r(r(kx * gDn[0]) * d[0]) + r(r(ky * gDn[1]) * d[1])) / d22)]
        g_kx = r(r(-ox * gO[0]) - r(r(r(d[0] / d[2]) - ox) * gDn[0]))
        g_ky = r(r(-oy * gO[1]) - r(r(r(d[1] / d[2]) - oy) * gDn[1]))
        g_o2 = [r(g_ox / o2[2]), r(g_oy / o2[2]),
                r(r(-r(r(g_ox * ox) + r(g_oy * oy)) / o2[2]) - r(r(2.0 * g_Oz) / r(o2[2] * o2[2])))]
        g_o = list(g_o2)
        if bug != "no_tau":
            g_tau = r(r(r(g_o2[0] * d[0]) + r(g_o2[1] * d[1])) + r(g_o2[2] * d[2]))
            g_d = [r(g_d[c] + r(g_o2[c] * tau)) for c in range(3)]
            g_o[2] = r(g_o[2] + r(-g_tau / d[2]))
            g_d[2] = r(g_d[2] + r(r(g_tau * r(1.0 + t[2])) / d22))
    else:
        g_o, g_d = so, sd
    if flags & L.USE_DIR:
        g_d = [r(g_d[c] - sv[c]) for c in range(3)]
    if norm and bug != "no_proj":
        dot = r(r(r(d[0] * g_d[0]) + r(d[1] * g_d[1])) + r(d[2] * g_d[2]))
        g_dt = [r(r(g_d[c] - r(d[c] * dot)) / nrm) for c in range(3)]
    elif norm:
        g_dt = [r(g_d[c] / nrm) for c in range(3)]
    else:
        g_dt = g_d
    gn = r(g_nrm / nrm)
    g_dt = [r(g_dt[c] + r(gn * dt[c])) for c in range(3)]
    red = [r(g_dt[i] * dc[j]) if j < 2 else -g_dt[i] for i in range(3) for j in range(3)] + list(g_o)
    g_dc0 = r(r(r(g_dt[0] * R[0]) + r(g_dt[1] * R[3])) + r(g_dt[2] * R[6]))
    g_dc1 = r(r(r(g_dt[0] * R[1]) + r(g_dt[1] * R[4])) + r(g_dt[2] * R[7]))
    g_kx = r(g_kx + r(g_dc0 * r(-ray["x"] / r(ray["kx"] * ray["kx"]))))
    g_ky = r(g_ky + r(g_dc1 * r(-ray["y"] / r(ray["ky"] * ray["ky"]))))
    red += [g_kx, g_ky]
    if explicit_depth:
        red += [zero, zero]
    elif flags & L.SHIFT_FIRST:
        red += [r(g_depth * r(ray["raw"] + ray["shift"])), r(g_depth * ray["scale"])]
    else:
        red += [r(g_depth * ray["raw"]), g_depth]
    return torch.stack(red, 1), g_depth


def reduce_ref(A, rayred, base, bug=None):
    """ray_reduce: base [16] + fixed-order sums over the rays of rayred [N, 16] (one warp per column) -> [16]"""
    x = rayred.T
    if bug == "skip32":
        x = x[:, 32:] if x.shape[1] > 32 else torch.zeros_like(x[:, :1])
    return A.r(base + lane_sum(A, x))


# ------------------------------------------------------------------------------------------------------------------ the stages
def _rowq(A, inp, shape, dev):
    """setup_ray inputs broadcast to row shape `shape` ([N] or [N, S]) in A's dtype"""
    N = shape[0]
    ex = lambda v: A.t(v, dev).reshape((N,) + (1,) * (len(shape) - 1)).expand(shape)
    sc = lambda v: A.t(v, dev).reshape((1,) * len(shape)).expand(shape)
    q = dict(kx=sc(inp["cam"][0, 0]), ky=sc(inp["cam"][1, 1]), R=[sc(inp["c2w"][i // 3, i % 3]) for i in range(9)],
             t=[sc(inp["c2w"][i, 3]) for i in range(3)], near=sc(inp["near"]), far=sc(inp["far"]))
    if inp.get("pixels") is not None:
        q["x"], q["y"] = ex(inp["pixels"][:, 0]), ex(inp["pixels"][:, 1])
    else:
        idx = np.asarray(inp["ray_idx"])
        q.update(col=ex(idx % inp["W"]), row=ex(idx // inp["W"]), W=sc(inp["W"]), H=sc(inp["H"]))
    if inp.get("depth") is not None:
        q["depth"] = ex(inp["depth"])
    else:
        q["raw"], q["raw_rint"] = ex(inp["raw"]), ex(inp["raw_rint"])
        q["scale"] = sc(1.0 if inp["scale"] is None else inp["scale"])
        q["shift"] = sc(0.0 if inp["shift"] is None else inp["shift"])
    return q


def _ray_scalars(ray, q):
    ray = dict(ray)
    for k in ("scale", "shift"):
        if k in q:
            ray[k] = q[k]
    return ray


def measure(st, inp, flags, engine, P):
    """every stage's normalised error and the wrong answers' from one stash (st: float64 tensors of the kernel's values)"""
    dev = st["rec"].device
    N, S = inp["N"], inp["S"]
    M = N * S
    out = {s: dict(err=0.0, teeth={}, detect={}) for s in STAGES}

    def check(stage, got, ref, sc):
        fin = torch.isfinite(ref)
        assert torch.equal(torch.isfinite(got), fin), (stage, "non-finite pattern differs")
        if fin.any():
            out[stage]["err"] = max(out[stage]["err"], nerr(got[fin], ref[fin], sc[fin]))

    def tooth(stage, kind, got, wrong, sc):
        fin = torch.isfinite(wrong) & torch.isfinite(got) & torch.isfinite(sc)
        d = (got - wrong).abs()
        v = torch.where(fin, d / sc, torch.zeros_like(d))
        v = float(torch.where(torch.isfinite(got) & ~torch.isfinite(wrong), torch.full_like(v, math.inf), v).max())
        out[stage]["teeth"][kind] = min(out[stage]["teeth"].get(kind, math.inf), v)

    def detect(stage, kind, got, wrong, sc):
        tooth(stage, kind, got, wrong, sc)
        out[stage]["detect"][kind] = out[stage]["teeth"].pop(kind)

    rec = {k: st["rec"][:, i].reshape(N, S) for i, k in enumerate(("r", "g", "b", "a", "s", "z"))}
    A32 = Arith(f32=True)
    rec32 = {k: v.float() for k, v in rec.items()}
    # ---- ray, sampling, point (rows: samples)
    A = Arith(track=True)
    q = _rowq(A, inp, (N, S), dev)
    noise = None if inp.get("noise") is None else A.t(inp["noise"], dev)
    p, z, v, _ = ray_stage(A, q, flags, S, noise)
    y = torch.cat([p, z[..., None], v], -1).reshape(M, 7)
    sc = scales(A, y, M)
    y = y.detach()
    check("ray", st["enc"][:, :3], y[:, :3], sc[:, :3])
    check("ray", rec["z"].reshape(M), y[:, 3], sc[:, 3])
    check("ray", st["z_vals"].reshape(M), y[:, 3], sc[:, 3])
    check("ray", st["denc"][:, :3], y[:, 4:], sc[:, 4:])
    # ---- encodings of the kernel's own point and view direction
    e, esc = encode_ref(st["enc"][:, :3], 10)
    check("enc", st["enc"][:, :63], e, esc)
    tooth("enc", "two_pi_f32", st["enc"][:, :63], encode_ref(st["enc"][:, :3], 10, TWO_PI_F32)[0], esc)
    e, esc = encode_ref(st["denc"][:, :3], 4)
    check("enc", st["denc"][:, :27], e, esc)
    # ---- compositing forward (rows: rays)
    A = Arith(track=True)
    q = _rowq(A, inp, (N,), dev)
    ray = setup_ray(A, q, flags)
    alpha, rgb, dp, dg = composite_fwd_ref(A, rec, ray, flags)
    y = torch.cat([rgb, dp[:, None], dg[:, None], alpha], 1)
    sc = scales(A, y, N)
    y = y.detach()
    check("cfwd", st["rgb"], y[:, :3], sc[:, :3])
    check("cfwd", st["depth_pred"], y[:, 3], sc[:, 3])
    check("cfwd", st["depth_gt"], y[:, 4], sc[:, 4])
    check("cfwd", st["alpha"], y[:, 5:], sc[:, 5:])
    got_f = torch.cat([st["rgb"], st["depth_pred"][:, None], st["depth_gt"][:, None], st["alpha"]], 1)
    # discrete decisions (mask, the sign of the prior depth) are taken on the fp32 values, which the emulation reproduces exactly
    ray32 = setup_ray(A32, _rowq(A32, inp, (N,), dev), flags)
    assert torch.equal(st["mask"] != 0, torch.isfinite(ray32["g"]) & (ray32["g"] != 0)), "mask"
    depth_sign = torch.sign(ray32["depth"]).double()

    def fwd32(bug=None, ray_=ray32):
        a_, c_, d_, g_ = composite_fwd_ref(A32, rec32, ray_, flags, bug)
        return torch.cat([c_, d_[:, None], g_[:, None], a_], 1).double()
    # near-opaque samples that have samples behind them (the dist_alpha last sample is opaque by definition)
    opaque = bool((alpha.detach()[:, :-1] >= 1 - 1e-7).any())
    if opaque:   # a lost eps (as a wrong carry behind transparent samples) moves the forward by ~1e-6 of a ray's colour: it must fail the gate, but cannot reach 10x it
        detect("cfwd", "no_eps", got_f, fwd32("no_eps"), sc)
    if S > 32:
        detect("cfwd", "carry", got_f, fwd32("carry"), sc)
    if "raw" in inp and (inp["raw"] != inp["raw_rint"]).any():
        tooth("cfwd", "rint_gather", got_f, fwd32(ray_=setup_ray(A32, _rowq(A32, inp, (N,), dev), flags, bug="rint")), sc)
    # ---- compositing adjoint (rows: rays)
    seeds = {k: A.t(inp[k], dev) for k in ("g_rgb", "g_dp", "g_dg")}
    A = Arith(track=True)
    ray = setup_ray(A, _rowq(A, inp, (N,), dev), flags)
    gs = composite_bwd_ref(A, rec, ray, seeds, flags)
    sc = scales(A, gs, N).reshape(N, S, 4)
    gs = gs.detach()
    got = st["gs"].reshape(N, S, 4)
    check("cbwd", got, gs, sc)
    seeds32 = {k: v.float() for k, v in seeds.items()}
    bwd32 = lambda bug: composite_bwd_ref(A32, rec32, ray32, seeds32, flags, bug).double()
    if opaque:   # total - prefix cancels only where the suffix is small against the total, i.e. behind a near-opaque sample
        tooth("cbwd", "total_minus_prefix", got, bwd32("total_minus_prefix"), sc)
        tooth("cbwd", "no_eps", got, bwd32("no_eps"), sc)
    if S > 32:
        tooth("cbwd", "carry", got, bwd32("carry"), sc)
    if flags & L.WHITE_BG and not flags & L.DIST_ALPHA:   # with dist_alpha the last sample is opaque and the background adds nothing
        tooth("cbwd", "no_gsum", got, bwd32("no_gsum"), sc)
    if flags & L.DIST_ALPHA:
        tooth("cbwd", "df_last", got, bwd32("df_last"), sc)
    # ---- encoding adjoints (rows: samples)
    D = P["fc_feature.weight"].shape[0]
    W0, W4 = P["layers0.0.weight"], P["layers1.0.weight"][:, D:D + 63]
    Wd = P["rgb_layers.0.weight"][:, D:D + 27]
    ge, gsc = gemm_ref(torch.cat([st["dy0"], st["dy4"]], 1), torch.cat([W0, W4], 0).T.contiguous(), tiny=True)
    A = Arith(track=True)
    gp = encode_bwd_ref(A, st["enc"][:, :3], A.err(ge, gsc), 10)
    sc = scales(A, gp, M)
    check("encadj", st["gp"][:, :3], gp.detach(), sc)
    A64 = Arith()
    p64 = st["enc"][:, :3]
    tooth("encadj", "octave", st["gp"][:, :3], encode_bwd_ref(A64, p64, ge, 10, "octave"), sc)
    tooth("encadj", "no_layer4", st["gp"][:, :3], encode_bwd_ref(A64, p64, st["dy0"] @ W0, 10), sc)
    (tooth if engine == "simt" else detect)("encadj", "w0_lo", st["gp"][:, :3],
                                            encode_bwd_ref(A64, p64, st["dy0"] @ bf16_hi(W0) + st["dy4"] @ W4, 10), sc)
    gev, gvsc = gemm_ref(st["dyr"], Wd.T.contiguous(), tiny=True)
    A = Arith(track=True)
    gv = encode_bwd_ref(A, st["denc"][:, :3], A.err(gev, gvsc), 4)
    sc = scales(A, gv, M)
    check("encadj", st["gv"][:, :3], gv.detach(), sc)
    tooth("encadj", "octave", st["gv"][:, :3], encode_bwd_ref(A64, st["denc"][:, :3], gev, 4, "octave"), sc)
    # ---- ray adjoint (rows: rays)
    explicit = inp.get("depth") is not None
    A = Arith(track=True)
    q = _rowq(A, inp, (N,), dev)
    ray = dict(_ray_scalars(setup_ray(A, q, flags), q), depth_sign=depth_sign)
    gpr, gvr = st["gp"][:, :3].reshape(N, S, 3), st["gv"][:, :3].reshape(N, S, 3)
    red, gdep = ray_bwd_ref(A, ray, gpr, gvr, rec["z"], st["depth_pred"], seeds, flags, explicit)
    y = torch.cat([red, gdep[:, None]], 1)
    sc = scales(A, y, N)
    y = y.detach()
    got = torch.cat([st["rayred"], st["g_depth"][:, None]], 1)
    check("raybwd", got, y, sc)
    for bug, applies in (("no_proj", flags & L.NORMALISE), ("no_tau", flags & L.NDC), ("no_gnrm", flags & L.NORMALISE)):
        if applies:
            q64 = _rowq(A64, inp, (N,), dev)
            ray64 = dict(_ray_scalars(setup_ray(A64, q64, flags), q64), depth_sign=depth_sign)
            w, wd = ray_bwd_ref(A64, ray64, gpr, gvr, rec["z"], st["depth_pred"], seeds, flags, explicit, bug)
            tooth("raybwd", bug, got, torch.cat([w, wd[:, None]], 1), sc)
    # ---- reduction (rows: the 16 rayred columns)
    A = Arith(track=True)
    base = A.t(inp["base"], dev)
    tot = reduce_ref(A, st["rayred"], base)
    sc = scales(A, tot[:, None], 16)[:, 0]
    tot = tot.detach()
    got = st["red_out"]
    have = torch.tensor(inp["red_written"], device=dev)
    check("reduce", got[have], tot[have], sc[have])
    tooth("reduce", "skip32", got[have], reduce_ref(A64, st["rayred"], base, "skip32")[have], sc[have])
    return out


# ---------------------------------------------------------------------------------------------------------------------- GPU run
def _flags(c):
    cfg = dict(O.DEFAULT_CFG)
    cfg.update(dist_alpha=c.get("dist_alpha", False), white_background=c.get("white_bg", False),
               sample_option="ndc" if c.get("ndc") else "uniform", normalise_ray=c.get("normalise", True))
    from nope_nerf_b200 import ops
    return ops.flags_from_cfg(cfg, "softplus", eval_=c.get("eval", False), shift_first=c.get("shift_first", False))


def _zero_raw(sc, sf, flags):
    """an fp32 raw prior depth whose distorted depth is exactly 0 (scale / shift in fp32)"""
    f = np.float32
    x0 = f(-sf) if flags & L.SHIFT_FIRST else f(-sf / sc)
    cand = [x0]
    for _ in range(64):
        cand += [np.nextafter(cand[-2] if len(cand) > 1 else x0, f(np.inf)), np.nextafter(cand[-1], f(-np.inf))]
    for x in cand:
        x = f(x)
        v = f(f(x + f(sf)) * f(sc)) if flags & L.SHIFT_FIRST else f(f(x * f(sc)) + f(sf))
        if v == 0:
            return x
    raise AssertionError("no fp32 raw depth maps to exactly 0")


def _logit_target(c, flags):
    """the largest density logit a case plants: near-opaque (alpha >= 1 - 1e-7: softplus >= 16.2; with dist_alpha sigma delta >= 16.2
    at sample spacings down to 0.08), or transparent (every alpha <= 2.5e-3)"""
    if "target" in c:
        return c["target"]
    if c.get("plant"):
        return 200.0 if flags & L.DIST_ALPHA else 17.0
    return None


CASES = {
    "default": dict(engine="tc", N=1024, S=128, plant=True),
    "default-301x17": dict(engine="tc", N=301, S=17, plant=True),
    "simt-301x17": dict(engine="simt", N=301, S=17, plant=True),
    "s32": dict(engine="tc", N=40, S=32),
    "s33": dict(engine="tc", N=40, S=33),
    "s1023": dict(engine="tc", N=9, S=1023),
    "s1024": dict(engine="tc", N=9, S=1024),
    "simt-s2": dict(engine="simt", N=64, S=2),
    "simt-s15": dict(engine="simt", N=64, S=15),
    "dist-white": dict(engine="tc", N=301, S=64, dist_alpha=True, white_bg=True, plant=True),
    "white": dict(engine="tc", N=301, S=64, white_bg=True, plant=True),
    "ndc": dict(engine="tc", N=301, S=64, ndc=True, dist_alpha=True, noise=False),
    "eval": dict(engine="tc", N=301, S=64, eval=True, plant=True),
    "eval-nonorm": dict(engine="tc", N=301, S=64, eval=True, normalise=False),
    "shift-first": dict(engine="tc", N=301, S=64, shift_first=True, plant=True),
    "no-scale-shift": dict(engine="tc", N=301, S=64, shift_first=True, scale=None, shift=None, plant=True, g_cam=False, g_ss=False),
    "explicit": dict(engine="tc", N=301, S=64, explicit=True),
    "transparent": dict(engine="tc", N=301, S=64, target=-6.0),
}


def run(name, P=None, D=256):
    """forward + backward of one case; returns (stash dict of float64 tensors, inputs dict, flags, params)"""
    from nope_nerf_b200 import ops
    c = CASES[name]
    N, S = c["N"], c["S"]
    flags = _flags(c)
    rng = np.random.default_rng(23)
    H, W = 48, 64
    cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    P = dict(O.init_params(seed=5, D=D)) if P is None else P
    r_, t_ = rng.normal(0, .05, (2, 3)).astype(np.float32), rng.normal(0, .05, (2, 3)).astype(np.float32)
    c2w = torch.empty(4, 4, device="cuda"); ops.pose_fwd_raw(cu(r_), cu(t_), None, 1, c2w)   # camera 1 of two
    assert torch.isfinite(c2w).all()
    cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0])).cuda()
    ray_idx = rng.permutation(H * W)[:N]
    dmap = rng.uniform(.6, 7.2, (24, 32)).astype(np.float32)
    noise = rng.uniform(0, 1, (N, S)).astype(np.float32)
    scale = c.get("scale", np.float32(1.05)); shift = c.get("shift", np.float32(0.02))
    inp = dict(N=N, S=S, H=H, W=W, near=np.float32(0.01), far=np.float32(10.0), noise=None if c.get("noise") is False else noise)
    if c.get("plant"):
        _, cell = O.gather_prior_depth(dmap, ray_idx, H, W)
        zr = _zero_raw(1.0 if scale is None else scale, 0.0 if shift is None else shift, flags)
        dmap.reshape(-1)[cell[:3]] = zr
        dmap.reshape(-1)[cell[3:6]] = -0.7
    kw = {}
    if c.get("explicit"):
        pix = O.pixels_from_idx(ray_idx, H, W)
        pix = pix + rng.uniform(-.01, .01, pix.shape).astype(np.float32)
        dep = rng.uniform(.5, 6, N).astype(np.float32); dep[:3] = 0; dep[3:6] *= -1
        kw = dict(pixels=cu(pix), depth=cu(dep))
        inp.update(pixels=pix.astype(np.float64), depth=dep.astype(np.float64))
    else:
        kw = dict(ray_idx=cu(ray_idx), depth_map=cu(dmap), scale=None if scale is None else torch.tensor([scale]).cuda(),
                  shift=None if shift is None else torch.tensor([shift]).cuda())
        raw, _ = O.gather_prior_depth(dmap, ray_idx, H, W)
        row, col = ray_idx // W, ray_idx % W
        sr = np.minimum(np.rint(row.astype(np.float32) * np.float32(24 / H)).astype(np.int64), 23)
        scc = np.minimum(np.rint(col.astype(np.float32) * np.float32(32 / W)).astype(np.int64), 31)
        inp.update(ray_idx=ray_idx, raw=raw.astype(np.float64), raw_rint=dmap[sr, scc].astype(np.float64), scale=scale, shift=shift)
    target = _logit_target(c, flags)
    lay = layout(N, S, D)
    call_kw = dict(N=N, S=S, flags=flags, engine=L.ENGINE_TC if c["engine"] == "tc" else L.ENGINE_SIMT, near=0.01, far=10.0,
                   noise=None if inp["noise"] is None else cu(noise), H=H, W=W, want_z_alpha=True, stash=True, hidden_dim=D, **kw)
    if target is not None:
        # the logits s = h7 . w + b of a first run; then (plant) w scaled by k and b moved so that the largest logit is the target and
        # the 90th percentile -3 (a few near-opaque samples, many transparent ones), or (transparent) b moved alone
        probe = ops.RenderCall(cu(O.flatten_params(P)), c2w, cam, **call_kw)
        s0 = probe.ws[lay["rec"]:lay["rec"] + N * S * 32].view(torch.float32).view(N * S, 8)[:, 4].double()
        probe.release()
        m = s0 - float(P["fc_density.bias"][0])
        k = (target + 3.0) / float(m.max() - torch.quantile(m, 0.9)) if c.get("plant") else 1.0
        P["fc_density.weight"] = (P["fc_density.weight"] * np.float32(k)).astype(np.float32)
        P["fc_density.bias"] = np.full_like(P["fc_density.bias"], target - k * float(m.max()))
    call = ops.RenderCall(cu(O.flatten_params(P)), c2w, cam, **call_kw)
    g_rgb = rng.normal(0, 1, (N, 3)).astype(np.float32)
    g_dp = rng.normal(0, 1, N).astype(np.float32); g_dg = rng.normal(0, 1, N).astype(np.float32)
    base = rng.normal(0, 1, 24).astype(np.float32)
    g_c2w = cu(base[:16].reshape(4, 4)); g_cam = cu(base[:16].reshape(4, 4)[::-1]); g_ss = cu(base[16:18])
    g_cam0, g_ss0 = g_cam.clone(), g_ss.clone()
    g_w = torch.zeros(L.num_params(D), device="cuda")
    g_depth = torch.full((N,), float("nan"), device="cuda")
    use_cam, use_ss = c.get("g_cam", True), c.get("g_ss", True)
    ws = call.ws   # the backward hands the workspace back to the pool; it stays alive, and nothing takes it before the copies below
    call.backward(cu(g_rgb), cu(g_dp), cu(g_dg), g_w, g_c2w, g_cam if use_cam else None, g_depth, g_ss if use_ss else None)
    torch.cuda.synchronize()
    Mp, M = lay["Mpad"], N * S
    f = lambda off, rows, cols: ws[off:off + rows * cols * 4].view(torch.float32).view(rows, cols)[:min(rows, M)].double().clone()
    st = dict(rec=f(lay["rec"], Mp, 8), enc=f(lay["enc"], Mp, 64), denc=f(lay["denc"], Mp, 32), gs=f(lay["gs"], Mp, 4),
              gp=f(lay["gp"], Mp, 4), gv=f(lay["gv"], Mp, 4), dy0=f(lay["dy"][0], Mp, D), dy4=f(lay["dy"][4], Mp, D),
              dyr=f(lay["dyr"], Mp, D // 2), rayred=f(lay["rayred"], N, 16))
    st.update(rgb=call.rgb.double(), depth_pred=call.depth_pred.double(), depth_gt=call.depth_gt.double(), mask=call.mask.clone(),
              z_vals=call.z_vals.double(), alpha=call.alpha.double(), g_depth=g_depth.double())
    # the reduction's 16 outputs: g_c2w rows 0..2 (R then t), g_cam[0] / g_cam[5], g_scale_shift
    gc = g_c2w.double()
    red_out = [gc[i // 3, i % 3] for i in range(9)] + [gc[i, 3] for i in range(3)]
    red_out += [g_cam.double().view(-1)[0], g_cam.double().view(-1)[5]] + [g_ss.double()[0], g_ss.double()[1]]
    st["red_out"] = torch.stack(red_out)
    bc, bk, bs = base[:16].reshape(4, 4).astype(np.float64), base[:16].reshape(4, 4)[::-1].reshape(-1).astype(np.float64), base[16:18]
    inp["base"] = np.concatenate([[bc[i // 3, i % 3] for i in range(9)], bc[:3, 3], [bk[0], bk[5]], bs.astype(np.float64)])
    written = [True] * 12 + [use_cam] * 2 + [use_ss and not c.get("explicit")] * 2
    inp["red_written"] = written
    # what the backward must leave alone: g_c2w row 3, g_cam outside [0] / [5], g_scale_shift with explicit depth
    assert torch.equal(g_c2w[3].cpu(), torch.from_numpy(base[12:16])), "g_c2w row 3 was written"
    keep = torch.ones(16, dtype=torch.bool); keep[[0, 5]] = False
    assert torch.equal(g_cam.view(-1)[keep], g_cam0.view(-1)[keep]), "g_cam written outside [0] / [5]"
    if not use_cam:
        assert torch.equal(g_cam, g_cam0)
    if not use_ss or c.get("explicit"):
        assert torch.equal(g_ss, g_ss0), "g_scale_shift was written"
    inp.update(c2w=c2w.double().cpu().numpy(), cam=cam.double().cpu().numpy(), g_rgb=g_rgb.astype(np.float64),
               g_dp=g_dp.astype(np.float64), g_dg=g_dg.astype(np.float64))
    Pd = {k: torch.from_numpy(np.asarray(v, np.float64)).cuda() for k, v in P.items()}
    return st, inp, flags, Pd


def _check(key, out, gates):
    for stage, gate in gates.items():
        r = out[stage]
        assert r["err"] <= gate, (key, stage, r["err"], gate)
        for kind, t in r["teeth"].items():
            assert t >= 10 * gate, (key, stage, "wrong answer '%s' within 10x of the gate" % kind, t, gate)
        for kind, t in r["detect"].items():
            assert t >= gate, (key, stage, "wrong answer '%s' within the gate" % kind, t, gate)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_ray_local(name):
    st, inp, flags, P = run(name)
    out = measure(st, inp, flags, CASES[name]["engine"], P)
    _check(name, out, SIMT_GATES if CASES[name]["engine"] == "simt" else GATES)


# ------------------------------------------------------------------------------------------------------------------------- host
def emulate(name, N=37, S=40, D=64, seed=3):
    """a stash as the kernels would leave it, from the float32 emulation of every stage (CPU): the same inputs as run(), random MLP
    outputs (logits ~ N(0, 3), near-opaque and transparent samples planted) and random dy0 / dy4 / dyr with some exact zeros"""
    c = CASES[name]
    S = c["S"] if c["S"] < 32 or c["S"] in (32, 33) else S
    flags = _flags(c)
    rng = np.random.default_rng(seed)
    H, W = 48, 64
    A = Arith(f32=True)
    dev = "cpu"
    inp = dict(N=N, S=S, H=H, W=W, near=np.float32(0.01), far=np.float32(10.0),
               noise=None if c.get("noise") is False else rng.uniform(0, 1, (N, S)).astype(np.float32))
    r_, t_ = rng.normal(0, .05, 3), rng.normal(0, .05, 3).astype(np.float32)
    c2w = np.eye(4, dtype=np.float32); c2w[:3, :3] = O.exp_so3(r_).astype(np.float32); c2w[:3, 3] = t_
    inp.update(c2w=c2w.astype(np.float64), cam=np.diag([1.2, -1.6, -1.0, 1.0]).astype(np.float32).astype(np.float64))
    ray_idx = rng.permutation(H * W)[:N]
    scale = c.get("scale", np.float32(1.05)); shift = c.get("shift", np.float32(0.02))
    if c.get("explicit"):
        pix = O.pixels_from_idx(ray_idx, H, W) + rng.uniform(-.01, .01, (N, 2)).astype(np.float32)
        dep = rng.uniform(.5, 6, N).astype(np.float32); dep[:3] = 0; dep[3:6] *= -1
        inp.update(pixels=pix.astype(np.float64), depth=dep.astype(np.float64))
    else:
        dmap = rng.uniform(.6, 7.2, (24, 32)).astype(np.float32)
        if c.get("plant"):
            _, cell = O.gather_prior_depth(dmap, ray_idx, H, W)
            dmap.reshape(-1)[cell[:3]] = _zero_raw(1.0 if scale is None else scale, 0.0 if shift is None else shift, flags)
            dmap.reshape(-1)[cell[3:6]] = -0.7
        raw, _ = O.gather_prior_depth(dmap, ray_idx, H, W)
        row, col = ray_idx // W, ray_idx % W
        sr = np.minimum(np.rint(row.astype(np.float32) * np.float32(0.5)).astype(np.int64), 23)
        scc = np.minimum(np.rint(col.astype(np.float32) * np.float32(0.5)).astype(np.int64), 31)
        inp.update(ray_idx=ray_idx, raw=raw.astype(np.float64), raw_rint=dmap[sr, scc].astype(np.float64), scale=scale, shift=shift)
    noise = None if inp["noise"] is None else A.t(inp["noise"], dev)
    p, z, v, _ = ray_stage(A, _rowq(A, inp, (N, S), dev), flags, S, noise)
    M = N * S
    p, z, v = p.reshape(M, 3), z.reshape(M), v.reshape(M, 3)
    enc = torch.cat([p] + [f(float(2 ** l) * p) for l in range(10) for f in (torch.sin, torch.cos)], 1)
    enc = torch.cat([enc[:, :3]] + [enc[:, 3 + 6 * l:9 + 6 * l] for l in range(10)], 1)
    denc = torch.cat([v] + [f(float(2 ** l) * v) for l in range(4) for f in (torch.sin, torch.cos)], 1)
    s = torch.from_numpy(rng.normal(0, 3, M).astype(np.float32))
    target = _logit_target(c, flags)
    if c.get("plant"):
        s[rng.choice(M, M // 50, replace=False)] = target
    elif target is not None:
        s = s + float(target - s.max())
    sig = torch.where(s > 20, s, torch.log1p(torch.exp(s)))
    a = sig if flags & L.DIST_ALPHA else 1.0 - torch.exp(-sig)
    col3 = torch.sigmoid(torch.from_numpy(rng.normal(0, 1, (M, 3)).astype(np.float32)))
    rec = torch.cat([col3, a[:, None], s[:, None], z[:, None], torch.zeros(M, 2)], 1)
    recd = {k: rec[:, i].reshape(N, S) for i, k in enumerate(("r", "g", "b", "a", "s", "z"))}
    q = _rowq(A, inp, (N,), dev)
    ray = _ray_scalars(setup_ray(A, q, flags), q)
    alpha, rgb, dp, dg = composite_fwd_ref(A, recd, ray, flags)
    inp.update(g_rgb=rng.normal(0, 1, (N, 3)), g_dp=rng.normal(0, 1, N), g_dg=rng.normal(0, 1, N))
    for k in ("g_rgb", "g_dp", "g_dg"):
        inp[k] = inp[k].astype(np.float32).astype(np.float64)
    seeds = {k: A.t(inp[k], dev) for k in ("g_rgb", "g_dp", "g_dg")}
    gs = composite_bwd_ref(A, recd, ray, seeds, flags).reshape(M, 4)
    P = {k: torch.from_numpy(np.asarray(v_, np.float32)) for k, v_ in O.init_params(seed=5, D=D).items()}
    dyz = lambda shape: torch.from_numpy((rng.normal(0, 1e-3, shape) * (rng.uniform(0, 1, shape) < 0.6)).astype(np.float32))
    dy0, dy4, dyr = dyz((M, D)), dyz((M, D)), dyz((M, D // 2))
    ge = dy0 @ P["layers0.0.weight"] + dy4 @ P["layers1.0.weight"][:, D:D + 63]
    gp = encode_bwd_ref(A, p, ge, 10)
    gv = encode_bwd_ref(A, v, dyr @ P["rgb_layers.0.weight"][:, D:D + 27], 4)
    red, gdep = ray_bwd_ref(A, ray, gp.reshape(N, S, 3), gv.reshape(N, S, 3), recd["z"], dp, seeds, flags, c.get("explicit", False))
    base = rng.normal(0, 1, 16).astype(np.float32)
    inp["base"] = base.astype(np.float64)
    use_cam, use_ss = c.get("g_cam", True), c.get("g_ss", True)
    inp["red_written"] = [True] * 12 + [use_cam] * 2 + [use_ss and not c.get("explicit")] * 2
    tot = reduce_ref(A, red, A.t(base, dev))
    pad = lambda x: torch.cat([x, torch.zeros(M, 1)], 1)
    st = dict(rec=rec, enc=pad(enc), denc=torch.cat([denc, torch.zeros(M, 5)], 1), gs=gs, gp=pad(gp), gv=pad(gv), dy0=dy0, dy4=dy4,
              dyr=dyr, rayred=red, rgb=rgb, depth_pred=dp, depth_gt=dg, z_vals=z.reshape(N, S), alpha=alpha, g_depth=gdep,
              red_out=tot, mask=(torch.isfinite(ray["g"]) & (ray["g"] != 0)).to(torch.uint8))
    st = {k: (v_ if k == "mask" else v_.double()) for k, v_ in st.items()}
    return st, inp, flags, {k: v_.double() for k, v_ in P.items()}


HOST_CASES = ["default", "simt-s2", "simt-s15", "s32", "s33", "dist-white", "white", "ndc", "eval", "eval-nonorm", "shift-first",
              "no-scale-shift", "explicit", "transparent"]


@pytest.mark.parametrize("name", HOST_CASES)
def test_emulation_within_model(name):
    """the float32 emulation of every stage scores a few units against its float64 reference and first-order scale, and every
    wrong answer scores at least 10x the stage's gate on the same data"""
    st, inp, flags, P = emulate(name)
    out = measure(st, inp, flags, CASES[name]["engine"], P)
    print(name, {s: round(out[s]["err"], 2) for s in STAGES})
    print(name, "teeth / gate", {(s, k): "%.3g" % (t / (SIMT_GATES if CASES[name]["engine"] == "simt" else GATES)[s])
                                 for s in STAGES for k, t in out[s]["teeth"].items()})
    for s in STAGES:
        if s != "encadj":   # the emulated GEMM is fp32 at any K order: scored against gemm_ref's scale, as the kernels are
            assert out[s]["err"] <= EMU_GATE, (name, s, out[s]["err"])
    assert out["encadj"]["err"] <= 4 * EMU_GATE, (name, out["encadj"]["err"])
    gates = SIMT_GATES if CASES[name]["engine"] == "simt" else GATES
    for s in STAGES:
        for kind, t in out[s]["teeth"].items():
            assert t >= 10 * gates[s], (name, s, kind, t, gates[s])
        for kind, t in out[s]["detect"].items():
            assert t >= gates[s], (name, s, kind, t, gates[s])
    expect = {("enc", "two_pi_f32"), ("encadj", "octave"), ("encadj", "no_layer4"),
              ("encadj", "w0_lo"), ("reduce", "skip32")}
    if CASES[name].get("plant"):
        expect |= {("cfwd", "no_eps"), ("cbwd", "no_eps"), ("cbwd", "total_minus_prefix")}
    if inp["S"] > 32:
        expect |= {("cfwd", "carry"), ("cbwd", "carry")}
    if flags & L.WHITE_BG and not flags & L.DIST_ALPHA:
        expect.add(("cbwd", "no_gsum"))
    if flags & L.DIST_ALPHA:
        expect.add(("cbwd", "df_last"))
    if flags & L.NORMALISE:
        expect |= {("raybwd", "no_proj"), ("raybwd", "no_gnrm")}
    if flags & L.NDC:
        expect.add(("raybwd", "no_tau"))
    if "raw" in inp and (inp["raw"] != inp["raw_rint"]).any():
        expect.add(("cfwd", "rint_gather"))
    have = {(s, k) for s in STAGES for k in list(out[s]["teeth"]) + list(out[s]["detect"])}
    assert expect <= have, (name, expect - have)


@pytest.mark.parametrize("ndc", (False, True))
def test_references_match_oracle(ndc):
    """the float64 references (device-agnostic torch) equal the numpy oracle's encode_position(_bwd) and render_forward /
    render_backward on one small case, to 1e-12 relative"""
    N, S, D = 5, 40, 64
    rng = np.random.default_rng(1)
    cfg = dict(O.DEFAULT_CFG, num_points=S, white_background=ndc, dist_alpha=ndc, sample_option="ndc" if ndc else "uniform")
    flags = _flags(dict(ndc=ndc, dist_alpha=ndc, white_bg=ndc, eval=ndc))
    P = O.init_params(seed=5, D=D, dtype=np.float64)
    c2w = O.make_c2w(rng.normal(0, .05, 3), rng.normal(0, .05, 3))
    pix = rng.uniform(-1, 1, (N, 2)); dep = rng.uniform(.5, 6, N); dep[1] *= -1
    noise = None if ndc else rng.uniform(0, 1, (N, S))
    kx, ky = 1.2, -1.6
    out, cache = O.render_forward(P, pix, dep, c2w, kx, ky, cfg, noise=noise, eval_=ndc)
    g_rgb, g_dp, g_dg = rng.normal(0, 1, (N, 3)), rng.normal(0, 1, N), rng.normal(0, 1, N)
    ref = O.render_backward(P, cache, g_rgb, g_dp, g_dg)
    close = lambda a, b: np.abs(np.asarray(a) - b).max() <= 1e-12 * max(np.abs(b).max(), 1e-300)
    A = Arith()
    inp = dict(N=N, S=S, near=0.01, far=10.0, pixels=pix, depth=dep, c2w=c2w, cam=np.diag([kx, ky, -1.0, 1.0]))
    p, z, v, _ = ray_stage(A, _rowq(A, inp, (N, S), "cpu"), flags, S, None if noise is None else torch.from_numpy(noise))
    assert close(p.numpy().reshape(-1, 3), cache["mcache"]["pts"]) and close(z.numpy(), cache["z"])
    assert close(v.numpy().reshape(-1, 3), cache["mcache"]["dirs"])
    e, _ = encode_ref(p.reshape(-1, 3), 10)
    assert close(e.numpy(), O.encode_position(cache["mcache"]["pts"], 10))
    g = rng.normal(0, 1, (N * S, 63))
    assert close(encode_bwd_ref(A, p.reshape(-1, 3), torch.from_numpy(g), 10).numpy(), O.encode_position_bwd(cache["mcache"]["pts"], 10, g))
    rec = dict(r=torch.from_numpy(cache["rgb_s"][..., 0]), g=torch.from_numpy(cache["rgb_s"][..., 1]),
               b=torch.from_numpy(cache["rgb_s"][..., 2]), a=torch.from_numpy(cache["a_s"]), z=torch.from_numpy(cache["z"]))
    q = _rowq(A, inp, (N,), "cpu")
    ray = _ray_scalars(setup_ray(A, q, flags), q)
    alpha, rgb, dp, dg = composite_fwd_ref(A, rec, ray, flags)
    assert close(alpha.numpy(), out["alpha"]) and close(rgb.numpy(), out["rgb"])
    assert close(dp.numpy(), out["depth_pred_full"]) and close(dg.numpy(), out["depth_gt_full"])
    seeds = dict(g_rgb=torch.from_numpy(g_rgb), g_dp=torch.from_numpy(g_dp), g_dg=torch.from_numpy(g_dg))
    gs = composite_bwd_ref(A, rec, ray, seeds, flags).numpy()
    _, g_pts, g_dirs = O.mlp_backward(P, cache["mcache"], gs[..., :3].reshape(-1, 3), gs[..., 3].reshape(-1))
    red, gdep = ray_bwd_ref(A, ray, torch.from_numpy(g_pts.reshape(N, S, 3)), torch.from_numpy(g_dirs.reshape(N, S, 3)), rec["z"], dp,
                            seeds, flags, True)
    tot = reduce_ref(A, red, torch.zeros(16, dtype=torch.float64)).numpy()
    assert close(tot[:9].reshape(3, 3), ref["c2w"][:3, :3]) and close(tot[9:12], ref["c2w"][:3, 3])
    assert close(tot[12:14], ref["kxy"]) and close(gdep.numpy(), ref["depth"])

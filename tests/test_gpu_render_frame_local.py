"""GPU: the differentiable frame's reverse rounds against float64, on fields that stay translucent through every 32-sample chunk.

The frame backward (ops.render_frame_bwd, and the training pair ops.FrameRenderCall / ops.ExactFrameRenderCall with jitter) runs rounds
k = C - 1 .. 0 over the chunks of every ray, from per-chunk transmittance checkpoints written by the forward and a suffix carry handed from
round to round.  The seeded fields of the other frame tests are opaque within the first chunk, where none of that carries weight; the
fields here are planted from a probe run's density logits (fc_density of O.init_params(hf_damp=True)):
  translucent  fc_density.bias moved alone, so that the float64 transmittance into the last chunk is at least 0.05 on every ray;
  scattered    fc_density.weight scaled and the bias moved (test_gpu_ray_local's plant), so that a few samples are near-opaque and rays
               lose their transmittance in different rounds (the chunk where it first drops below 1e-3 takes at least 4 values).
Every case asserts its own coverage.

(1) end to end: rgb, depth_pred, depth_gt, every dW / db, g_c2w, g_cam[0] / [5], g_scale_shift and g_depth against float64 autograd of the
whole render from the call's inputs (test_gpu_ray_local's ray, sampling and compositing references, the MLP in torch), with the ReLU gates
the engine itself took (nnb_render_fwd with NNB_STASH on the same inputs: the tensor-core gate bits, the exact engine's h > 0), so that
no fp32-vs-float64 gate flip enters.  The frame's chunk stash is first checked to hold the stash path's rows of chunk 0 bit for bit.
Error: per tensor |got - ref|max / |ref|max.
(2) stage-local, from the training pair's workspace after the call, with test_gpu_ray_local's error model (Arith / scales / nerr) on the
stash path's records of the same inputs:
  ckpt     ckpt[k][n], k < C - 1, against the float64 transmittance carry;
  suffix   suffix[n] after the last round (the sum of w gw over the ray);
  cbwd0    chunk 0's gs rows of the chunk stash against composite_bwd_ref; their suffix comes in from chunks C - 1 .. 1;
  rayacc   the lane partials raypart[N][9][32] of frame_ray_acc against their sums over the rounds of the samples' gp, gv and z;
  rayfin   rayred[N][16] (and g_depth) of frame_ray_finish against ray_bwd's adjoint (ray_adjoint_ref) of the warp sums of the kernel's
           own raypart;
  reduce   g_c2w, g_cam[0] / [5] and g_scale_shift against reduce_ref of the kernel's rayred;
  layers0  test_gpu_layer_local's forward and data-gradient checks on chunk 0's rows of the chunk stash (the frame's stash and
           data-gradient modes).
(3) early termination: render_frame_engine(t_min > 0, want_stats=True) on a scattered field stops every ray at the chunk where the
float64 carry first drops below t_min (rays within 1e-3 of it at some checkpoint are left out), with t_final the training forward's
checkpoint bits; rays that never stop keep the t_min = 0 bits.  The rays stop in at least 4 different rounds.

Wrong answers, each evaluated in float64 from the same data (the composite adjoint replaced by test_gpu_ray_local.composite_bwd_ref with
the bug, pulled back through the same autograd graph; the ray adjoint through ray_bwd_ref / reduce_ref): rounds k >= 1 dropped;
round k with the checkpoint of chunk k - 1, and with 1; the suffix carry reset every round; dist_alpha's df != 0 at the last sample;
frame_ray_acc with z of the previous chunk, and with the last round's partial added twice; the reduction without its first 32 rays.
On translucent fields each scores at least 10x its gate (rounds dropped: on every non-zero dW tensor); elsewhere it must exceed the gate.
The stage-local wrong answers are scored as test_gpu_ray_local scores them (float32 emulation); the suffix formed as total - prefix
in fp32 must only exceed the cbwd0 gate.

Largest errors measured on the unmodified kernels (NVIDIA H100 80GB HBM3, 700 W power limit), and the gates (at most 4x those):
  end to end, translucent   tc 4.7e-4 (t48-dist one call, fc_density.bias) -> 1.9e-3     simt 2.0e-4 (t48-dist, fc_density.bias) -> 8.2e-4
  end to end, scattered     tc 8.9e-4 (s1000, g_cam)       -> 3.6e-3     simt 7.1e-5 (s1000, g_cam)              -> 2.9e-4
  per element (pose, depth; |ref| >= 1e-2 |ref|max): translucent tc 1.5e-4 -> 5.8e-4, simt 1.8e-4 -> 7.2e-4 (t100-nonorm);
                                                      scattered tc 1.4e-3 (s1000) -> 5.8e-3, simt 9.5e-4 (s256) -> 3.8e-3
  ckpt 0.19 (t1024-d64) -> 0.75   suffix 0.25 (s1000) -> 1.0   cbwd0 0.70 (t1000) -> 2.8   rayacc 1.0 (simt, t48-dist) -> 4.0
  rayfin 0.98 (t100-eval) -> 3.9   reduce 0.21 (t256) -> 0.8   (both engines)
  layers0  tc fwd 7.4 (t48-dist) -> 30, dgrad 432 (t100-d128) -> 1700;  simt fwd 47.9 (t33) -> 190, dgrad 59.4 (t48-dist) -> 230
rayacc is asserted on the exact engine only.  There the frame's chunk 0 gp / gv equal the stash path's bit for bit (so the stash
path's per-sample gp / gv are the kernel's own inputs of every round); tc_dgrad_frame's split-bf16 encoding-adjoint GEMMs do not give
the stash path's bits, so on tensor cores frame_ray_acc is covered by rayfin (from the kernel's own lane partials) and end to end.

Wrong answers.  End to end, on translucent fields, each scores at least 10x its gate: rounds k >= 1 dropped (on every non-zero dW tensor
from S = 48; at S = 33, with one sample in the last chunk, 8.7e-3 on the weakest and 0.082 on the strongest), checkpoint of chunk k - 1
0.069 (t1000), checkpoint 1 0.60, suffix reset 0.091, df_last 0.34, first 32 rays dropped 0.13.  frame_ray_acc's two wrong answers move
the end-to-end pose terms by only 1e-4 .. 8e-3, at or below the tensor-core gate; they are reported there and asserted on rayacc.  On
scattered fields the end-to-end answers must exceed the gate.  Stage-local, every wrong answer scores at least 767 (suffix, checkpoint
of chunk k - 1, t1024-d128), >= 10x its gate: rayacc z of the previous chunk 2.9e5, last partial twice 2.9e6, round 1 skipped 1.9e6;
reduce first 32 rays 2.1e4.  The suffix formed as total - prefix scores 0.003 .. 1.8 on cbwd0, inside its gate: without near-opaque
samples in front of translucent ones nothing cancels, so it is reported, not asserted.  layers0 asserts test_gpu_layer_local's wrong
answers at 10x, except: on tensor cores W's fp16 lo half in the forward (199 .. 283) and the alpha head factor in the data gradient
(4478, S = 1024) must exceed the gate; on scattered fields the data gradient's bf16 lo half (156) and head factor (40.5) are reported.

Mutation check (each one line in nnb_frame.cuh on a scratch build; cases t100-eval, t256, t1024-d128 on both engines):
  (a) carry_s reset to 0 every round: every case fails end to end (dW 0.8 .. 3 of their maximum); test_gpu_render_frame_grad.py and
      test_gpu_render_frame_exact_grad.py fail too (14 of 90 selected tests, dW of layers0.0 0.27 .. 1.2).
  (b) carry read from ckpt[k - 2] for k >= 2: every case fails end to end (dW 0.07 .. 0.95); the two existing modules pass (90 of 90),
      which is the gap this module closes.
  (c) frame_ray_acc skipping round 1: every case fails end to end on g_c2w / g_cam (8e-3 .. 0.087, 4 .. 100x the gates); the existing
      modules fail on their pose terms (19 of 90).
The module takes about 2.5 minutes on the H100.
"""
import gc
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from nope_nerf_b200 import _lib as L
from oracle import nerf_oracle as O
import test_gpu_ray_local as RL
import test_gpu_layer_local as LL
from test_gpu_layer_local import nerr
from test_gpu_relu_mask import decode, gate_offset, layout

H, W = 48, 64
NEAR, FAR = 0.01, 10.0
TRUNK = [("layers0", 0), ("layers0", 2), ("layers0", 4), ("layers0", 6), ("layers1", 0), ("layers1", 2), ("layers1", 4), ("layers1", 6)]
# end-to-end gates (|got - ref|max / |ref|max per tensor) and stage-local gates (normalised error), per engine; see the docstring
E2E_GATES = dict(translucent=dict(tc=1.9e-3, simt=8.2e-4), scattered=dict(tc=3.6e-3, simt=2.9e-4))
STAGE_GATES = dict(ckpt=0.75, suffix=1.0, cbwd0=2.8, rayacc=4.0, rayfin=3.9, reduce=0.8)   # both engines
LAYER_GATES = dict(tc=dict(fwd=30.0, dgrad=1700.0), simt=dict(fwd=190.0, dgrad=230.0))   # layers0, per engine
# pose and depth terms per element: |got - ref| / |ref| where |ref| >= ELEM_FLOOR |ref|max
ELEM_GATES = dict(translucent=dict(tc=5.8e-4, simt=7.2e-4), scattered=dict(tc=5.8e-3, simt=3.8e-3))
ELEM_FLOOR = 1e-2
# frame_ray_acc's wrong answers move the end-to-end pose terms by about the tensor-core gate (see the docstring): reported there,
# asserted on the rayacc stage
REPORT_ONLY = ("z_prev_chunk", "last_partial_twice")
T_LAST_MIN = 0.05      # translucent: float64 transmittance into the last chunk, every ray
T_LAST_TARGET = 0.12   # the planted minimum over the rays
DROP_T = 1e-3          # scattered: the transmittance level whose first chunk must vary over the rays


# ---------------------------------------------------------------------------------------------------------------------- the cases
def _flags(c):
    from nope_nerf_b200 import ops
    cfg = dict(O.DEFAULT_CFG)
    cfg.update(dist_alpha=c.get("dist_alpha", False), white_background=c.get("white_bg", False),
               sample_option="ndc" if c.get("ndc") else "uniform", normalise_ray=c.get("normalise", True),
               use_ray_dir=c.get("use_dir", True))
    return ops.flags_from_cfg(cfg, c.get("occ", "softplus"), eval_=c.get("eval", False))


CASES = {
    "t33": dict(N=37, S=33, field="translucent"),
    "t48-dist": dict(N=301, S=48, field="translucent", dist_alpha=True),
    "t100-d64": dict(N=1024, S=100, D=64, field="translucent"),
    "t100-d128": dict(N=1024, S=100, D=128, field="translucent"),
    "t100": dict(N=1024, S=100, field="translucent"),
    "t100-relu-dist": dict(N=301, S=100, field="translucent", occ="relu", dist_alpha=True),
    "t100-relu": dict(N=301, S=100, field="translucent", occ="relu"),
    "t100-white": dict(N=301, S=100, field="translucent", white_bg=True),
    "t100-ndc": dict(N=301, S=100, field="translucent", ndc=True, dist_alpha=True),
    "t100-eval": dict(N=301, S=100, field="translucent", eval=True),
    "t100-nonorm": dict(N=301, S=100, field="translucent", normalise=False, use_dir=False),
    "t100-depth": dict(N=301, S=100, field="translucent", explicit=True),
    "t256": dict(N=5, S=256, field="translucent"),
    "t1000": dict(N=37, S=1000, field="translucent", dist_alpha=True),
    "t1024-d64": dict(N=37, S=1024, D=64, field="translucent"),
    "t1024-d128": dict(N=1, S=1024, D=128, field="translucent"),
    "t1024": dict(N=37, S=1024, field="translucent"),
    "s256": dict(N=301, S=256, field="scattered"),
    "s1000": dict(N=37, S=1000, field="scattered", dist_alpha=True),
}


def inputs(name, seed=0, case=None):
    """the case's fp32 inputs (numpy): pose, intrinsics, rays, prior depth or explicit depth, jitter and cotangents; case: a case dict
    that replaces CASES[name]"""
    c = CASES[name] if case is None else case
    N, S = c["N"], c["S"]
    rng = np.random.default_rng(seed)
    c2w = O.make_c2w(np.array([0.02, -0.03, 0.01], np.float32), np.array([0.05, 0.0, -0.04], np.float32)).astype(np.float32)
    cam = np.diag([1.2, -1.6, -1.0, 1.0]).astype(np.float32)
    ray_idx = rng.permutation(H * W)[:N]
    dmap = rng.uniform(0.6, 7.2, (24, 32)).astype(np.float32)
    inp = dict(N=N, S=S, H=H, W=W, near=np.float32(NEAR), far=np.float32(FAR), c2w=c2w, cam=cam, ray_idx=ray_idx,
               noise=rng.uniform(0, 1, (N, S)).astype(np.float32), g_rgb=rng.normal(0, 1, (N, 3)).astype(np.float32),
               g_dp=rng.normal(0, 0.1, N).astype(np.float32), g_dg=rng.normal(0, 0.1, N).astype(np.float32))
    if c.get("explicit"):
        dep = rng.uniform(0.6, 7.2, N).astype(np.float32); dep[::7] *= -1   # negative prior depth: the sign in g_depth
        inp.update(depth=dep, scale=None, shift=None)
    else:
        raw, _ = O.gather_prior_depth(dmap, ray_idx, H, W)
        inp.update(dmap=dmap, raw=raw, scale=np.float32(1.05), shift=np.float32(0.02))
    return inp


def oracle_logits(P, inp, flags, noise=True):
    """float64 density logits [N, S] and z [N, S] of the numpy oracle at the case's inputs (the host side of the planting)"""
    cfg = _cfg(flags, inp["S"])
    pix = O.pixels_from_idx(inp["ray_idx"], H, W, np.float64)
    depth = (inp["depth"] if "depth" in inp else inp["raw"] * inp["scale"] + inp["shift"]).astype(np.float64)
    P64 = {k: np.asarray(v, np.float64) for k, v in P.items()}
    _, cache = O.render_forward(P64, pix, depth, inp["c2w"].astype(np.float64), float(inp["cam"][0, 0]), float(inp["cam"][1, 1]), cfg,
                                noise=inp["noise"].astype(np.float64) if noise else None)
    return cache["mcache"]["s"].reshape(inp["N"], inp["S"]), cache["z"]


def _cfg(flags, S):
    return dict(O.DEFAULT_CFG, num_points=S, depth_range=(float(np.float32(NEAR)), float(np.float32(FAR))), dist_alpha=bool(flags & L.DIST_ALPHA),
                white_background=bool(flags & L.WHITE_BG), sample_option="ndc" if flags & L.NDC else "uniform",
                normalise_ray=bool(flags & L.NORMALISE), use_ray_dir=bool(flags & L.USE_DIR),
                occ_activation="softplus" if flags & L.SOFTPLUS else "relu")


def transmittance_np(s, z, flags):
    """float64 transmittance [N, S + 1] (T before every sample, and after the last) of logits s with sample depths z"""
    sig = np.where(s > 20, s, np.log1p(np.exp(np.minimum(s, 20)))) if flags & L.SOFTPLUS else np.maximum(s, 0)
    if flags & L.DIST_ALPHA:
        alpha = 1 - np.exp(-sig[:, :-1] * (z[:, 1:] - z[:, :-1]))
        alpha = np.concatenate([alpha, np.ones_like(alpha[:, :1])], 1)
    else:
        alpha = 1 - np.exp(-sig)
    om = 1 - alpha + O.EPSILON
    return np.concatenate([np.ones_like(om[:, :1]), np.cumprod(om, 1)], 1)


def plant(P, s, z, flags, field):
    """P with the density head moved (returns a new dict); s: a probe's logits [N, S] at the current head, z its sample depths"""
    P = dict(P)
    b0 = float(P["fc_density.bias"][0])
    S = s.shape[1]
    if field == "translucent":   # bisection on the bias shift: the smallest transmittance into the last chunk is T_LAST_TARGET
        last = 32 * ((S - 1) // 32)
        t_last = lambda db: transmittance_np(s + db, z, flags)[:, last].min()
        lo, hi = -60.0, 60.0
        for _ in range(80):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if t_last(mid) > T_LAST_TARGET else (lo, mid)
        P["fc_density.bias"] = np.full_like(P["fc_density.bias"], b0 + lo)
    else:   # the largest logit near-opaque, the 90th percentile -3 (test_gpu_ray_local's plant)
        target = 200.0 if flags & L.DIST_ALPHA else 17.0
        m = s - b0
        k = (target + 3.0) / float(m.max() - np.quantile(m, 0.9))
        P["fc_density.weight"] = (P["fc_density.weight"] * np.float32(k)).astype(np.float32)
        P["fc_density.bias"] = np.full_like(P["fc_density.bias"], target - k * float(m.max()))
    return P


def first_drop(T, level):
    """the chunk in which each ray's transmittance T [N, S + 1] first falls below level (C: never)"""
    S = T.shape[1] - 1
    below = T[:, 1:] < level
    return np.where(below.any(1), below.argmax(1) // 32, (S + 31) // 32)


# ------------------------------------------------------------------------------------------------------------ float64 reference
def field_ref(W, p, v, gates, s_gate, flags):
    """the MLP in float64 with fixed ReLU gates: p, v [M, 3] -> (rgb [M, 3], a [M]); gates: 9 bool [M, cols] (h0..h7, rgb hidden),
    s_gate: the ReLU density head's gate (the kernel's logit > 0)"""
    e = RL.encode_ref(p, 10)[0]
    h = e
    for li, (blk, i) in enumerate(TRUNK):
        if li == 4:
            h = torch.cat([h, e], 1)
        h = (h @ W["%s.%d.weight" % (blk, i)].T + W["%s.%d.bias" % (blk, i)]) * gates[li]
    s = (h @ W["fc_density.weight"].T + W["fc_density.bias"])[:, 0]
    sig = F.softplus(s, beta=1, threshold=20) if flags & L.SOFTPLUS else s * s_gate
    a = sig if flags & L.DIST_ALPHA else 1.0 - torch.exp(-sig)
    feat = h @ W["fc_feature.weight"].T + W["fc_feature.bias"]
    hr = (torch.cat([feat, RL.encode_ref(v, 4)[0]], 1) @ W["rgb_layers.0.weight"].T + W["rgb_layers.0.bias"]) * gates[8]
    return torch.sigmoid(hr @ W["fc_rgb.weight"].T + W["fc_rgb.bias"]), a


def reference(P, inp, flags, gates, s_gate, noise, dev="cuda"):
    """float64 autograd of the whole render: outputs, gradients, and a function giving the gradients under a wrong answer"""
    N, S = inp["N"], inp["S"]
    M = N * S
    A = RL.Arith()
    t64 = lambda x: torch.as_tensor(np.asarray(x, np.float64), device=dev)
    Wt = {k: t64(v).requires_grad_(True) for k, v in P.items()}
    c2w, cam = t64(inp["c2w"]).requires_grad_(True), t64(inp["cam"]).requires_grad_(True)
    q_in = dict(N=N, S=S, H=H, W=W, near=inp["near"], far=inp["far"], c2w=c2w, cam=cam, ray_idx=inp["ray_idx"])
    leaves = dict(Wt, g_c2w=c2w, g_cam=cam)
    if "depth" in inp:
        q_in["depth"] = t64(inp["depth"]).requires_grad_(True); leaves["g_depth"] = q_in["depth"]
    else:
        sc, sf = t64(inp["scale"]).requires_grad_(True), t64(inp["shift"]).requires_grad_(True)
        q_in.update(raw=inp["raw"], raw_rint=inp["raw"], scale=sc, shift=sf)
        leaves["g_scale"], leaves["g_shift"] = sc, sf
    nz = None if noise is None else t64(noise)
    p, z, v, _ = RL.ray_stage(A, RL._rowq(A, q_in, (N, S), dev), flags, S, nz)
    rgb_s, a_s = field_ref(Wt, p.reshape(M, 3), v.reshape(M, 3), gates, s_gate, flags)
    rec = dict(r=rgb_s[:, 0].reshape(N, S), g=rgb_s[:, 1].reshape(N, S), b=rgb_s[:, 2].reshape(N, S), a=a_s.reshape(N, S), z=z)
    q = RL._rowq(A, q_in, (N,), dev)
    ray = RL._ray_scalars(RL.setup_ray(A, q, flags), q)
    alpha, rgb, dp, dg = RL.composite_fwd_ref(A, rec, ray, flags)
    seeds = {k: t64(inp[k]) for k in ("g_rgb", "g_dp", "g_dg")}
    loss = (seeds["g_rgb"] * rgb).sum() + (seeds["g_dp"] * dp).sum() + (seeds["g_dg"] * dg).sum()
    names = list(leaves)
    mids = [rgb_s, a_s, p] + ([v] if v.requires_grad else [])
    g = torch.autograd.grad(loss, [leaves[k] for k in names] + mids, retain_graph=True, allow_unused=True)
    zero = lambda x: torch.zeros_like(x)
    G = {k: (zero(leaves[k]) if x is None else x) for k, x in zip(names, g)}
    g_rgb_s, g_a_s, gp = g[len(names):len(names) + 3]
    gv = g[len(names) + 3] if v.requires_grad else torch.zeros_like(p)
    rec_d = {k: x.detach() for k, x in rec.items()}
    ray_d = {k: ([y.detach() for y in x] if isinstance(x, list) else x.detach()) for k, x in ray.items()}
    with torch.no_grad():
        gs = RL.composite_bwd_ref(A, rec_d, ray_d, seeds, flags)
    # the composite adjoint the wrong answers replace is the one autograd took
    gs_auto = torch.cat([g_rgb_s.reshape(N, S, 3), g_a_s.reshape(N, S, 1)], 2)
    assert float((gs - gs_auto).abs().max()) <= 1e-9 * float(gs_auto.abs().max()), "composite_bwd_ref is not the float64 adjoint"
    z_d, dp_d, gp3, gv3 = z.detach(), dp.detach(), gp.reshape(N, S, 3), gv.reshape(N, S, 3)
    explicit = "depth" in inp

    def red(gp_, gv_, z_):
        rr, _ = RL.ray_bwd_ref(A, ray_d, gp_, gv_, z_, dp_d, seeds, flags, explicit)
        return rr

    red0 = red(gp3, gv3, z_d)
    tot0 = RL.reduce_ref(A, red0, torch.zeros(16, dtype=torch.float64, device=dev))
    # the ray adjoint's reduction reproduces autograd's pose gradients (every rayred term is accounted for)
    pose0 = _pose16(G)
    assert float((tot0 - pose0).abs().max()) <= 1e-9 * max(float(pose0.abs().max()), 1e-300), "ray_bwd_ref is not the float64 adjoint"

    def wrong(bug):
        """the gradients under a wrong answer: G + J^T (gs_bug - gs), or the pose terms from a wrong ray adjoint"""
        out = {k: x.clone() for k, x in G.items()}
        if bug in ("drop_late", "carry", "carry_one", "suffix_reset", "df_last"):
            with torch.no_grad():
                d = RL.composite_bwd_ref(A, rec_d, ray_d, seeds, flags, bug) - gs
            dg_ = torch.autograd.grad([rgb_s, a_s], [leaves[k] for k in names], [d[..., :3].reshape(M, 3), d[..., 3].reshape(M)],
                                      retain_graph=True, allow_unused=True)
            for k, x in zip(names, dg_):
                if x is not None:
                    out[k] = out[k] + x
            return out
        if bug == "z_prev_chunk":
            zw = torch.cat([z_d[:, :32], z_d[:, :-32]], 1)
            tot = RL.reduce_ref(A, red(gp3, gv3, zw), torch.zeros_like(tot0))
        elif bug == "last_partial_twice":
            dbl = torch.ones(S, dtype=torch.float64, device=dev); dbl[:32] = 2.0
            tot = RL.reduce_ref(A, red(gp3 * dbl[None, :, None], gv3 * dbl[None, :, None], z_d), torch.zeros_like(tot0))
        else:
            assert bug == "skip32"
            tot = RL.reduce_ref(A, red0, torch.zeros_like(tot0), "skip32")
        return _unpose16(out, tot - tot0)

    outs = dict(rgb=rgb.detach(), depth_pred=dp.detach(), depth_gt=dg.detach())
    T = torch.cat([torch.ones(N, 1, dtype=torch.float64, device=dev),
                   torch.cumprod(1.0 - alpha.detach() + O.EPSILON, 1)], 1)
    return outs, G, wrong, T


def _pose16(G):
    """the 16 reduced pose terms (ray_reduce's order) from a gradient dict"""
    gc, gk = G["g_c2w"], G["g_cam"].reshape(-1)
    v = [gc[i // 3, i % 3] for i in range(9)] + [gc[i, 3] for i in range(3)] + [gk[0], gk[5]]
    z = gc.new_zeros(())
    v += [G.get("g_scale", z).reshape(()), G.get("g_shift", z).reshape(())]
    return torch.stack(v)


def _unpose16(G, d):
    G["g_c2w"] = G["g_c2w"].clone(); G["g_cam"] = G["g_cam"].clone()
    for i in range(9):
        G["g_c2w"][i // 3, i % 3] += d[i]
    for i in range(3):
        G["g_c2w"][i, 3] += d[9 + i]
    G["g_cam"][0, 0] += d[12]; G["g_cam"][1, 1] += d[13]
    if "g_scale" in G:
        G["g_scale"] = G["g_scale"] + d[14]; G["g_shift"] = G["g_shift"] + d[15]
    return G


def compare(got, ref):
    """per tensor |got - ref|max / |ref|max over the outputs, every dW / db and the pose terms"""
    out = {}
    for k in list(ref):
        r, g = ref[k].double(), got[k].double()
        m = float(r.abs().max())
        out[k] = float((g - r).abs().max()) / m if m > 0 else (0.0 if float(g.abs().max()) == 0 else math.inf)
    return out


def compare_elements(got, ref):
    """per element |got - ref| / |ref| of the pose and depth terms, over the elements with |ref| >= ELEM_FLOOR |ref|max"""
    out = {}
    for k in ("g_c2w", "g_cam", "g_scale_shift", "g_depth"):
        if k in ref:
            r, g = ref[k].double().reshape(-1), got[k].double().reshape(-1)
            big = r.abs() >= ELEM_FLOOR * r.abs().max()
            if big.any():
                out[k] = float(((g - r).abs() / r.abs())[big].max())
    return out


def _grad_tensors(G):
    """a reference / wrong-answer gradient dict -> the tensors the kernel writes (g_scale_shift as one)"""
    out = {k: v for k, v in G.items() if k not in ("g_scale", "g_shift")}
    if "g_scale" in G:
        out["g_scale_shift"] = torch.stack([G["g_scale"].reshape(()), G["g_shift"].reshape(())])
    return out


# ------------------------------------------------------------------------------------------------------------------ layout mirror
def _align(x, a=256):
    return (x + a - 1) // a * a


def frame_layout(N, S, D, engine):
    """byte offsets of frame_bwd_layout_bytes (nnb_frame.cuh) on `engine` ('tc' or 'simt'): ckpt [C - 1][N], suffix [N], raypart
    [N][9][32], the chunk stash (its own make_layout of R rows per ray, lay) and the total"""
    e = L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT
    off = L.lib.nnb_render_frame_workspace_bytes_engine(N, S, D, e)   # frame_layout_bytes(N, the forward weight image)
    C = (S + 31) // 32
    R = 32 if engine == "tc" else min(S, 32)
    out = dict(C=C, R=R)
    for k, n in (("ckpt", 4 * N * (C - 1)), ("suffix", 4 * N), ("raypart", 1152 * N)):
        out[k] = off; off += _align(n)
    lay = layout(N, R, D)
    out["chunk"], out["lay"] = off, lay
    off += _align(lay["total"] if engine == "tc" else lay["gates"])   # the exact engine's stash has no gate bits
    off += _align(34 * D * D + 576 * D) if engine == "tc" else 0       # the transposed weight image
    out["total"] = off
    return out


# ------------------------------------------------------------------------------------------------------------------------ GPU run
def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _call_kw(inp, flags, D):
    kw = dict(N=inp["N"], S=inp["S"], flags=flags, near=NEAR, far=FAR, ray_idx=_cu(inp["ray_idx"]), H=H, W=W, hidden_dim=D)
    if "depth" in inp:
        kw["depth"] = _cu(inp["depth"])
    else:
        kw.update(depth_map=_cu(inp["dmap"]), scale=torch.tensor([float(inp["scale"])]).cuda(),
                  shift=torch.tensor([float(inp["shift"])]).cuda())
    return kw


def _f32(ws, off, rows, cols):
    return ws[off:off + rows * cols * 4].view(torch.float32).view(rows, cols)


def stash_run(P, inp, flags, D, engine, noise, backward=False):
    """nnb_render_fwd (NNB_STASH) on the engine: records [N S, 8], the gates the engine took (9 bool [N S, cols]) and its h stash;
    with backward, nnb_render_bwd's per-sample point and direction adjoints gp / gv [N S, 3] too"""
    from nope_nerf_b200 import ops
    N, S = inp["N"], inp["S"]
    call = ops.RenderCall(_cu(O.flatten_params(P)), _cu(inp["c2w"]), _cu(inp["cam"]), stash=True,
                          engine=L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT, noise=_cu(inp["noise"]) if noise else None,
                          **_call_kw(inp, flags, D))
    ws, lay, M = call.ws, layout(N, S, D), N * S
    if backward:   # hands the workspace back to the pool; ws stays alive, and nothing takes it before the copies below
        g = _grads(D, N)
        call.backward(_cu(inp["g_rgb"]), _cu(inp["g_dp"]), _cu(inp["g_dg"]), g["w"], g["g_c2w"], g["g_cam"],
                      g["g_depth"] if "depth" in inp else None, g["g_scale_shift"])
    torch.cuda.synchronize()
    st = dict(rec=_f32(ws, lay["rec"], lay["Mpad"], 8)[:M].clone(),
              h=[_f32(ws, lay["h"][l] if l < 8 else lay["hr"], lay["Mpad"], D if l < 8 else D // 2)[:M].clone() for l in range(9)])
    if engine == "tc":
        st["gates"] = [_decode(ws, lay, l, D)[:M] for l in range(9)]
    else:
        st["gates"] = [h > 0 for h in st["h"]]
    if backward:
        st["gp"], st["gv"] = _f32(ws, lay["gp"], lay["Mpad"], 4)[:M, :3].clone(), _f32(ws, lay["gv"], lay["Mpad"], 4)[:M, :3].clone()
    else:
        call.release()
    return st


def _decode(ws, lay, l, D, base=0):
    cols = D if l < 8 else D // 2
    g0 = base + lay["gates"] + gate_offset(lay, l)
    return torch.from_numpy(decode(ws[g0:g0 + lay["Mpad"] * cols // 8].cpu().numpy(), lay["n_tiles"], cols)).cuda()


def _grads(D, N):
    return dict(w=torch.zeros(L.num_params(D), device="cuda"), g_c2w=torch.zeros(4, 4, device="cuda"),
                g_cam=torch.zeros(4, 4, device="cuda"), g_scale_shift=torch.zeros(2, device="cuda"),
                g_depth=torch.full((N,), float("nan"), device="cuda"))


def _got(outs, g, D, explicit):
    got = dict(rgb=outs[0], depth_pred=outs[1], depth_gt=outs[2])
    got.update({k: torch.from_numpy(v).cuda() for k, v in O.unflatten_params(g["w"].cpu().numpy(), D).items()})
    got.update(g_c2w=g["g_c2w"], g_cam=g["g_cam"], g_scale_shift=g["g_scale_shift"])
    if explicit:
        got["g_depth"] = g["g_depth"]
    return got


def one_call(P, inp, flags, D, engine):
    from nope_nerf_b200 import ops
    g = _grads(D, inp["N"])
    kw = _call_kw(inp, flags, D)
    outs = ops.render_frame_bwd(_cu(O.flatten_params(P)), _cu(inp["c2w"]), _cu(inp["cam"]), _cu(inp["g_rgb"]), _cu(inp["g_dp"]),
                                _cu(inp["g_dg"]), g["w"], g["g_c2w"], g["g_cam"], g["g_depth"] if "depth" in inp else None,
                                g["g_scale_shift"], engine=L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT, **kw)
    torch.cuda.synchronize()
    return _got(outs, g, D, "depth" in inp)


def pair(P, inp, flags, D, engine, noise=True, backward=True):
    """the training pair with jitter; returns (outputs and gradients, the workspace read back after the call)"""
    from nope_nerf_b200 import ops
    cls = ops.FrameRenderCall if engine == "tc" else ops.ExactFrameRenderCall
    call = cls(_cu(O.flatten_params(P)), _cu(inp["c2w"]), _cu(inp["cam"]), engine=L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT,
               noise=_cu(inp["noise"]) if noise else None, **_call_kw(inp, flags, D))
    outs = tuple(t.clone() for t in (call.rgb, call.depth_pred, call.depth_gt))
    ws = call.ws   # the backward hands the workspace back to the pool; it stays alive, and nothing takes it before the copies below
    g = _grads(D, inp["N"])
    if backward:
        call.backward(_cu(inp["g_rgb"]), _cu(inp["g_dp"]), _cu(inp["g_dg"]), g["w"], g["g_c2w"], g["g_cam"],
                      g["g_depth"] if "depth" in inp else None, g["g_scale_shift"])
    torch.cuda.synchronize()
    N, S = inp["N"], inp["S"]
    fl = frame_layout(N, S, D, engine)
    assert ws.numel() == fl["total"], "frame workspace layout"
    C, R, lay, base = fl["C"], fl["R"], fl["lay"], fl["chunk"]
    rd = dict(ckpt=_f32(ws, fl["ckpt"], max(C - 1, 1), N)[:C - 1].clone(), suffix=_f32(ws, fl["suffix"], 1, N)[0].clone(),
              rec=_f32(ws, base + lay["rec"], lay["Mpad"], 8)[:N * R].clone(), gs=_f32(ws, base + lay["gs"], lay["Mpad"], 4)[:N * R].clone(),
              h=[_f32(ws, base + (lay["h"][l] if l < 8 else lay["hr"]), lay["Mpad"], D if l < 8 else D // 2)[:N * R].clone()
                 for l in range(9)])
    rows = lambda key, cols: _f32(ws, base + lay[key], lay["Mpad"], cols)[:N * R].clone()
    rd.update(dy=[_f32(ws, base + lay["dy"][l], lay["Mpad"], D)[:N * R].clone() for l in range(8)], feat=rows("feat", D),
              hr=rd["h"][8], enc=rows("enc", 64), denc=rows("denc", 32), dfeat=rows("dfeat", D), dyr=rows("dyr", D // 2),
              dyc=rows("dyc", 4), gp=rows("gp", 4)[:, :3], gv=rows("gv", 4)[:, :3],
              raypart=_f32(ws, fl["raypart"], N * 9, 32).clone().view(N, 9, 32), rayred=_f32(ws, base + lay["rayred"], N, 16).clone())
    if engine == "tc":
        rd["gates"] = [_decode(ws, lay, l, D, base)[:N * R] for l in range(9)]
    if not backward:
        call.release()
    return _got(outs, g, D, "depth" in inp), rd


def _chunk0_rows(N, S, R):
    """stash-path rows n S + j of chunk 0, in the chunk stash's row order R n + j (j < min(S, 32))"""
    j = torch.arange(min(S, 32), device="cuda")
    n = torch.arange(N, device="cuda")
    return (n[:, None] * S + j[None]).reshape(-1), (n[:, None] * R + j[None]).reshape(-1)


_PLANTED = {}


def planted(name):
    """(P, inp, flags, D) with the case's field planted from a probe run's logits (cached per case)"""
    if name in _PLANTED:
        return _PLANTED[name]
    c = CASES[name]
    D = c.get("D", 256)
    flags = _flags(c)
    inp = inputs(name)
    P = dict(O.init_params(seed=7, D=D, hf_damp=True))
    st = stash_run(P, inp, flags, D, "tc" if inp["S"] >= 16 else "simt", noise=False)
    s0 = st["rec"][:, 4].double().reshape(inp["N"], inp["S"]).cpu().numpy()
    z0 = st["rec"][:, 5].double().reshape(inp["N"], inp["S"]).cpu().numpy()
    P = plant(P, s0, z0, flags, c["field"])
    _PLANTED[name] = (P, inp, flags, D)
    return _PLANTED[name]


@pytest.fixture(scope="module", autouse=True)
def _release_pool():
    """the workspaces this module adds to the library's pool are dropped when it finishes"""
    yield
    from nope_nerf_b200 import ops
    ops._pool.free.clear()
    _PLANTED.clear()
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------ measurement
BUGS = ("drop_late", "carry", "carry_one", "suffix_reset", "df_last", "z_prev_chunk", "last_partial_twice", "skip32")


def _applies(bug, inp, flags):
    return {"df_last": bool(flags & L.DIST_ALPHA), "skip32": inp["N"] > 32,
            "carry": inp["S"] > 64}.get(bug, inp["S"] > 32)   # the checkpoint of chunk k - 1 differs from 1 only for k >= 2


def _e2e(name, engine, entry, st, got):
    P, inp, flags, D = planted(name)
    s_gate = (st["rec"][:, 4] > 0).double()
    gates = [g.double() for g in st["gates"]]
    noise = inp["noise"] if entry == "pair" and not flags & L.NDC else None
    outs, G, wrong, T = reference(P, inp, flags, gates, s_gate, noise)
    ref = dict(outs, **_grad_tensors(G))
    err = compare(got, ref)
    res = dict(err=err, teeth={}, T=T, S=inp["S"], elem=compare_elements(got, ref))
    for bug in BUGS:
        if _applies(bug, inp, flags):
            wr = dict(outs, **_grad_tensors(wrong(bug)))
            sc = {k: float((got[k].double() - wr[k]).abs().max()) / max(float(ref[k].abs().max()), 1e-300) for k in ref
                  if k not in outs}
            res["teeth"][bug] = sc
    return res


def frame_lanes_ref(A, gp, gv, z, bug=None):
    """frame_ray_acc over the rounds k = C - 1 .. 0: the lane partials [N, 9, 32] of sum gp, sum z gp, sum gv (lane = sample 32 k +
    lane), from per-sample gp / gv [N, S, 3] and z [N, S].  Bugs: z_prev_chunk (z of chunk k - 1 in round k >= 1), last_partial_twice
    (the last round's terms added twice), skip_round1 (round 1 dropped)"""
    if bug == "z_prev_chunk":
        z = torch.cat([z[:, :32], z[:, :-32]], 1)
    cg = [RL.chunks(gp[..., c], 0.0) for c in range(3)]
    cv = [RL.chunks(gv[..., c], 0.0) for c in range(3)]
    cz = RL.chunks(z, 0.0)
    C = cz.shape[1]
    acc = None
    for k in range(C - 1, -1, -1):
        term = [g[:, k] for g in cg] + [A.r(cz[:, k] * g[:, k]) for g in cg] + [v[:, k] for v in cv]
        if bug == "skip_round1" and k == 1:
            continue
        reps = 2 if bug == "last_partial_twice" and k == 0 else 1
        for _ in range(reps):
            acc = term if acc is None else [A.r(a + t) for a, t in zip(acc, term)]
    return torch.stack(acc, 1)


def _qin(inp):
    q = dict(N=inp["N"], S=inp["S"], H=H, W=W, near=inp["near"], far=inp["far"], c2w=np.asarray(inp["c2w"], np.float64),
             cam=np.asarray(inp["cam"], np.float64), ray_idx=inp["ray_idx"])
    if "depth" in inp:
        q["depth"] = inp["depth"].astype(np.float64)
    else:
        q.update(raw=inp["raw"].astype(np.float64), raw_rint=inp["raw"].astype(np.float64), scale=inp["scale"], shift=inp["shift"])
    return q


STAGES = ("ckpt", "suffix", "cbwd0", "rayacc", "rayfin", "reduce")


def measure_stages(d, inp, flags, dev="cuda"):
    """every reverse-round stage's normalised error, and its wrong answers', from the kernel's own inputs.  d (float64 tensors): rec
    {r, g, b, a, z: [N, S]} and gp / gv [N, S, 3] of the stash path on the same inputs; the frame's ckpt [C - 1, N], suffix [N], chunk
    0's gs [N, min(S, 32), 4], raypart [N, 9, 32], rayred [N, 16], g_depth [N] (explicit depth) and the reduced pose terms red [16]"""
    N, S = inp["N"], inp["S"]
    C = (S + 31) // 32
    k0 = min(S, 32)
    rec = d["rec"]
    rec32 = {k: v.float() for k, v in rec.items()}
    q_in = _qin(inp)
    seeds = {k: torch.as_tensor(np.asarray(inp[k], np.float64), device=dev) for k in ("g_rgb", "g_dp", "g_dg")}
    seeds32 = {k: v.float() for k, v in seeds.items()}
    explicit = "depth" in inp
    out = {s: dict(err=0.0, teeth={}, detect={}) for s in STAGES}

    def check(stage, got, ref, sc):
        out[stage]["err"] = max(out[stage]["err"], nerr(got, ref, sc))

    def tooth(stage, kind, got, wrong, sc, detect=False):
        out[stage]["detect" if detect else "teeth"][kind] = float(((got - wrong).abs() / sc).max())
    # ---- ckpt: the transmittance after chunk k, k < C - 1
    if C > 1:
        A = RL.Arith(track=True)
        _, Tc = RL.transmittance(A, RL.alpha_of(A, rec, flags))
        y = Tc[:, 1:, 0]
        sc = RL.scales(A, y, N)
        check("ckpt", d["ckpt"].T, y.detach(), sc)
        A32 = RL.Arith(f32=True)
        for bug in ("carry", "carry_one"):   # the carry into chunk k + 1 formed from the wrong checkpoint
            if S > 64 or bug == "carry_one":
                _, T32 = RL.transmittance(A32, RL.alpha_of(A32, rec32, flags), bug)
                tooth("ckpt", bug, d["ckpt"].T, T32[:, 1:, 0].double(), sc)
    # ---- suffix and chunk 0's adjoint
    A = RL.Arith(track=True)
    ray = RL.setup_ray(A, RL._rowq(A, q_in, (N,), dev), flags)
    gs, suf = RL.composite_bwd_ref(A, rec, ray, seeds, flags, want_suffix=True)
    sc = RL.scales(A, torch.cat([gs[:, :k0].reshape(N, -1), suf[:, None]], 1), N)
    gs, suf = gs.detach()[:, :k0].reshape(N, -1), suf.detach()
    got_gs = d["gs0"].reshape(N, -1)
    check("cbwd0", got_gs, gs, sc[:, :-1])
    check("suffix", d["suffix"], suf, sc[:, -1])
    A32 = RL.Arith(f32=True)
    ray32 = RL.setup_ray(A32, RL._rowq(A32, q_in, (N,), dev), flags)
    for bug in ("drop_late", "carry", "carry_one", "suffix_reset", "total_minus_prefix"):
        if S <= 32 or (bug == "carry" and S <= 64):
            continue
        w_gs, w_suf = RL.composite_bwd_ref(A32, rec32, ray32, seeds32, flags, bug, want_suffix=True)
        tooth("cbwd0", bug, got_gs, w_gs.double()[:, :k0].reshape(N, -1), sc[:, :-1], detect=bug == "total_minus_prefix")
        if bug != "total_minus_prefix":
            tooth("suffix", bug, d["suffix"], w_suf.double(), sc[:, -1])
    # ---- rayacc: the lane partials of frame_ray_acc from the samples' gp, gv and z
    A = RL.Arith(track=True)
    part = frame_lanes_ref(A, d["gp"], d["gv"], rec["z"])
    sc = RL.scales(A, part, N).reshape(N, 9, 32)
    part = part.detach()
    check("rayacc", d["raypart"], part, sc)
    A64 = RL.Arith()
    for bug in ("z_prev_chunk", "last_partial_twice", "skip_round1"):
        if S > 32:
            tooth("rayacc", bug, d["raypart"], frame_lanes_ref(A64, d["gp"], d["gv"], rec["z"], bug), sc)
    # ---- rayfin: ray_bwd's adjoint from the kernel's own lane partials
    A = RL.Arith(track=True)
    q = RL._rowq(A, q_in, (N,), dev)
    ray = dict(RL._ray_scalars(RL.setup_ray(A, q, flags), q), depth_sign=torch.sign(torch.as_tensor(
        RL.setup_ray(A32, RL._rowq(A32, q_in, (N,), dev), flags)["depth"])).double())
    sums = [[RL.warp_sum(A, d["raypart"][:, 3 * j + c]) for c in range(3)] for j in range(3)]
    red, gdep = RL.ray_adjoint_ref(A, ray, *sums, d["depth_pred"], seeds, flags, explicit)
    y = torch.cat([red, gdep[:, None]], 1)
    sc = RL.scales(A, y, N)
    y = y.detach()
    got = torch.cat([d["rayred"], (d["g_depth"] if explicit else gdep.detach())[:, None]], 1)
    check("rayfin", got, y, sc)
    # ---- reduce: the pose, camera and scale / shift gradients from the kernel's rayred (zero base)
    A = RL.Arith(track=True)
    tot = RL.reduce_ref(A, d["rayred"], torch.zeros(16, dtype=torch.float64, device=dev))
    sc = RL.scales(A, tot[:, None], 16)[:, 0]
    have = torch.tensor([True] * 14 + [not explicit] * 2, device=dev)
    check("reduce", d["red"][have], tot.detach()[have], sc[have])
    if N > 32:
        tooth("reduce", "skip32", d["red"][have], RL.reduce_ref(A64, d["rayred"], torch.zeros_like(tot), "skip32")[have], sc[have])
    return out


def layers0(rd, P, D, engine, flags):
    """test_gpu_layer_local's forward and data-gradient checks on chunk 0's rows of the chunk stash (the frame's own stash and
    data-gradient modes)"""
    W = {k: torch.from_numpy(np.asarray(v, np.float64)).cuda() for k, v in P.items()}
    st = {"h%d" % l: rd["h"][l] for l in range(8)}
    st.update({"dy%d" % l: rd["dy"][l] for l in range(8)})
    st.update({k: rd[k] for k in ("feat", "hr", "enc", "denc", "rec", "dfeat", "dyr", "dyc")}, gs=rd["gs"], flags=flags)
    st = {k: (v.double() if torch.is_tensor(v) else v) for k, v in st.items()}
    st["enc"], st["denc"] = st["enc"][:, :63], st["denc"][:, :27]
    return dict(fwd=LL.forward_errors(st, W, D, engine == "tc"), dgrad=LL.dgrad_errors(st, W, D))


def _stage_data(st, rd, got, inp, engine):
    """measure_stages' inputs from the stash path's run (st, same inputs) and the pair's workspace (rd) and outputs (got)"""
    N, S = inp["N"], inp["S"]
    R, k0 = (32 if engine == "tc" else min(S, 32)), min(S, 32)
    rec = {k: st["rec"][:, i].double().reshape(N, S) for i, k in enumerate(("r", "g", "b", "a", "s", "z"))}
    gc, gk = got["g_c2w"].double(), got["g_cam"].double().reshape(-1)
    red = torch.stack([gc[i // 3, i % 3] for i in range(9)] + [gc[i, 3] for i in range(3)] + [gk[0], gk[5]] +
                      list(got["g_scale_shift"].double()))
    return dict(rec=rec, gp=st["gp"].double().reshape(N, S, 3), gv=st["gv"].double().reshape(N, S, 3), ckpt=rd["ckpt"].double(),
                suffix=rd["suffix"].double(), gs0=rd["gs"].double().reshape(N, R, 4)[:, :k0], raypart=rd["raypart"].double(),
                rayred=rd["rayred"].double(), depth_pred=got["depth_pred"].double(),
                g_depth=got["g_depth"].double() if "g_depth" in got else None, red=red)


def _check_coverage(name, T):
    """the case's field carries weight where the test needs it (T: float64 transmittance [N, S + 1] of the reference)"""
    c = CASES[name]
    S = c["S"]
    Tn = T.cpu().numpy()
    if c["field"] == "translucent":
        t_last = Tn[:, 32 * ((S - 1) // 32)]
        assert t_last.min() >= T_LAST_MIN, (name, "opaque before the last chunk", float(t_last.min()))
    else:
        drop = first_drop(Tn, DROP_T)
        assert len(set(drop[drop < (S + 31) // 32].tolist())) >= 4, (name, "rays lose their transmittance in too few rounds", drop)


def _check_chunk_stash(st, rd, inp, engine):
    """the frame's chunk stash holds the stash path's rows of chunk 0 bit for bit: records, h stash and (tensor cores) gate bits"""
    N, S = inp["N"], inp["S"]
    R = 32 if engine == "tc" else min(S, 32)
    a, b = _chunk0_rows(N, S, R)
    assert torch.equal(rd["rec"][b, :6], st["rec"][a, :6]), "chunk stash records"
    for l in range(9):
        assert torch.equal(rd["h"][l][b], st["h"][l][a]), ("chunk stash h", l)
        if engine == "tc":
            assert torch.equal(rd["gates"][l][b], st["gates"][l][a]), ("chunk stash gate bits", l)
    print("chunk 0's gp / gv equal the stash path's bit for bit:", torch.equal(rd["gp"][b], st["gp"][a]), torch.equal(rd["gv"][b], st["gv"][a]))


def _check_e2e(key, res, engine, field):
    gate = E2E_GATES[field][engine]
    worst = max(res["err"].values())
    assert worst <= gate, (key, "end to end", {k: v for k, v in res["err"].items() if v > gate}, gate)
    dW = [k for k in res["err"] if k.endswith(("weight", "bias"))]
    for bug, sc in res["teeth"].items():
        best = max(sc.values())
        if bug in REPORT_ONLY:
            continue
        if bug == "drop_late" and field == "translucent" and res["S"] > 33:   # at S = 33 the last chunk holds one sample
            low = {k: sc[k] for k in dW if sc[k] < 10 * gate}
            assert not low, (key, "rounds k >= 1 dropped within 10x of the gate on", low)
        elif field == "translucent":
            assert best >= 10 * gate, (key, "wrong answer '%s' within 10x of the gate" % bug, best, gate)
        else:   # scattered: late rounds carry little weight by design
            assert best > gate, (key, "wrong answer '%s' within the gate" % bug, best, gate)
    for k, e in res["elem"].items():
        assert e <= ELEM_GATES[field][engine], (key, "per element", k, e, ELEM_GATES[field][engine])


def _check_stage(key, out, engine, field):
    for stage, gate in STAGE_GATES.items():
        if stage == "rayacc" and engine == "tc":   # the stash path's gp are not the frame's own on tensor cores (see the docstring)
            continue
        r = out[stage]
        assert r["err"] <= gate, (key, stage, r["err"], gate)
        for kind, t in r["teeth"].items():
            assert t >= 10 * gate, (key, stage, "wrong answer '%s' within 10x of the gate" % kind, t, gate)


def _summary(res):
    return dict(err=max(res["err"].values()), worst=max(res["err"], key=res["err"].get), elem=res["elem"],
                teeth={b: "%.3g" % max(v.values()) for b, v in res["teeth"].items()},
                drop_late_min_dW="%.3g" % min((v for k, v in res["teeth"].get("drop_late", {}).items()
                                                if k.endswith(("weight", "bias"))), default=math.inf))


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ("tc", "simt"))
@pytest.mark.parametrize("name", list(CASES))
def test_frame_local(name, engine):
    P, inp, flags, D = planted(name)
    field = CASES[name]["field"]
    ndc = bool(flags & L.NDC)
    # ---- the training pair with jitter
    st = stash_run(P, inp, flags, D, engine, noise=not ndc, backward=True)
    got, rd = pair(P, inp, flags, D, engine, noise=not ndc)
    _check_chunk_stash(st, rd, inp, engine)
    res = _e2e(name, engine, "pair", st, got)
    _check_coverage(name, res["T"])
    stage = measure_stages(_stage_data(st, rd, got, inp, engine), inp, flags)
    lay0 = layers0(rd, P, D, engine, flags)
    print((name, engine, "pair"), _summary(res), {s: "%.3g" % v["err"] for s, v in stage.items()},
          {(s, k): "%.3g" % t for s, v in stage.items() for k, t in list(v["teeth"].items()) + list(v["detect"].items())})
    LL._report((name, engine, "layers0"), lay0)
    _check_e2e((name, engine, "pair"), res, engine, field)
    _check_stage((name, engine, "pair"), stage, engine, field)
    # scattered fields scale fc_density.weight by ~10: there dropping W's bf16 lo half and the alpha head factor score 40 .. 160, reported
    # on tensor cores W's fp16 lo half dropped (forward) and the alpha head factor (data gradient) reach 199 .. 283 and 4478 at S >= 256:
    # they must exceed the gate; on scattered fields (fc_density.weight scaled by ~10) the data gradient's two score 40 .. 160, reported
    detect = {("fwd", "lo"), ("dgrad", "head_factor")} if engine == "tc" else set()
    skip = {("dgrad", "lo"), ("dgrad", "head_factor")} if field == "scattered" else set()
    LL._check((name, engine, "layers0"), lay0, LAYER_GATES[engine], skip_teeth=detect | skip)
    for stage, kind in detect - skip:
        assert lay0[stage]["teeth"][kind] > LAYER_GATES[engine][stage], (name, engine, "layers0", stage, kind)
    # ---- the one-call backward (no jitter): the gates of the stash path without noise
    if not ndc:
        st = stash_run(P, inp, flags, D, engine, noise=False)
    got = one_call(P, inp, flags, D, engine)
    res = _e2e(name, engine, "one", st, got)
    _check_coverage(name, res["T"])
    print((name, engine, "one"), _summary(res))
    _check_e2e((name, engine, "one"), res, engine, field)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ("tc", "simt"))
def test_early_termination_on_a_scattered_field(engine):
    """render_frame_engine(t_min): each ray stops after the chunk where its float64 carry first falls below t_min, with the training
    forward's checkpoint bits as t_final; rays that never fall below keep the t_min = 0 bits; the rays stop in at least 4 rounds"""
    from nope_nerf_b200 import ops
    name, t_min = "s256", DROP_T
    P, inp, flags, D = planted(name)
    N, S = inp["N"], inp["S"]
    C = (S + 31) // 32
    e = L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT
    st = stash_run(P, inp, flags, D, engine, noise=False)
    rec = {k: st["rec"][:, i].double().reshape(N, S) for i, k in enumerate(("r", "g", "b", "a", "s", "z"))}
    om, Tc = RL.transmittance(RL.Arith(), RL.alpha_of(RL.Arith(), rec, flags))
    carry = torch.cat([Tc[:, 1:, 0], (Tc[:, -1, 0] * om[:, -1].prod(1))[:, None]], 1).cpu().numpy()   # [N, C]: after every chunk
    below = carry < t_min
    stop = np.where(below.any(1), below.argmax(1) + 1, C)
    near = (np.abs(carry / t_min - 1) < 1e-3).any(1)
    assert len(set(stop[~near & (stop < C)].tolist())) >= 4, ("rays stop in too few rounds", stop)
    flat, c2w, cam = _cu(O.flatten_params(P)), _cu(inp["c2w"]), _cu(inp["cam"])
    kw = _call_kw(inp, flags, D)
    *_, n0, t0 = ops.render_frame_engine(flat, c2w, cam, engine=e, t_min=0.0, want_stats=True, **kw)
    *_, n_eval, t_final = ops.render_frame_engine(flat, c2w, cam, engine=e, t_min=t_min, want_stats=True, **kw)
    _, rd = pair(P, inp, flags, D, engine, noise=False, backward=False)
    torch.cuda.synchronize()
    n_eval, t_final, n0, t0 = n_eval.cpu().numpy(), t_final.cpu(), n0.cpu().numpy(), t0.cpu()
    assert (n0 == S).all()
    ok = ~near
    assert np.array_equal(n_eval[ok], np.minimum(32 * stop[ok], S)), ("n_eval", n_eval[ok], 32 * stop[ok])
    ckpt = rd["ckpt"].cpu()
    for n in range(N):
        k = (int(n_eval[n]) + 31) // 32
        if k < C:
            assert torch.equal(t_final[n], ckpt[k - 1, n]), (n, "t_final is not the checkpoint")
        else:
            assert torch.equal(t_final[n], t0[n]), (n, "t_final of a ray that never stops")
    print(engine, "rays per stopping round:", np.bincount(stop[ok], minlength=C + 1)[1:])

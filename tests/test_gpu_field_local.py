"""Layer-local float64 checks of explicit-point field queries on the exact-fp32 engine, with weight gradients.

OfficialStaticNerf.forward(p, ray_d) with autograd runs nnb_field_fwd (NNB_STASH, NNB_ENGINE_SIMT) and nnb_field_bwd with g_pts,
g_dirs and g_weights; so does the first half of gradient().  This path differs from rendering: the direction encoding is per point (the
ones when dirs is NULL), the cotangent is copied into the stash for rows < M only, and M is any size, not N S.  Every stage is rebuilt
in float64 from the kernel's OWN inputs, read back from the workspace through the layout(M, 1, D) mirror (test_gpu_relu_mask.layout,
checked against nnb_debug_layout below):
  enc      the stash's point and direction encodings against encode_ref of the input points and directions (or the ones);
  layers   every forward GEMM, the density head (alpha, sigma or the raw logit) and colour head, the data-gradient chain from the cotangent,
           and every weight-gradient job, including the encoding slice of layers1.0 and the direction slice of rgb_layers.0
           (test_gpu_layer_local's forward_errors / dgrad_errors / wgrad_errors and error model);
  encadj   g_pts and g_dirs from the kernel's dy0, dy4 and dyr through encode_bwd (test_gpu_ray_local's Arith / scales machinery).
out_rgba must be the stash's records, and g_pts / g_dirs the stash's gp / gv, bit for bit.

Largest normalised errors measured over all cases below on the unmodified kernels (NVIDIA H100 80GB HBM3, 700 W power limit), and the
gates, which are those of the exact engine's render cases (test_gpu_layer_local.SIMT_GATES, test_gpu_ray_local.SIMT_GATES):
  enc     0.99  (D = 64, 16901)          -> 4.1        forward          49.8  (D = 256, 16901, alpha)  -> 190
  encadj  1.54  (D = 256, 16901, alpha)  -> 7.5        data gradient    51.0  (D = 256, 5117, alpha)   -> 280
                                                       weight gradient   139  (D = 256, 5117, logit)   -> 680
Wrong answers (each must score at least 10x its gate in every case, from the same stash): those of test_gpu_layer_local on every layer
(one K-step, one bias or added term, the weights' or dY's lo half, the layer's own ReLU gate, the heaviest 32-sample chunk), the
density head's alpha factor dropped or added and the other activation's slope (not with the raw logit); octave L - 1 dropped from
encode_bwd and layer 4's encoding slice dropped (g_pts); and the direction slice of rgb_layers.0's weight gradient dropped.  The
smallest measured is 3290 for the weights' fp16 lo half dropped in the forward (D = 64, M = 1; 17x its gate).  W0's bf16 lo half
dropped from g_pts must exceed the gate only: it scores 44.6 at M = 1 (6x the gate; test_gpu_ray_local asserts 10x on the render
path)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
import test_gpu_layer_local as LL
from test_gpu_ray_local import Arith, SIMT_GATES, encode_bwd_ref, encode_ref, scales
from test_gpu_relu_mask import layout

SIZES = (1, 63, 64, 65, 5117, 16901)
DIMS = (64, 128, 256)
HEADS = ("alpha", "sigma", "logit")


def head_flags(head):
    from nope_nerf_b200 import _lib as L
    return L.SOFTPLUS | {"alpha": 0, "sigma": L.DIST_ALPHA, "logit": L.RAW_DENSITY}[head]


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def run(D, M, head, with_dirs):
    """nnb_field_fwd + nnb_field_bwd on seeded points; returns (stash dict of float64 [M, cols], float64 weights, float64 weight
    gradients, float64 inputs and outputs)"""
    from nope_nerf_b200 import ops, _lib as L
    rng = np.random.default_rng(1000 * D + M)
    P = O.init_params(seed=7 + D, D=D, hf_damp=True)
    flat = _cu(O.flatten_params(P))
    p = rng.uniform(-1.5, 1.5, (M, 3)).astype(np.float32)
    d = rng.normal(size=(M, 3)); d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    # a non-uniform cotangent on all four outputs: per-point magnitudes over three decades, no zeros
    g = (rng.normal(size=(M, 4)) * 10.0 ** rng.uniform(-2, 1, (M, 1))).astype(np.float32)
    p_c, d_c, g_c = _cu(p), (_cu(d) if with_dirs else None), _cu(g)
    flags = head_flags(head) | L.STASH
    ws = torch.empty(L.lib.nnb_workspace_bytes_dim(M, 1, flags, L.ENGINE_SIMT, D), dtype=torch.uint8, device="cuda")
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p_c); a.dirs = L.ptr(d_c); a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_SIMT
    a.hidden_dim = D; a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    out = torch.full((M, 4), float("nan"), device="cuda")
    gp = torch.full((M, 4), float("nan"), device="cuda"); gd = torch.full((M, 4), float("nan"), device="cuda")
    gw = torch.zeros(L.num_params(D), device="cuda")
    assert L.lib.nnb_field_fwd(C.byref(a), L.ptr(out), ops._stream()) == 0, L.lib.nnb_last_error()
    assert L.lib.nnb_field_bwd(C.byref(a), L.ptr(g_c), L.ptr(gp), L.ptr(gd), L.ptr(gw), ops._stream()) == 0, L.lib.nnb_last_error()
    torch.cuda.synchronize()
    lay = layout(M, 1, D)
    Mp, DR = lay["Mpad"], D // 2
    f = LL._f32
    st = {"h%d" % l: f(ws, lay["h"][l], Mp, D) for l in range(8)}
    st.update({"dy%d" % l: f(ws, lay["dy"][l], Mp, D) for l in range(8)})
    st.update(feat=f(ws, lay["feat"], Mp, D), hr=f(ws, lay["hr"], Mp, DR), enc=f(ws, lay["enc"], Mp, 64)[:, :63],
              denc=f(ws, lay["denc"], Mp, 32)[:, :27], rec=f(ws, lay["rec"], Mp, 8), dfeat=f(ws, lay["dfeat"], Mp, D),
              dyr=f(ws, lay["dyr"], Mp, DR), dyc=f(ws, lay["dyc"], Mp, 4), gs=f(ws, lay["gs"], Mp, 4), gp=f(ws, lay["gp"], Mp, 4),
              gv=f(ws, lay["gv"], Mp, 4))
    st = {k: v[:M].double() for k, v in st.items()}
    st["flags"] = flags
    G = {k: torch.from_numpy(v.astype(np.float64)).cuda() for k, v in O.unflatten_params(gw.cpu().numpy(), D).items()}
    W = {k: torch.from_numpy(np.asarray(v, np.float64)).cuda() for k, v in P.items()}
    dirs = d if with_dirs else np.ones_like(p)
    io = dict(p=_cu(p).double(), d=_cu(dirs).double(), g=g_c.double(), out=out.double(), gp=gp.double(), gd=gd.double())
    return st, W, G, io


def encadj_errors(st, W, D, io):
    """g_pts = encode_bwd<10>(p, dy0 W0 + dy4 W4[:, D:D+63]) and g_dirs = encode_bwd<4>(dirs, dyr W_rgbh[:, D:D+27]) from the kernel's
    dy stash (test_gpu_ray_local's encadj stage), with its wrong answers"""
    M = st["dy0"].shape[0]
    err, teeth = 0.0, {}
    W0, W4, Wd = W["layers0.0.weight"], W["layers1.0.weight"][:, D:D + 63], W["rgb_layers.0.weight"][:, D:D + 27]
    ge, gsc = LL.gemm_ref(torch.cat([st["dy0"], st["dy4"]], 1), torch.cat([W0, W4], 0).T.contiguous(), tiny=True)
    A = Arith(track=True)
    ref = encode_bwd_ref(A, io["p"], A.err(ge, gsc), 10)
    sc = scales(A, ref, M)
    got = io["gp"][:, :3]
    err = max(err, LL.nerr(got, ref.detach(), sc))
    A64 = Arith()
    teeth["octave"] = LL.nerr(got, encode_bwd_ref(A64, io["p"], ge, 10, "octave"), sc)
    teeth["no_layer4"] = LL.nerr(got, encode_bwd_ref(A64, io["p"], st["dy0"] @ W0, 10), sc)
    detect = dict(w0_lo=LL.nerr(got, encode_bwd_ref(A64, io["p"], st["dy0"] @ LL.bf16_hi(W0) + st["dy4"] @ W4, 10), sc))
    gev, gvsc = LL.gemm_ref(st["dyr"], Wd.T.contiguous(), tiny=True)
    A = Arith(track=True)
    ref = encode_bwd_ref(A, io["d"], A.err(gev, gvsc), 4)
    sc = scales(A, ref, M)
    got = io["gd"][:, :3]
    err = max(err, LL.nerr(got, ref.detach(), sc))
    teeth["octave"] = min(teeth["octave"], LL.nerr(got, encode_bwd_ref(A64, io["d"], gev, 4, "octave"), sc))
    return dict(err=err, teeth=teeth, detect=detect)


def enc_errors(st, io):
    """the stash's encodings of the kernel's inputs: x itself exactly, sin / cos within encode_ref's scale"""
    err = 0.0
    for key, x, levels in (("enc", io["p"], 10), ("denc", io["d"], 4)):
        assert torch.equal(st[key][:, :3], x), key
        ref, sc = encode_ref(x, levels)
        err = max(err, LL.nerr(st[key], ref, sc))
    return dict(err=err, teeth={})


def measure(D, M, head, with_dirs):
    st, W, G, io = run(D, M, head, with_dirs)
    # the call's outputs are the stash's values, and its cotangent the stash's gs
    assert torch.equal(io["out"], st["rec"][:, :4]), "out_rgba differs from the records"
    assert torch.equal(st["gs"], io["g"]), "the stash's cotangent differs from g_rgba"
    assert torch.equal(io["gp"][:, :3], st["gp"][:, :3]) and torch.equal(io["gd"][:, :3], st["gv"][:, :3])
    out = dict(enc=enc_errors(st, io), fwd=LL.forward_errors(st, W, D, False), dgrad=LL.dgrad_errors(st, W, D),
               wgrad=LL.wgrad_errors(st, G, D), encadj=encadj_errors(st, W, D, io))
    # the direction slice of rgb_layers.0's weight gradient dropped
    y, sc = LL.gemm_ref(st["dyr"].T.contiguous(), st["denc"].T.contiguous(), tiny=True)
    out["wgrad"]["teeth"]["no_dir_slice"] = LL.nerr(G["rgb_layers.0.weight"][:, D:D + 27], torch.zeros_like(y), sc)
    return out


GATES = dict(LL.SIMT_GATES, enc=SIMT_GATES["enc"], encadj=SIMT_GATES["encadj"])


@pytest.mark.gpu
@pytest.mark.parametrize("with_dirs", (True, False), ids=("dirs", "nodirs"))
@pytest.mark.parametrize("head", HEADS)
@pytest.mark.parametrize("M", SIZES)
@pytest.mark.parametrize("D", DIMS)
def test_field_layer_local(D, M, head, with_dirs):
    key = ("field", D, M, head, with_dirs)
    out = measure(D, M, head, with_dirs)
    LL._report(key, out)
    print("  detect", out["encadj"]["detect"])
    LL._check(key, out, GATES)
    for kind, t in out["encadj"]["detect"].items():
        assert t >= GATES["encadj"], (key, "encadj", "wrong answer '%s' within the gate" % kind, t)
    if head != "logit":
        assert {"head_factor", "head_slope"} <= set(out["dgrad"]["teeth"])
    assert "no_dir_slice" in out["wgrad"]["teeth"]


# ------------------------------------------------------------------------------------------------------------------------- host
@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("M", SIZES)
def test_field_layout_mirror(M, D):
    """layout(M, 1, D) is the exact engine's explicit-point workspace: nnb_field_bwd's make_layout(M, 1, flags, NNB_ENGINE_SIMT, D),
    for every head flag (they do not change the layout); the stash offsets against nnb_debug_layout (D = 256)"""
    from nope_nerf_b200 import _lib as L
    lay = layout(M, 1, D)
    for head in HEADS:
        assert L.lib.nnb_workspace_bytes_dim(M, 1, head_flags(head) | L.STASH, L.ENGINE_SIMT, D) == lay["gates"], head
    if D == 256:
        out = (C.c_size_t * 14)()
        assert L.lib.nnb_debug_layout(C.c_int32(M), C.c_int32(1), C.c_uint32(L.STASH), C.c_int32(L.ENGINE_SIMT), out) == 0
        assert list(out) == [lay["rec"]] + lay["h"] + [lay["feat"], lay["hr"], lay["enc"], lay["denc"], lay["gates"]]

"""GPU: the render and field calls read no workspace byte they did not write.

Each call below runs three times on a workspace the test allocates itself (not RenderCall's pool), filled first with zeros, with bytes
0xFF (NaN in every float) and with the words 0x7E7E7E7E (8.5e37, large and finite).  Every output and gradient must be finite and the
same bits in the three runs.  A kernel that read uninitialised workspace, for example the padding rows [M, Mpad) of a ragged size,
would give other bits, or NaN, whenever the caching allocator hands back dirty memory.
  nnb_render_fwd + nnb_render_bwd, both engines, D = 64 and 256, N x S in {5 x 32, 301 x 17, 9 x 1023, 1024 x 128}: rgb, depth_pred,
    depth_gt, mask, z_vals, alpha; g_weights, g_c2w, g_cam, g_depth, g_scale_shift.
  nnb_field_fwd (NNB_STASH) + nnb_field_bwd on the exact engine with weight gradients, M in {1, 65, 5117}: out_rgba, g_pts, g_dirs,
    g_weights.
  nnb_field_hvp, M in {1, 65, 5117}: g_pts, g_weights.
These workspaces hold floats, fp16 / bf16 weight images and ReLU gate bits only (make_layout, nnb_workspace.cuh), so no fill can make
a kernel index memory with a poisoned value."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu

FILLS = {"zeros": 0x00000000, "nan": -1, "big": 0x7E7E7E7E}   # int32 words: 0xFFFFFFFF is -1
RENDER_SIZES = ((5, 32), (301, 17), (9, 1023), (1024, 128))
FIELD_SIZES = (1, 65, 5117)
DIMS = (64, 256)


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _workspace(nbytes, word):
    ws = torch.empty((max(nbytes, 256) + 255) // 256 * 256, dtype=torch.uint8, device="cuda")
    ws.view(torch.int32).fill_(word)
    return ws


def _render(engine, D, N, S, word):
    """one forward + backward with every output and gradient requested; returns {name: CPU tensor}"""
    from nope_nerf_b200 import ops, _lib as L
    rng = np.random.default_rng(31)
    H, W = 48, 64
    flat = _cu(O.flatten_params(O.init_params(seed=5, D=D)))
    c2w = torch.empty(4, 4, device="cuda")
    ops.pose_fwd_raw(_cu(rng.normal(0, .05, (2, 3)).astype(np.float32)), _cu(rng.normal(0, .05, (2, 3)).astype(np.float32)), None, 1, c2w)
    cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0])).cuda()
    ray_idx = _cu(rng.permutation(H * W)[:N])
    dmap = _cu(rng.uniform(.6, 7.2, (24, 32)).astype(np.float32))
    scale, shift = torch.tensor([1.05]).cuda(), torch.tensor([0.02]).cuda()
    noise = _cu(rng.uniform(0, 1, (N, S)).astype(np.float32))
    flags = ops.flags_from_cfg(dict(O.DEFAULT_CFG), "softplus") | L.STASH
    nan = lambda *shape: torch.full(shape, float("nan"), device="cuda")
    out = dict(rgb=nan(N, 3), depth_pred=nan(N), depth_gt=nan(N), mask=torch.full((N,), 0xAB, dtype=torch.uint8, device="cuda"),
               z_vals=nan(N, S), alpha=nan(N, S))
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.c2w = L.ptr(c2w); a.cam = L.ptr(cam); a.ray_idx = L.ptr(ray_idx); a.depth_map = L.ptr(dmap)
    a.h_d, a.w_d = 24, 32
    a.scale = L.ptr(scale); a.shift = L.ptr(shift); a.noise = L.ptr(noise)
    a.N, a.S, a.H, a.W = N, S, H, W
    a.near_, a.far_ = 0.01, 10.0
    a.flags = flags; a.engine = engine; a.hidden_dim = D
    for k, v in out.items():
        setattr(a, k, L.ptr(v))
    ws = _workspace(L.lib.nnb_workspace_bytes_dim(N, S, flags, engine, D), word)
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    assert L.lib.nnb_render_fwd(C.byref(a), ops._stream()) == 0, L.lib.nnb_last_error()
    seeds = [_cu(rng.normal(0, 1, shape).astype(np.float32)) for shape in ((N, 3), (N,), (N,))]
    grads = dict(g_weights=torch.zeros(L.num_params(D), device="cuda"), g_c2w=torch.zeros(4, 4, device="cuda"),
                 g_cam=torch.zeros(4, 4, device="cuda"), g_depth=nan(N), g_scale_shift=torch.zeros(2, device="cuda"))
    b = L.RenderBwdArgs()
    b.fwd = a
    b.g_rgb, b.g_depth_pred, b.g_depth_gt = (L.ptr(s) for s in seeds)
    for k, v in grads.items():
        setattr(b, k, L.ptr(v))
    assert L.lib.nnb_render_bwd(C.byref(b), ops._stream()) == 0, L.lib.nnb_last_error()
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in dict(out, **grads).items()}


def _field_inputs(D, M):
    rng = np.random.default_rng(5 + M)
    flat = _cu(O.flatten_params(O.init_params(seed=7 + D, D=D, hf_damp=True)))
    p = _cu(rng.uniform(-1.5, 1.5, (M, 3)).astype(np.float32))
    d = rng.normal(size=(M, 3))
    d = _cu((d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32))
    g = _cu(rng.normal(size=(M, 4)).astype(np.float32))
    return flat, p, d, g


def _field_args(L, flat, p, d, M, D, flags, ws):
    a = L.RenderArgs()
    a.weights = L.ptr(flat); a.pts = L.ptr(p); a.dirs = L.ptr(d); a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_SIMT
    a.hidden_dim = D; a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    return a


def _field(D, M, word):
    """nnb_field_fwd (NNB_STASH) + nnb_field_bwd with weight gradients on the exact engine"""
    from nope_nerf_b200 import ops, _lib as L
    flat, p, d, g = _field_inputs(D, M)
    flags = L.SOFTPLUS | L.STASH
    ws = _workspace(L.lib.nnb_workspace_bytes_dim(M, 1, flags, L.ENGINE_SIMT, D), word)
    a = _field_args(L, flat, p, d, M, D, flags, ws)
    out = dict(out=torch.full((M, 4), float("nan"), device="cuda"), g_pts=torch.full((M, 4), float("nan"), device="cuda"),
               g_dirs=torch.full((M, 4), float("nan"), device="cuda"), g_weights=torch.zeros(L.num_params(D), device="cuda"))
    assert L.lib.nnb_field_fwd(C.byref(a), L.ptr(out["out"]), ops._stream()) == 0, L.lib.nnb_last_error()
    assert L.lib.nnb_field_bwd(C.byref(a), L.ptr(g), L.ptr(out["g_pts"]), L.ptr(out["g_dirs"]), L.ptr(out["g_weights"]),
                               ops._stream()) == 0, L.lib.nnb_last_error()
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


def _hvp(D, M, word):
    from nope_nerf_b200 import ops, _lib as L
    flat, p, d, g = _field_inputs(D, M)
    u = g.clone(); u[:, 3] = 0
    flags = L.SOFTPLUS | L.STASH | L.HVP
    ws = _workspace(L.lib.nnb_workspace_bytes_dim(M, 1, flags, L.ENGINE_SIMT, D), word)
    a = _field_args(L, flat, p, None, M, D, flags, ws)
    out = dict(g_pts=torch.full((M, 4), float("nan"), device="cuda"), g_weights=torch.zeros(L.num_params(D), device="cuda"))
    assert L.lib.nnb_field_hvp(C.byref(a), L.ptr(u), L.ptr(out["g_pts"]), L.ptr(out["g_weights"]), ops._stream()) == 0, \
        L.lib.nnb_last_error()
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


def _same_bits(key, runs, xyz_only=()):
    """every run's outputs finite and bit-identical to the zero-filled run's"""
    ref = runs["zeros"]
    for k, v in ref.items():
        if k in xyz_only:   # [M, 4] arrays of which the library defines xyz
            v = v[:, :3].contiguous()
        if v.is_floating_point():
            assert (v != 0).any(), (key, k, "nothing written")
        for fill, out in runs.items():
            w = out[k][:, :3].contiguous() if k in xyz_only else out[k]
            if v.is_floating_point():
                assert torch.isfinite(w).all(), (key, k, fill, "non-finite")
                same = torch.equal(v.view(torch.int32), w.view(torch.int32))
            else:
                same = torch.equal(v, w)
            assert same, (key, k, fill, "differs from the zero-filled workspace's run", float((v.double() - w.double()).abs().max()))


@pytest.mark.parametrize("engine", ("tc", "simt"))
@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("N,S", RENDER_SIZES)
def test_render_poisoned_workspace(engine, D, N, S):
    from nope_nerf_b200 import _lib as L
    e = L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT
    _same_bits((engine, D, N, S), {f: _render(e, D, N, S, w) for f, w in FILLS.items()})


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("M", FIELD_SIZES)
def test_field_bwd_poisoned_workspace(D, M):
    _same_bits(("field", D, M), {f: _field(D, M, w) for f, w in FILLS.items()}, xyz_only=("g_pts", "g_dirs"))


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("M", FIELD_SIZES)
def test_field_hvp_poisoned_workspace(D, M):
    _same_bits(("hvp", D, M), {f: _hvp(D, M, w) for f, w in FILLS.items()}, xyz_only=("g_pts",))

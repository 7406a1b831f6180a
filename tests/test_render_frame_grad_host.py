"""Host side of nnb_render_frame_bwd (the differentiable volumetric frame): the workspace rule (only the checkpoints grow with S), every
documented error code (returned before anything is launched), the ctypes bindings and the Python surface.  Needs no device."""
import ctypes as C

import pytest
import torch

from nope_nerf_b200 import _lib as L


def _align(x, a=256):
    return (x + a - 1) // a * a


def expected_bytes(N, S, D):
    """the documented layout: nnb_render_frame's workspace | checkpoints [ceil(S / 32) - 1][N] | suffix carries [N] | ray lane partials
    [N][9][32] | the chunk stash (nnb_workspace_bytes_dim(N, 32, NNB_STASH, NNB_ENGINE_TC) without its two weight images) | the transposed
    weight image, each 256-byte aligned"""
    ks = D // 16
    img_t = 34 * D * D + 576 * D
    stage = 64 * D
    img = (4 + 3 * ks + (4 + ks) + 3 * ks + ks + ks - ks) * stage + ks * stage // 2
    chunk = L.lib.nnb_workspace_bytes_dim(N, 32, L.STASH, L.ENGINE_TC, D) - _align(img) - _align(img_t)
    return (L.lib.nnb_render_frame_workspace_bytes(N, S, D) + _align(4 * N * ((S + 31) // 32 - 1)) + _align(4 * N) + _align(1152 * N)
            + chunk + _align(img_t))


def test_workspace_matches_its_formula():
    for N in (1, 3, 5, 127, 4096, 100000):
        for S in (16, 17, 32, 33, 128, 512, 1000, 1024):
            for D in L.HIDDEN_DIMS:
                assert L.lib.nnb_render_frame_bwd_workspace_bytes(N, S, D) == expected_bytes(N, S, D), (N, S, D)


def test_only_the_checkpoints_grow_with_S():
    N = 4096
    base = L.lib.nnb_render_frame_bwd_workspace_bytes(N, 32, 256)
    for S in (128, 512, 1024):
        grow = L.lib.nnb_render_frame_bwd_workspace_bytes(N, S, 256) - base
        assert grow == _align(4 * N * ((S + 31) // 32 - 1)), S
        assert grow <= 4 * N * (S // 32)
    assert L.lib.nnb_render_frame_bwd_workspace_bytes(N, 1024, 256) < L.lib.nnb_workspace_bytes_dim(N, 1024, L.STASH, L.ENGINE_TC, 256) // 30


def test_workspace_query_rejects_bad_sizes_and_widths():
    for D in (1, 96, 512):
        assert L.lib.nnb_render_frame_bwd_workspace_bytes(1000, 128, D) == 0
    for N, S in ((0, 128), (-1, 128), (1000, 15), (1000, 2), (1000, 1025)):
        assert L.lib.nnb_render_frame_bwd_workspace_bytes(N, S, 256) == 0


def _rc(**over):
    b = L.RenderBwdArgs()
    a = b.fwd
    a.weights, a.c2w, a.cam, a.ray_idx, a.depth_map = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000
    a.rgb, a.depth_pred, a.depth_gt, a.mask = 0x60000, 0x70000, 0x80000, 0x90000
    a.N, a.S, a.H, a.W, a.h_d, a.w_d = 1000, 128, 25, 40, 1, 1
    a.near_, a.far_ = 0.0, 1.0
    a.flags = L.SOFTPLUS; a.engine = L.ENGINE_TC; a.hidden_dim = 256
    a.workspace = 0x100000; a.workspace_bytes = 0
    b.g_rgb, b.g_c2w = 0xd0000, 0xe0000
    for k, v in over.items():
        setattr(b if k.startswith("g_") else a, k, v)
    return L.lib.nnb_render_frame_bwd(C.byref(b), None)


def test_every_documented_error_code():
    assert L.lib.nnb_render_frame_bwd(None, None) == -1
    assert _rc(engine=L.ENGINE_SIMT) == -4 and _rc(engine=7) == -4
    assert _rc(flags=512) == -7
    for flag in (L.STASH, L.HVP, L.OCC_ONLY, L.RAW_DENSITY):
        assert _rc(flags=flag) == -6
    assert _rc(hidden_dim=96) == -8
    assert _rc(N=0) == -2 and _rc(S=1025) == -2 and _rc(S=15) == -4
    for k in ("noise", "z_vals", "alpha", "pts", "dirs"):
        assert _rc(**{k: 0xa0000}) == -6, k
    for k in ("weights", "c2w", "cam", "rgb", "mask"):
        assert _rc(**{k: None}) == -3, k
    assert _rc(g_rgb=None) == -3 and _rc(g_c2w=None) == -3
    assert _rc() == -5
    need = L.lib.nnb_render_frame_bwd_workspace_bytes(1000, 128, 256)
    assert _rc(workspace_bytes=need - 1) == -5
    assert _rc(workspace=0x100080, workspace_bytes=need) == -5


def test_bindings_and_python_surface():
    from nope_nerf_b200 import ops
    assert L.lib.nnb_render_frame_bwd.argtypes == [C.POINTER(L.RenderBwdArgs), C.c_void_p]
    assert L.lib.nnb_render_frame_bwd_workspace_bytes.restype is C.c_size_t
    eye = torch.eye(4)
    meta = dict(N=1, S=32, flags=0, engine=None, near=0, far=1)
    with pytest.raises(ValueError, match="noise"):
        ops.render_frame_grad(dict(meta, noise=eye), eye, eye, eye, None, None, None, [])
    with pytest.raises(ValueError, match="tensor-core"):
        ops.render_frame_grad(dict(meta, S=8), eye, eye, eye, None, None, None, [])
    with pytest.raises(ValueError, match="tensor-core"):
        ops.render_frame_grad(dict(meta, engine=L.ENGINE_SIMT), eye, eye, eye, None, None, None, [])


def test_renderer_option_is_off_by_default():
    import nope_nerf_b200.model as mdl
    from _cfg import default_cfg
    cfg = default_cfg()
    r = mdl.Renderer(mdl.OfficialStaticNerf(cfg), cfg["rendering"], device=torch.device("cpu"))
    assert r.frame_grad is False
    assert mdl.Renderer(mdl.OfficialStaticNerf(cfg), cfg["rendering"], device=torch.device("cpu"), frame_grad=True).frame_grad is True

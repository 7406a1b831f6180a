"""Host side of nnb_render_frame_train_fwd / nnb_render_frame_train_bwd (the differentiable frame as a forward / backward pair for
training): the ctypes bindings, every documented error code (returned before anything is launched), the ValueErrors of
FrameRenderCall and Trainer(frame_grad=True), and that both options are off by default.  Needs no device."""
import ctypes as C

import pytest
import torch

from nope_nerf_b200 import _lib as L


def test_bindings():
    assert L.lib.nnb_render_frame_train_fwd.argtypes == [C.POINTER(L.RenderArgs), C.c_void_p]
    assert L.lib.nnb_render_frame_train_bwd.argtypes == [C.POINTER(L.RenderBwdArgs), C.c_void_p]
    assert L.lib.nnb_render_frame_train_fwd.restype is C.c_int and L.lib.nnb_render_frame_train_bwd.restype is C.c_int
    assert L.lib.nnb_version() == 105


def _args(**over):
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
    return b


def _rc_fwd(**over):
    return L.lib.nnb_render_frame_train_fwd(C.byref(_args(**over).fwd), None)


def _rc_bwd(**over):
    return L.lib.nnb_render_frame_train_bwd(C.byref(_args(**over)), None)


@pytest.mark.parametrize("rc", [_rc_fwd, _rc_bwd], ids=["fwd", "bwd"])
def test_every_documented_error_code(rc):
    assert rc(engine=L.ENGINE_SIMT) == -4 and rc(engine=7) == -4
    assert rc(flags=512) == -7
    for flag in (L.STASH, L.HVP, L.OCC_ONLY, L.RAW_DENSITY):
        assert rc(flags=flag) == -6
    assert rc(hidden_dim=96) == -8
    assert rc(N=0) == -2 and rc(S=1025) == -2 and rc(S=15) == -4
    assert rc(noise=0xa0000) == -5          # jitter is accepted: the call reaches the workspace check
    assert rc(noise=0xa0000, flags=L.SOFTPLUS | L.NDC) == -5
    for k in ("z_vals", "alpha", "pts", "dirs"):
        assert rc(**{k: 0xa0000}) == -6, k
    for k in ("weights", "c2w", "cam", "rgb", "mask"):
        assert rc(**{k: None}) == -3, k
    assert rc() == -5
    need = L.lib.nnb_render_frame_bwd_workspace_bytes(1000, 128, 256)
    assert rc(workspace_bytes=need - 1) == -5
    assert rc(workspace=0x100080, workspace_bytes=need) == -5


def test_null_args_and_gradient_pointers():
    assert L.lib.nnb_render_frame_train_fwd(None, None) == -1
    assert L.lib.nnb_render_frame_train_bwd(None, None) == -1
    assert _rc_bwd(g_rgb=None) == -3 and _rc_bwd(g_c2w=None) == -3
    assert _rc_fwd(g_rgb=None) == -5 and _rc_fwd(g_c2w=None) == -5     # the forward takes no gradients


def test_one_call_frame_entries_keep_rejecting_noise():
    b = _args(noise=0xa0000)
    assert L.lib.nnb_render_frame_bwd(C.byref(b), None) == -6
    f = L.FrameArgs()
    f.fwd = b.fwd
    assert L.lib.nnb_render_frame(C.byref(f), None) == -6
    assert L.lib.nnb_render_frame_engine(C.byref(f), None) == -6


def test_frame_render_call_value_errors():
    """raised before any device check: the CPU tensors below would otherwise fail RenderCall's CUDA check"""
    from nope_nerf_b200 import ops
    eye = torch.eye(4)
    kw = dict(N=1, S=32, flags=0, near=0, far=1)
    assert issubclass(ops.FrameRenderCall, ops.RenderCall) and ops.FrameRenderCall.frame and not ops.RenderCall.frame
    with pytest.raises(ValueError, match="want_z_alpha"):
        ops.FrameRenderCall(eye, eye, eye, engine=None, want_z_alpha=True, **kw)
    with pytest.raises(ValueError, match="tensor-core"):
        ops.FrameRenderCall(eye, eye, eye, engine=L.ENGINE_SIMT, **kw)
    with pytest.raises(ValueError, match="tensor-core"):
        ops.FrameRenderCall(eye, eye, eye, engine=None, **dict(kw, S=8))
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.FrameRenderCall(eye, eye, eye, engine=None, **kw)
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.RenderCall(eye, eye, eye, engine=L.ENGINE_SIMT, want_z_alpha=True, **kw)


def _trainer(engine=None, S=128, **kw):
    import nope_nerf_b200.model as mdl
    from _cfg import default_cfg
    cfg = default_cfg()
    cfg["rendering"]["num_points"] = S
    dev = torch.device("cpu")
    rend = mdl.Renderer(mdl.OfficialStaticNerf(cfg), cfg["rendering"], device=dev)
    rend.engine = engine
    model = mdl.get_model(rend, cfg, device=dev)
    return mdl.Trainer(model, torch.optim.Adam(model.parameters(), lr=1e-3), cfg["training"], device=dev, **kw)


def test_trainer_option(monkeypatch):
    from nope_nerf_b200 import ops
    monkeypatch.setattr(ops, "_DEFAULT_ENGINE", [L.ENGINE_TC])
    assert _trainer().frame_grad is False
    assert _trainer(frame_grad=True).frame_grad is True
    assert _trainer(engine=L.ENGINE_TC, S=16, frame_grad=True).frame_grad is True
    with pytest.raises(ValueError, match="tensor-core"):
        _trainer(S=8, frame_grad=True)
    with pytest.raises(ValueError, match="tensor-core"):
        _trainer(engine=L.ENGINE_SIMT, frame_grad=True)
    assert _trainer(engine=L.ENGINE_SIMT).frame_grad is False
    monkeypatch.setattr(ops, "_DEFAULT_ENGINE", [L.ENGINE_SIMT])
    with pytest.raises(ValueError, match="tensor-core"):
        _trainer(frame_grad=True)

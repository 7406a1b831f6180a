"""Host side of nnb_render_frame_train_fwd_tmin / nnb_render_frame_train_bwd_tmin (the frame's training pair with early ray termination):
the ctypes bindings, the argument checks (returned before anything is launched), ops.frame_render_call and its caching, the Trainer's
frame_grad_t_min validation, and that RenderCall's signature is unchanged.  Needs no device."""
import ctypes as C
import inspect
import math

import pytest
import torch

from nope_nerf_b200 import _lib as L


def test_bindings():
    for name in ("nnb_render_frame_train_fwd_tmin", "nnb_render_frame_train_bwd_tmin"):
        assert name in L.EXPORTS and hasattr(L.lib, name), name
    assert L.lib.nnb_render_frame_train_fwd_tmin.argtypes == [C.POINTER(L.FrameArgs), C.c_void_p]
    assert L.lib.nnb_render_frame_train_bwd_tmin.argtypes == [C.POINTER(L.RenderBwdArgs), C.c_void_p]
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
        if k not in ("t_min", "n_eval", "t_final"):
            setattr(b if k.startswith("g_") else a, k, v)
    return b


def _rc_fwd(**over):
    f = L.FrameArgs()
    f.fwd = _args(**over).fwd
    f.t_min = over.get("t_min", 1e-4)
    f.n_eval = over.get("n_eval", None); f.t_final = over.get("t_final", None)
    return L.lib.nnb_render_frame_train_fwd_tmin(C.byref(f), None)


def _rc_bwd(**over):
    return L.lib.nnb_render_frame_train_bwd_tmin(C.byref(_args(**over)), None)


@pytest.mark.parametrize("rc", [_rc_fwd, _rc_bwd], ids=["fwd", "bwd"])
def test_argument_checks(rc):
    assert rc(engine=L.ENGINE_SIMT) == -4 and rc(engine=7) == -4
    assert rc(flags=512) == -7
    for flag in (L.STASH, L.HVP, L.OCC_ONLY, L.RAW_DENSITY):
        assert rc(flags=flag) == -6
    assert rc(hidden_dim=96) == -8
    assert rc(N=0) == -2 and rc(S=1025) == -2 and rc(S=15) == -4
    assert rc(noise=0xa0000) == -5          # jitter is accepted: the call reaches the workspace check
    for k in ("z_vals", "alpha", "pts", "dirs"):
        assert rc(**{k: 0xa0000}) == -6, k
    for k in ("weights", "c2w", "cam", "rgb", "mask"):
        assert rc(**{k: None}) == -3, k
    assert rc() == -5
    need = L.lib.nnb_render_frame_bwd_workspace_bytes(1000, 128, 256)
    assert rc(workspace_bytes=need - 1) == -5
    assert rc(workspace=0x100080, workspace_bytes=need) == -5


def test_t_min_and_stats_checks():
    assert _rc_fwd(t_min=-1e-4) == -2 and _rc_fwd(t_min=float("nan")) == -2 and _rc_fwd(t_min=-math.inf) == -2
    assert _rc_fwd(t_min=0.0) == -5 and _rc_fwd(t_min=math.inf) == -5      # both reach the workspace check
    assert _rc_fwd(t_min=-1.0, engine=L.ENGINE_SIMT) == -4                  # the engine is checked first
    assert _rc_fwd(t_min=-1.0, flags=L.STASH) == -6                         # then the flags, then t_min
    assert _rc_fwd(t_min=-1.0, weights=None) == -2                          # t_min before the pointers
    assert _rc_fwd(n_eval=0xa0002) == -3 and _rc_fwd(t_final=0xa0001) == -3
    assert _rc_fwd(n_eval=0xa0000, t_final=0xb0000) == -5


def test_null_args_and_gradient_pointers():
    assert L.lib.nnb_render_frame_train_fwd_tmin(None, None) == -1
    assert L.lib.nnb_render_frame_train_bwd_tmin(None, None) == -1
    assert _rc_bwd(g_rgb=None) == -3 and _rc_bwd(g_c2w=None) == -3
    assert _rc_fwd(g_rgb=None) == -5 and _rc_fwd(g_c2w=None) == -5     # the forward takes no gradients


def test_frame_render_call_caching_and_values():
    from nope_nerf_b200 import ops
    assert ops.FrameRenderCall.t_min is None and ops.RenderCall.t_min is None and ops.ExactFrameRenderCall.t_min is None
    c = ops.frame_render_call(1e-4)
    assert c is ops.frame_render_call(1e-4) and c is ops.frame_render_call(float(C.c_float(1e-4).value))
    assert issubclass(c, ops.FrameRenderCall) and c.frame and not c.exact_frame
    assert c.t_min == C.c_float(1e-4).value
    z = ops.frame_render_call(0.0)
    assert z is ops.frame_render_call(0) and z is not c and z.t_min == 0.0
    for bad in (-1e-4, float("nan"), -math.inf):
        with pytest.raises(ValueError, match="t_min"):
            ops.frame_render_call(bad)
    eye = torch.eye(4)
    kw = dict(N=1, S=32, flags=0, near=0, far=1)
    with pytest.raises(ValueError, match="tensor-core"):   # FrameRenderCall's checks, before any device check
        c(eye, eye, eye, engine=L.ENGINE_SIMT, **kw)
    with pytest.raises(ValueError, match="want_z_alpha"):
        c(eye, eye, eye, engine=None, want_z_alpha=True, **kw)
    with pytest.raises(RuntimeError, match="CUDA device"):
        c(eye, eye, eye, engine=None, **kw)


def test_render_call_signature_unchanged():
    from nope_nerf_b200 import ops
    params = list(inspect.signature(ops.RenderCall.__init__).parameters)
    assert params == ["self", "weights", "c2w", "cam", "N", "S", "flags", "engine", "near", "far", "ray_idx", "pixels", "depth",
                      "depth_map", "scale", "shift", "noise", "H", "W", "want_z_alpha", "stash", "hidden_dim"]
    assert inspect.signature(ops.frame_render_call(1e-4).__init__) == inspect.signature(ops.RenderCall.__init__)


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
    t = _trainer(frame_grad=True)
    assert t.frame_grad_t_min is None and t._train_render_call(True) is ops.FrameRenderCall
    for v in (1e-4, 0.0, 0):
        t = _trainer(frame_grad=True, frame_grad_t_min=v)
        assert t._train_render_call(True) is ops.frame_render_call(v) and t._train_render_call(False) is ops.RenderCall
    assert _trainer(frame_grad=True, frame_grad_engine="tc", frame_grad_t_min=1e-4)._train_render_call(True) is ops.frame_render_call(1e-4)
    with pytest.raises(ValueError, match="frame_grad=True"):
        _trainer(frame_grad_t_min=1e-4)
    with pytest.raises(ValueError, match="simt"):
        _trainer(frame_grad=True, frame_grad_engine="simt", frame_grad_t_min=1e-4)
    for bad in (-1e-4, float("nan")):
        with pytest.raises(ValueError, match="t_min"):
            _trainer(frame_grad=True, frame_grad_t_min=bad)
    with pytest.raises(ValueError, match="tensor-core"):
        _trainer(S=8, frame_grad=True, frame_grad_t_min=1e-4)

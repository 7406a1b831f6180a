"""Host side of the differentiable frame on the exact-fp32 engine (nnb_render_frame_bwd_engine, nnb_render_frame_train_fwd_engine /
_bwd_engine, nnb_render_frame_bwd_workspace_bytes_engine): the bindings, the workspace formula (a chunk stash of min(S, 32) rows per ray),
every documented error code (returned before anything is launched), and the ValueErrors and defaults of ExactFrameRenderCall,
render_frame_grad, Renderer and Trainer.  Needs no device."""
import ctypes as C
import inspect

import pytest
import torch

from nope_nerf_b200 import _lib as L

NEW = ("nnb_render_frame_bwd_workspace_bytes_engine", "nnb_render_frame_bwd_engine", "nnb_render_frame_train_fwd_engine",
       "nnb_render_frame_train_bwd_engine")


def _align(x, a=256):
    return (x + a - 1) // a * a


def expected_bytes(N, S, D):
    """frame_bwd_layout_bytes(N, S, 0, make_layout(N, min(S, 32), NNB_STASH, NNB_ENGINE_SIMT, D).total, 0): the exact frame's workspace
    | checkpoints [ceil(S / 32) - 1][N] | suffix carries [N] | ray lane partials [N][9][32] | the chunk stash, each 256-byte aligned"""
    chunk = L.lib.nnb_workspace_bytes_dim(N, min(S, 32), L.STASH, L.ENGINE_SIMT, D)
    return (L.lib.nnb_render_frame_workspace_bytes_engine(N, S, D, L.ENGINE_SIMT) + _align(4 * N * ((S + 31) // 32 - 1)) + _align(4 * N)
            + _align(1152 * N) + _align(chunk))


def test_bindings():
    for name in NEW:
        assert name in L.EXPORTS and hasattr(L.lib, name), name
    assert L.lib.nnb_render_frame_bwd_workspace_bytes_engine.restype is C.c_size_t
    assert L.lib.nnb_render_frame_bwd_workspace_bytes_engine.argtypes == [C.c_int32] * 4
    assert L.lib.nnb_render_frame_bwd_engine.argtypes == [C.POINTER(L.RenderBwdArgs), C.c_void_p]
    assert L.lib.nnb_render_frame_train_fwd_engine.argtypes == [C.POINTER(L.RenderArgs), C.c_void_p]
    assert L.lib.nnb_render_frame_train_bwd_engine.argtypes == [C.POINTER(L.RenderBwdArgs), C.c_void_p]
    assert L.lib.nnb_version() == 105


def test_workspace_matches_its_formula():
    ws = L.lib.nnb_render_frame_bwd_workspace_bytes_engine
    for N in (1, 3, 5, 127, 4096, 100000):
        for S in (2, 8, 15, 16, 31, 32, 33, 128, 1000, 1024):
            for D in L.HIDDEN_DIMS:
                assert ws(N, S, D, L.ENGINE_SIMT) == expected_bytes(N, S, D), (N, S, D)
                assert ws(N, S, D, L.ENGINE_TC) == L.lib.nnb_render_frame_bwd_workspace_bytes(N, S, D), (N, S, D)


def test_workspace_stays_flat_in_S_and_far_below_the_stash_path():
    ws = L.lib.nnb_render_frame_bwd_workspace_bytes_engine
    N = 4096
    base = ws(N, 32, 256, L.ENGINE_SIMT)
    for S in (128, 512, 1024):
        assert ws(N, S, 256, L.ENGINE_SIMT) - base == _align(4 * N * ((S + 31) // 32 - 1)), S
    assert ws(N, 1024, 256, L.ENGINE_SIMT) < L.lib.nnb_workspace_bytes_dim(N, 1024, L.STASH, L.ENGINE_SIMT, 256) // 30
    assert ws(N, 8, 256, L.ENGINE_SIMT) < ws(N, 32, 256, L.ENGINE_SIMT)   # packed rows: a ray keeps S rows below 32


def test_workspace_query_rejects_bad_sizes_widths_and_engines():
    ws = L.lib.nnb_render_frame_bwd_workspace_bytes_engine
    for D in (1, 96, 512):
        assert ws(1000, 128, D, L.ENGINE_SIMT) == 0
    for N, S in ((0, 128), (-1, 128), (1000, 1), (1000, 0), (1000, 1025)):
        assert ws(N, S, 256, L.ENGINE_SIMT) == 0, (N, S)
    assert ws(1000, 15, 256, L.ENGINE_TC) == 0 and ws(1000, 2, 256, L.ENGINE_TC) == 0
    for engine in (-1, 2, 7):
        assert ws(1000, 128, 256, engine) == 0


def _args(**over):
    b = L.RenderBwdArgs()
    a = b.fwd
    a.weights, a.c2w, a.cam, a.ray_idx, a.depth_map = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000
    a.rgb, a.depth_pred, a.depth_gt, a.mask = 0x60000, 0x70000, 0x80000, 0x90000
    a.N, a.S, a.H, a.W, a.h_d, a.w_d = 1000, 128, 25, 40, 1, 1
    a.near_, a.far_ = 0.0, 1.0
    a.flags = L.SOFTPLUS; a.engine = L.ENGINE_SIMT; a.hidden_dim = 256
    a.workspace = 0x100000; a.workspace_bytes = 0
    b.g_rgb, b.g_c2w = 0xd0000, 0xe0000
    for k, v in over.items():
        setattr(b if k.startswith("g_") else a, k, v)
    return b


def _rc_bwd1(**over):
    return L.lib.nnb_render_frame_bwd_engine(C.byref(_args(**over)), None)


def _rc_fwd(**over):
    return L.lib.nnb_render_frame_train_fwd_engine(C.byref(_args(**over).fwd), None)


def _rc_bwd(**over):
    return L.lib.nnb_render_frame_train_bwd_engine(C.byref(_args(**over)), None)


CALLS = [_rc_bwd1, _rc_fwd, _rc_bwd]


@pytest.mark.parametrize("rc", CALLS, ids=["bwd", "train_fwd", "train_bwd"])
def test_every_documented_error_code(rc):
    assert rc(engine=7) == -4 and rc(engine=-1) == -4
    assert rc(flags=512) == -7
    for flag in (L.STASH, L.HVP, L.OCC_ONLY, L.RAW_DENSITY):
        assert rc(flags=flag) == -6
    assert rc(hidden_dim=96) == -8
    assert rc(N=0) == -2 and rc(S=1025) == -2 and rc(S=1) == -2
    for S in (2, 8, 15, 31, 33, 1024):                # the exact engine takes any S from 2: the call reaches the workspace check
        assert rc(S=S) == -5, S
    assert rc(engine=L.ENGINE_TC, S=15) == -4      # the tensor-core form keeps its range
    for k in ("z_vals", "alpha", "pts", "dirs"):
        assert rc(**{k: 0xa0000}) == -6, k
    for k in ("weights", "c2w", "cam", "rgb", "mask"):
        assert rc(**{k: None}) == -3, k
    assert rc() == -5
    for S in (8, 128):
        need = L.lib.nnb_render_frame_bwd_workspace_bytes_engine(1000, S, 256, L.ENGINE_SIMT)
        assert rc(S=S, workspace_bytes=need - 1) == -5
        assert rc(S=S, workspace=0x100080, workspace_bytes=need) == -5
        assert rc(S=S, workspace=None, workspace_bytes=need) == -5


def test_null_args_noise_and_gradient_pointers():
    assert L.lib.nnb_render_frame_bwd_engine(None, None) == -1
    assert L.lib.nnb_render_frame_train_fwd_engine(None, None) == -1
    assert L.lib.nnb_render_frame_train_bwd_engine(None, None) == -1
    for engine in (L.ENGINE_SIMT, L.ENGINE_TC):
        assert _rc_bwd1(engine=engine, noise=0xa0000) == -6        # the one-call backward takes no jitter
        assert _rc_fwd(engine=engine, noise=0xa0000) == -5         # the pair does: it reaches the workspace check
        assert _rc_bwd(engine=engine, noise=0xa0000) == -5
        for rc in (_rc_bwd1, _rc_bwd):
            assert rc(engine=engine, g_rgb=None) == -3 and rc(engine=engine, g_c2w=None) == -3
        assert _rc_fwd(engine=engine, g_rgb=None) == -5 and _rc_fwd(engine=engine, g_c2w=None) == -5


def test_calls_without_the_suffix_keep_their_contracts():
    b = _args(engine=L.ENGINE_SIMT)
    assert L.lib.nnb_render_frame_bwd(C.byref(b), None) == -4
    assert L.lib.nnb_render_frame_train_fwd(C.byref(b.fwd), None) == -4
    assert L.lib.nnb_render_frame_train_bwd(C.byref(b), None) == -4
    b = _args(engine=L.ENGINE_TC, S=15)
    assert L.lib.nnb_render_frame_bwd(C.byref(b), None) == -4
    assert L.lib.nnb_render_frame_bwd_workspace_bytes(1000, 15, 256) == 0


def test_exact_frame_render_call_value_errors():
    """raised before any device check: the CPU tensors below would otherwise fail RenderCall's CUDA check"""
    from nope_nerf_b200 import ops
    eye = torch.eye(4)
    kw = dict(N=1, S=32, flags=0, near=0, far=1)
    assert issubclass(ops.ExactFrameRenderCall, ops.FrameRenderCall)
    assert ops.ExactFrameRenderCall.exact_frame and not ops.FrameRenderCall.exact_frame and not ops.RenderCall.exact_frame
    with pytest.raises(ValueError, match="want_z_alpha"):
        ops.ExactFrameRenderCall(eye, eye, eye, engine=None, want_z_alpha=True, **kw)
    for S in (1, 1025):
        with pytest.raises(ValueError, match="2 <= S <= 1024"):
            ops.ExactFrameRenderCall(eye, eye, eye, engine=None, **dict(kw, S=S))
    for engine, S in ((None, 32), (L.ENGINE_TC, 8), (L.ENGINE_SIMT, 2), (L.ENGINE_TC, 1024)):   # any engine, any S in range
        with pytest.raises(RuntimeError, match="CUDA device"):
            ops.ExactFrameRenderCall(eye, eye, eye, engine=engine, **dict(kw, S=S))
    # the tensor-core class keeps its rule
    with pytest.raises(ValueError, match="tensor-core"):
        ops.FrameRenderCall(eye, eye, eye, engine=L.ENGINE_SIMT, **kw)
    with pytest.raises(ValueError, match="tensor-core"):
        ops.FrameRenderCall(eye, eye, eye, engine=None, **dict(kw, S=8))


def test_render_frame_grad_and_bwd_surface():
    from nope_nerf_b200 import ops
    assert inspect.signature(ops.render_frame_grad).parameters["frame_engine"].default is None
    assert inspect.signature(ops.render_frame_bwd).parameters["engine"].default == L.ENGINE_TC
    eye = torch.eye(4)
    meta = dict(N=1, S=32, flags=0, engine=None, near=0, far=1)
    with pytest.raises(ValueError, match="noise"):
        ops.render_frame_grad(dict(meta, noise=eye), eye, eye, eye, None, None, None, [], frame_engine=L.ENGINE_SIMT)
    for S in (1, 1025):
        with pytest.raises(ValueError, match="2 <= S <= 1024"):
            ops.render_frame_grad(dict(meta, S=S), eye, eye, eye, None, None, None, [], frame_engine=L.ENGINE_SIMT)
    with pytest.raises(ValueError, match="frame_engine"):
        ops.render_frame_grad(meta, eye, eye, eye, None, None, None, [], frame_engine=7)
    for fe in (None, L.ENGINE_TC):   # the tensor-core rule is unchanged
        with pytest.raises(ValueError, match="tensor-core"):
            ops.render_frame_grad(dict(meta, S=8), eye, eye, eye, None, None, None, [], frame_engine=fe)


def _renderer(**kw):
    import nope_nerf_b200.model as mdl
    from _cfg import default_cfg
    cfg = default_cfg()
    return mdl.Renderer(mdl.OfficialStaticNerf(cfg), cfg["rendering"], device=torch.device("cpu"), **kw)


def test_renderer_option():
    assert _renderer().frame_grad_engine is None
    assert _renderer(frame_grad=True).frame_grad_engine is None
    for v in ("tc", "simt"):
        assert _renderer(frame_grad=True, frame_grad_engine=v).frame_grad_engine == v
        with pytest.raises(ValueError, match="frame_grad=True"):
            _renderer(frame_grad_engine=v)
    for v in ("exact", 1, "SIMT"):
        with pytest.raises(ValueError, match="frame_grad_engine"):
            _renderer(frame_grad=True, frame_grad_engine=v)


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
    t = _trainer()
    assert t.frame_grad_engine is None and t._train_render_call(True) is ops.RenderCall
    t = _trainer(frame_grad=True)
    assert t._train_render_call(True) is ops.FrameRenderCall and t._train_render_call(False) is ops.RenderCall
    for engine, S in ((None, 128), (L.ENGINE_SIMT, 128), (None, 8), (L.ENGINE_TC, 2), (L.ENGINE_SIMT, 1024)):
        t = _trainer(engine=engine, S=S, frame_grad=True, frame_grad_engine="simt")
        assert t.frame_grad_engine == "simt"
        assert t._train_render_call(True) is ops.ExactFrameRenderCall and t._train_render_call(False) is ops.RenderCall
    for S in (1, 1025):
        with pytest.raises(ValueError, match="num_points"):
            _trainer(S=S, frame_grad=True, frame_grad_engine="simt")
    assert _trainer(frame_grad=True, frame_grad_engine="tc")._train_render_call(True) is ops.FrameRenderCall
    with pytest.raises(ValueError, match="tensor-core"):
        _trainer(S=8, frame_grad=True, frame_grad_engine="tc")
    for v in ("tc", "simt"):
        with pytest.raises(ValueError, match="frame_grad=True"):
            _trainer(frame_grad_engine=v)
    with pytest.raises(ValueError, match="frame_grad_engine"):
        _trainer(frame_grad=True, frame_grad_engine="exact")

"""Host side of nnb_render_fwd_tmin_engine / nnb_render_bwd_tmin_engine / nnb_render_tmin_workspace_bytes_engine (training with early ray
termination on the per-sample stash, on either engine): the ctypes bindings, the argument checks and their order on both engines
(returned before anything is launched), the workspace query, ops.exact_stash_render_call and its caching, the Trainer's
train_t_min_engine validation and routing, and that every CUDA source still compiles for sm_90a.  Needs no device."""
import ctypes as C
import inspect
import math

import pytest
import torch

from nope_nerf_b200 import _lib as L
from test_render_frame_train_tmin_host import _args, _trainer
from test_render_tmin_host import test_every_source_compiles_for_sm90a as _compiles

NAMES = ("nnb_render_fwd_tmin_engine", "nnb_render_bwd_tmin_engine", "nnb_render_tmin_workspace_bytes_engine")


def test_bindings():
    for name in NAMES:
        assert name in L.EXPORTS and hasattr(L.lib, name), name
    assert L.lib.nnb_render_fwd_tmin_engine.argtypes == [C.POINTER(L.FrameArgs), C.c_void_p]
    assert L.lib.nnb_render_bwd_tmin_engine.argtypes == [C.POINTER(L.RenderBwdArgs), C.c_void_p]
    assert L.lib.nnb_render_tmin_workspace_bytes_engine.argtypes == [C.c_int32] * 4
    assert L.lib.nnb_render_tmin_workspace_bytes_engine.restype == C.c_size_t
    assert L.lib.nnb_version() == 105


def _rc_fwd(**over):
    f = L.FrameArgs()
    f.fwd = _args(**over).fwd
    f.t_min = over.get("t_min", 1e-4)
    f.n_eval = over.get("n_eval", None); f.t_final = over.get("t_final", None)
    return L.lib.nnb_render_fwd_tmin_engine(C.byref(f), None)


def _rc_bwd(**over):
    return L.lib.nnb_render_bwd_tmin_engine(C.byref(_args(**over)), None)


def _rc_fwd_plain(**over):
    f = L.FrameArgs()
    f.fwd = _args(**over).fwd
    f.t_min = over.get("t_min", 1e-4)
    f.n_eval = over.get("n_eval", None); f.t_final = over.get("t_final", None)
    return L.lib.nnb_render_fwd_tmin(C.byref(f), None)


def test_workspace_bytes():
    ws = L.lib.nnb_render_tmin_workspace_bytes_engine
    SIMT, TC = L.ENGINE_SIMT, L.ENGINE_TC
    for bad in ((0, 128, 256), (-1, 128, 256), (1000, 1, 256), (1000, 1025, 256), (1000, 128, 96), (1000, 0, 256)):
        assert ws(*bad, SIMT) == 0 and ws(*bad, TC) == 0, bad
    assert ws(1000, 128, 256, 7) == 0 and ws(1000, 128, 256, -1) == 0
    assert ws(1000, 15, 256, TC) == 0 and ws(1000, 15, 256, SIMT) > 0   # the exact engine takes S below 16
    for N, S, D in ((1000, 128, 256), (1, 16, 64), (4096, 512, 256), (1023, 33, 128), (5, 1024, 64)):
        assert ws(N, S, D, TC) == L.lib.nnb_render_tmin_workspace_bytes(N, S, D), (N, S, D)
    for N, S, D in ((1000, 128, 256), (1, 2, 64), (257, 8, 64), (301, 17, 128), (4096, 512, 256), (1023, 33, 128), (5, 1024, 64),
                    (1024, 32, 256)):
        stash = L.lib.nnb_workspace_bytes_dim(N, S, L.STASH, L.ENGINE_SIMT, D)
        assert ws(N, S, D, SIMT) >= stash > 0, (N, S, D)
    assert ws(1000, 128, 0, SIMT) == ws(1000, 128, 256, SIMT)
    assert ws(1001, 128, 256, SIMT) > ws(1000, 128, 256, SIMT) and ws(1000, 160, 256, SIMT) > ws(1000, 128, 256, SIMT)
    # no weight images: below the tensor-core pair's workspace
    assert ws(1000, 128, 256, SIMT) < ws(1000, 128, 256, TC)


@pytest.mark.parametrize("engine", ["tc", "simt"])
@pytest.mark.parametrize("rc", [_rc_fwd, _rc_bwd], ids=["fwd", "bwd"])
def test_argument_checks(rc, engine):
    e = L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT
    r = lambda **k: rc(**dict(dict(engine=e), **k))
    assert r(engine=7) == -4 and r(engine=-1) == -4
    assert r(flags=512) == -7
    for flag in (L.STASH, L.HVP, L.OCC_ONLY, L.RAW_DENSITY):
        assert r(flags=flag) == -6
    assert r(hidden_dim=96) == -8
    assert r(N=0) == -2 and r(S=1025) == -2 and r(S=1) == -2
    assert r(S=15) == (-4 if engine == "tc" else -5)   # the exact engine runs below 16 samples
    assert r(S=2) == (-4 if engine == "tc" else -5)
    assert r(noise=0xa0000) == -5          # jitter is accepted: the call reaches the workspace check
    for k in ("z_vals", "alpha", "pts", "dirs"):
        assert r(**{k: 0xa0000}) == -6, k
    for k in ("weights", "c2w", "cam", "rgb", "mask"):
        assert r(**{k: None}) == -3, k
    assert r() == -5
    need = L.lib.nnb_render_tmin_workspace_bytes_engine(1000, 128, 256, e)
    assert r(workspace_bytes=need - 1) == -5
    assert r(workspace=0x100080, workspace_bytes=need) == -5
    # the order of the checks: engine, flags, width, sizes, per-sample outputs, (t_min,) pointers, workspace
    assert r(engine=7, flags=512) == -4 and r(flags=512, hidden_dim=96) == -7
    assert r(hidden_dim=96, N=0) == -8 and r(N=0, z_vals=0xa0000) == -2 and r(z_vals=0xa0000, weights=None) == -6
    assert r(weights=None, workspace_bytes=0) == -3


def test_tc_engine_is_the_plain_call():
    """on NNB_ENGINE_TC every code is nnb_render_fwd_tmin's; the plain calls keep refusing NNB_ENGINE_SIMT"""
    cases = [dict(), dict(flags=512), dict(flags=L.STASH), dict(hidden_dim=96), dict(N=0), dict(S=15), dict(S=1025), dict(z_vals=0xa0000),
             dict(t_min=-1.0), dict(weights=None), dict(n_eval=0xa0002), dict(noise=0xa0000)]
    for over in cases:
        assert _rc_fwd(**over) == _rc_fwd_plain(**over), over
    assert _rc_fwd_plain(engine=L.ENGINE_SIMT) == -4
    assert L.lib.nnb_render_bwd_tmin(C.byref(_args(engine=L.ENGINE_SIMT)), None) == -4
    assert L.lib.nnb_render_tmin_workspace_bytes(1000, 8, 256) == 0


def test_t_min_and_stats_checks():
    S = dict(engine=L.ENGINE_SIMT)
    assert _rc_fwd(t_min=-1e-4, **S) == -2 and _rc_fwd(t_min=float("nan"), **S) == -2 and _rc_fwd(t_min=-math.inf, **S) == -2
    assert _rc_fwd(t_min=0.0, **S) == -5 and _rc_fwd(t_min=math.inf, **S) == -5      # both reach the workspace check
    assert _rc_fwd(t_min=-1.0, engine=7) == -4                                      # the engine is checked first
    assert _rc_fwd(t_min=-1.0, flags=L.STASH, **S) == -6                            # then the flags, then t_min
    assert _rc_fwd(t_min=-1.0, weights=None, **S) == -2                             # t_min before the pointers
    assert _rc_fwd(n_eval=0xa0002, **S) == -3 and _rc_fwd(t_final=0xa0001, **S) == -3
    assert _rc_fwd(n_eval=0xa0000, t_final=0xb0000, **S) == -5


def test_null_args_and_gradient_pointers():
    assert L.lib.nnb_render_fwd_tmin_engine(None, None) == -1
    assert L.lib.nnb_render_bwd_tmin_engine(None, None) == -1
    S = dict(engine=L.ENGINE_SIMT)
    assert _rc_bwd(g_rgb=None, **S) == -3 and _rc_bwd(g_c2w=None, **S) == -3
    assert _rc_bwd(g_weights=None, **S) == -5                                 # pose only: reaches the workspace check
    assert _rc_fwd(g_rgb=None, **S) == -5 and _rc_fwd(g_c2w=None, **S) == -5   # the forward takes no gradients


def test_exact_stash_render_call_caching_and_values():
    from nope_nerf_b200 import ops
    assert ops.RenderCall.exact_stash is False and ops.stash_render_call(1e-4).exact_stash is False
    c = ops.exact_stash_render_call(1e-4)
    assert c is ops.exact_stash_render_call(1e-4) and c is ops.exact_stash_render_call(float(C.c_float(1e-4).value))
    assert issubclass(c, ops.RenderCall) and not issubclass(c, ops.FrameRenderCall)
    assert c.exact_stash and c.stash_tmin and not c.frame and not c.exact_frame and c.t_min == C.c_float(1e-4).value
    assert c is not ops.stash_render_call(1e-4) and c is not ops.frame_render_call(1e-4)
    z = ops.exact_stash_render_call(0.0)
    assert z is ops.exact_stash_render_call(0) and z is not c and z.t_min == 0.0
    for bad in (-1e-4, float("nan"), -math.inf):
        with pytest.raises(ValueError, match="t_min"):
            ops.exact_stash_render_call(bad)
    assert inspect.signature(c.__init__) == inspect.signature(ops.RenderCall.__init__)
    eye = torch.eye(4)
    kw = dict(N=1, flags=0, near=0, far=1)
    for S in (1, 1025):   # checked before any device check
        with pytest.raises(ValueError, match="2 <= S <= 1024"):
            c(eye, eye, eye, engine=None, S=S, **kw)
    with pytest.raises(ValueError, match="want_z_alpha"):
        c(eye, eye, eye, engine=None, S=32, want_z_alpha=True, **kw)
    for engine, S in ((L.ENGINE_TC, 8), (L.ENGINE_SIMT, 128), (None, 2), (None, 1024)):   # any engine, any S in 2..1024
        with pytest.raises(RuntimeError, match="CUDA device"):
            c(eye, eye, eye, engine=engine, S=S, **kw)
    with pytest.raises(ValueError, match="tensor-core"):   # unchanged
        ops.stash_render_call(1e-4)(eye, eye, eye, engine=L.ENGINE_SIMT, S=32, **kw)


def test_trainer_option(monkeypatch):
    from nope_nerf_b200 import ops
    monkeypatch.setattr(ops, "_DEFAULT_ENGINE", [L.ENGINE_TC])
    t = _trainer()
    assert t.train_t_min_engine is None and t._train_render_call(True) is ops.RenderCall
    for v in (1e-4, 0.0, 0):
        for eng, cls in ((None, ops.stash_render_call(v)), ("tc", ops.stash_render_call(v)), ("simt", ops.exact_stash_render_call(v))):
            t = _trainer(train_t_min=v, train_t_min_engine=eng)
            assert t._train_render_call(True) is cls and t._train_render_call(False) is ops.RenderCall, (v, eng)
    # 'simt' at any num_points in 2..1024, whatever the renderer's engine
    for engine, S in ((L.ENGINE_SIMT, 128), (L.ENGINE_TC, 8), (None, 2), (None, 1024), (L.ENGINE_SIMT, 15)):
        t = _trainer(engine=engine, S=S, train_t_min=1e-4, train_t_min_engine="simt")
        assert t._train_render_call(True) is ops.exact_stash_render_call(1e-4)
    for S in (1, 1025):
        with pytest.raises(ValueError, match="2..1024"):
            _trainer(S=S, train_t_min=1e-4, train_t_min_engine="simt")
    # None / 'tc' keep the tensor-core requirement
    for eng in (None, "tc"):
        with pytest.raises(ValueError, match="tensor-core"):
            _trainer(engine=L.ENGINE_SIMT, train_t_min=1e-4, train_t_min_engine=eng)
        with pytest.raises(ValueError, match="tensor-core"):
            _trainer(S=8, train_t_min=1e-4, train_t_min_engine=eng)
    for bad in ("SIMT", "exact", 1, True):
        with pytest.raises(ValueError, match="train_t_min_engine"):
            _trainer(train_t_min=1e-4, train_t_min_engine=bad)
    for eng in ("tc", "simt"):
        with pytest.raises(ValueError, match="needs train_t_min"):
            _trainer(train_t_min_engine=eng)
        with pytest.raises(ValueError, match="frame_grad"):
            _trainer(frame_grad=True, train_t_min=1e-4, train_t_min_engine=eng)
        with pytest.raises(ValueError, match="frame_grad"):
            _trainer(frame_grad=True, frame_grad_engine="simt", train_t_min=1e-4, train_t_min_engine=eng)
    for bad in (-1e-4, float("nan")):
        with pytest.raises(ValueError, match="t_min"):
            _trainer(train_t_min=bad, train_t_min_engine="simt")
    with pytest.raises(ValueError, match="simt"):   # the frame pair at t > 0 stays on the tensor cores
        _trainer(frame_grad=True, frame_grad_engine="simt", frame_grad_t_min=1e-4)


def test_every_source_compiles_for_sm90a(tmp_path):
    _compiles(tmp_path)

"""Host side of nnb_render_fwd_tmin / nnb_render_bwd_tmin (training with early ray termination on the per-sample stash): the ctypes
bindings, the argument checks and their order (returned before anything is launched), the workspace query, ops.stash_render_call and its
caching, the Trainer's train_t_min validation, and that every CUDA source still compiles for sm_90a.  Needs no device."""
import ctypes as C
import inspect
import math
import os
import shutil
import subprocess

import pytest
import torch

from nope_nerf_b200 import _lib as L
from test_render_frame_train_tmin_host import _args, _trainer


def test_bindings():
    for name in ("nnb_render_fwd_tmin", "nnb_render_bwd_tmin", "nnb_render_tmin_workspace_bytes"):
        assert name in L.EXPORTS and hasattr(L.lib, name), name
    assert L.lib.nnb_render_fwd_tmin.argtypes == [C.POINTER(L.FrameArgs), C.c_void_p]
    assert L.lib.nnb_render_bwd_tmin.argtypes == [C.POINTER(L.RenderBwdArgs), C.c_void_p]
    assert L.lib.nnb_render_tmin_workspace_bytes.argtypes == [C.c_int32, C.c_int32, C.c_int32]
    assert L.lib.nnb_render_tmin_workspace_bytes.restype == C.c_size_t
    assert L.lib.nnb_version() == 105


def _rc_fwd(**over):
    f = L.FrameArgs()
    f.fwd = _args(**over).fwd
    f.t_min = over.get("t_min", 1e-4)
    f.n_eval = over.get("n_eval", None); f.t_final = over.get("t_final", None)
    return L.lib.nnb_render_fwd_tmin(C.byref(f), None)


def _rc_bwd(**over):
    return L.lib.nnb_render_bwd_tmin(C.byref(_args(**over)), None)


def test_workspace_bytes():
    ws = L.lib.nnb_render_tmin_workspace_bytes
    for bad in ((0, 128, 256), (-1, 128, 256), (1000, 15, 256), (1000, 1025, 256), (1000, 128, 96), (1000, 1, 256)):
        assert ws(*bad) == 0, bad
    for N, S, D in ((1000, 128, 256), (1, 16, 64), (4096, 512, 256), (1023, 33, 128), (5, 1024, 64)):
        stash = L.lib.nnb_workspace_bytes_dim(N, S, L.STASH, L.ENGINE_TC, D)
        assert ws(N, S, D) >= stash > 0, (N, S, D)
    assert ws(1000, 128, 0) == ws(1000, 128, 256)
    assert ws(1001, 128, 256) > ws(1000, 128, 256) and ws(1000, 160, 256) > ws(1000, 128, 256)


@pytest.mark.parametrize("rc", [_rc_fwd, _rc_bwd], ids=["fwd", "bwd"])
def test_argument_checks(rc):
    assert rc(engine=L.ENGINE_SIMT) == -4 and rc(engine=7) == -4
    assert rc(flags=512) == -7
    for flag in (L.STASH, L.HVP, L.OCC_ONLY, L.RAW_DENSITY):
        assert rc(flags=flag) == -6
    assert rc(hidden_dim=96) == -8
    assert rc(N=0) == -2 and rc(S=1025) == -2 and rc(S=1) == -2 and rc(S=15) == -4
    assert rc(noise=0xa0000) == -5          # jitter is accepted: the call reaches the workspace check
    for k in ("z_vals", "alpha", "pts", "dirs"):
        assert rc(**{k: 0xa0000}) == -6, k
    for k in ("weights", "c2w", "cam", "rgb", "mask"):
        assert rc(**{k: None}) == -3, k
    assert rc() == -5
    need = L.lib.nnb_render_tmin_workspace_bytes(1000, 128, 256)
    assert need > L.lib.nnb_render_frame_bwd_workspace_bytes(1000, 128, 256)
    assert rc(workspace_bytes=need - 1) == -5
    assert rc(workspace_bytes=L.lib.nnb_render_frame_bwd_workspace_bytes(1000, 128, 256)) == -5   # the frame pair's is too small
    assert rc(workspace=0x100080, workspace_bytes=need) == -5
    # the order of the checks: engine, flags, width, sizes, per-sample outputs, (t_min,) pointers, workspace
    assert rc(engine=L.ENGINE_SIMT, flags=512) == -4 and rc(flags=512, hidden_dim=96) == -7
    assert rc(hidden_dim=96, N=0) == -8 and rc(N=0, z_vals=0xa0000) == -2 and rc(z_vals=0xa0000, weights=None) == -6
    assert rc(weights=None, workspace_bytes=0) == -3


def test_t_min_and_stats_checks():
    assert _rc_fwd(t_min=-1e-4) == -2 and _rc_fwd(t_min=float("nan")) == -2 and _rc_fwd(t_min=-math.inf) == -2
    assert _rc_fwd(t_min=0.0) == -5 and _rc_fwd(t_min=math.inf) == -5      # both reach the workspace check
    assert _rc_fwd(t_min=-1.0, engine=L.ENGINE_SIMT) == -4                  # the engine is checked first
    assert _rc_fwd(t_min=-1.0, flags=L.STASH) == -6                         # then the flags, then t_min
    assert _rc_fwd(t_min=-1.0, weights=None) == -2                          # t_min before the pointers
    assert _rc_fwd(n_eval=0xa0002) == -3 and _rc_fwd(t_final=0xa0001) == -3
    assert _rc_fwd(n_eval=0xa0000, t_final=0xb0000) == -5


def test_null_args_and_gradient_pointers():
    assert L.lib.nnb_render_fwd_tmin(None, None) == -1
    assert L.lib.nnb_render_bwd_tmin(None, None) == -1
    assert _rc_bwd(g_rgb=None) == -3 and _rc_bwd(g_c2w=None) == -3
    assert _rc_bwd(g_weights=None) == -5                                 # pose only: reaches the workspace check
    assert _rc_fwd(g_rgb=None) == -5 and _rc_fwd(g_c2w=None) == -5     # the forward takes no gradients


def test_stash_render_call_caching_and_values():
    from nope_nerf_b200 import ops
    assert ops.RenderCall.stash_tmin is False and ops.FrameRenderCall.stash_tmin is False
    c = ops.stash_render_call(1e-4)
    assert c is ops.stash_render_call(1e-4) and c is ops.stash_render_call(float(C.c_float(1e-4).value))
    assert issubclass(c, ops.RenderCall) and not issubclass(c, ops.FrameRenderCall)
    assert c.stash_tmin and not c.frame and not c.exact_frame and c.t_min == C.c_float(1e-4).value
    assert c is not ops.frame_render_call(1e-4)
    z = ops.stash_render_call(0.0)
    assert z is ops.stash_render_call(0) and z is not c and z.t_min == 0.0
    for bad in (-1e-4, float("nan"), -math.inf):
        with pytest.raises(ValueError, match="t_min"):
            ops.stash_render_call(bad)
    assert inspect.signature(c.__init__) == inspect.signature(ops.RenderCall.__init__)
    eye = torch.eye(4)
    kw = dict(N=1, S=32, flags=0, near=0, far=1)
    with pytest.raises(ValueError, match="tensor-core"):   # checked before any device check
        c(eye, eye, eye, engine=L.ENGINE_SIMT, **kw)
    with pytest.raises(ValueError, match="tensor-core"):
        c(eye, eye, eye, engine=None, N=1, S=8, flags=0, near=0, far=1)
    with pytest.raises(ValueError, match="want_z_alpha"):
        c(eye, eye, eye, engine=None, want_z_alpha=True, **kw)
    with pytest.raises(RuntimeError, match="CUDA device"):
        c(eye, eye, eye, engine=None, **kw)


def test_trainer_option(monkeypatch):
    from nope_nerf_b200 import ops
    monkeypatch.setattr(ops, "_DEFAULT_ENGINE", [L.ENGINE_TC])
    t = _trainer()
    assert t.train_t_min is None and t._train_render_call(True) is ops.RenderCall
    for v in (1e-4, 0.0, 0):
        t = _trainer(train_t_min=v)
        assert t._train_render_call(True) is ops.stash_render_call(v) and t._train_render_call(False) is ops.RenderCall
    assert _trainer(engine=L.ENGINE_TC, train_t_min=1e-4)._train_render_call(True) is ops.stash_render_call(1e-4)
    with pytest.raises(ValueError, match="frame_grad"):
        _trainer(frame_grad=True, train_t_min=1e-4)
    with pytest.raises(ValueError, match="frame_grad"):
        _trainer(frame_grad=True, frame_grad_t_min=1e-4, train_t_min=1e-4)
    for bad in (-1e-4, float("nan")):
        with pytest.raises(ValueError, match="t_min"):
            _trainer(train_t_min=bad)
    with pytest.raises(ValueError, match="tensor-core"):
        _trainer(S=8, train_t_min=1e-4)
    with pytest.raises(ValueError, match="tensor-core"):
        _trainer(engine=L.ENGINE_SIMT, train_t_min=1e-4)


def test_every_source_compiles_for_sm90a(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    from nope_nerf_b200 import build as B
    srcs = sorted(f for f in os.listdir(B.CSRC) if f.endswith(".cu"))
    procs = {s: subprocess.Popen([nvcc] + B.NVCC_FLAGS + ["-c", os.path.join(B.CSRC, s), "-o", str(tmp_path / (s + ".o"))],
                                 stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for s in srcs}
    for s, p in procs.items():
        _, err = p.communicate()
        assert p.returncode == 0, (s, err[-2000:])
        elf = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-lelf", str(tmp_path / (s + ".o"))], capture_output=True,
                             text=True)
        assert "sm_90a" in elf.stdout, (s, elf.stdout)

"""Host side of nnb_geometry_frame (the geometry view of any set of pixels in one tensor-core call): the workspace rule, the argument
checks (every documented error code, returned before anything is launched), the ctypes bindings and the Python surface
(Renderer.phong_frame's input checks, the default-off renderer option).  Needs no device: rejected calls never reach the GPU."""
import ctypes as C
import inspect

import pytest
import torch

from nope_nerf_b200 import _lib as L
from _cfg import default_cfg


def _align(x, a=256):
    return (x + a - 1) // a * a


def expected_bytes(N, n_steps, D):
    """the documented layout: hit count | rays | compacted rows | nnb_ray_march's, nnb_field_vjp's (occupancy-only) workspaces | the
    points mode's forward weight image, each 256-byte aligned"""
    ks = D // 16
    stage = 64 * D
    n_fwd = 4 + 3 * ks + (4 + ks) + 3 * ks + ks + ks
    img_pts = (n_fwd - ks) * stage + ks * stage // 2 + 2 * stage // 2
    own = _align(4) + 2 * _align(12 * N) + 2 * _align(4 * N) + 2 * _align(12 * N) + _align(4 * N) + 3 * _align(16 * N)
    return (own + _align(L.lib.nnb_ray_march_workspace_bytes(N, n_steps, D))
            + _align(L.lib.nnb_field_vjp_workspace_bytes(N, L.RAW_DENSITY | L.OCC_ONLY, D)) + _align(img_pts))


def test_workspace_matches_its_formula():
    for N in (1, 127, 128, 129, 4096, 129600, 1080 * 1920):
        for n_steps in (2, 128, 512, 513):
            for D in L.HIDDEN_DIMS:
                assert L.lib.nnb_geometry_frame_workspace_bytes(N, n_steps, D) == expected_bytes(N, n_steps, D), (N, n_steps, D)
    assert L.lib.nnb_geometry_frame_workspace_bytes(1000, 512, 0) == expected_bytes(1000, 512, 256)   # 0 means 256


def test_documented_size_of_a_1080p_frame():
    """the byte count the header states for one 1080 x 1920 frame at D = 256 and the 512 steps of the geometry view"""
    n = L.lib.nnb_geometry_frame_workspace_bytes(1080 * 1920, 512, 256)
    assert n == 945541632, n
    import os
    from _util import ROOT
    hdr = open(os.path.join(ROOT, "include", "nope_nerf_b200.h")).read()
    assert "{:,}".format(n).replace(",", " ") in hdr


def test_workspace_query_rejects_bad_sizes_and_widths():
    for D in (1, 32, 96, 192, 255, 512, -256):
        assert L.lib.nnb_geometry_frame_workspace_bytes(1000, 512, D) == 0
    for N, n_steps in ((0, 512), (-1, 512), (1000, 1), (1000, 0), (1000, -5)):
        assert L.lib.nnb_geometry_frame_workspace_bytes(N, n_steps, 256) == 0


def _args(**over):
    """a call whose pointers are fake, aligned device addresses: every call below is rejected before one is dereferenced"""
    a = L.GeometryArgs()
    a.weights, a.T, a.pixels, a.frac, a.rgb, a.rgb_surf = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
    a.N = 1000; a.n_steps = 512; a.n_secant = 8; a.hidden_dim = 256
    a.near_ = 0.0; a.tau = 0.5; a.radius = 4.0; a.flags = 0; a.engine = L.ENGINE_TC
    a.workspace = 0x100000; a.workspace_bytes = 0      # too small for anything
    for k, v in over.items():
        setattr(a, k, v)
    return a


def _rc(**over):
    return L.lib.nnb_geometry_frame(C.byref(_args(**over)), None)


def test_every_documented_error_code():
    assert _rc(engine=L.ENGINE_SIMT) == -4 and _rc(engine=7) == -4
    for bit in (512, 1024, 4096, 8192, 1 << 16, 1 << 31):
        assert _rc(flags=bit) == -7
    for flag in (L.NDC, L.STASH, L.RAW_DENSITY, L.OCC_ONLY, L.HVP):
        assert _rc(flags=flag) == -6
    for D in (1, 96, 512):
        assert _rc(hidden_dim=D) == -8
    assert _rc(N=-1) == -2 and _rc(n_steps=1) == -2 and _rc(n_secant=-1) == -2
    for k in ("weights", "T", "pixels", "frac", "rgb", "rgb_surf"):
        assert _rc(**{k: None}) == -3, k
    for k in ("weights", "T", "pixels", "frac", "rgb", "rgb_surf", "ray0", "ray_dir", "far_", "depth"):
        assert _rc(**{k: 0x70002}) == -3, k
    assert _rc(grad=0x70008) == -3
    assert "grad" in L.lib.nnb_last_error().decode()
    assert _rc() == -5                                                            # undersized
    need = L.lib.nnb_geometry_frame_workspace_bytes(1000, 512, 256)
    assert _rc(workspace_bytes=need - 1) == -5
    assert _rc(workspace=None, workspace_bytes=need) == -5
    assert _rc(workspace=0x100080, workspace_bytes=need) == -5                   # not 256-byte aligned
    assert L.lib.nnb_geometry_frame(None, None) == -1


def test_empty_call_launches_nothing():
    """N == 0 returns 0 before any pointer or workspace is looked at (this machine may have no device at all)"""
    assert _rc(N=0, weights=None, T=None, workspace=None) == 0


def test_bindings():
    assert L.lib.nnb_geometry_frame_workspace_bytes.restype is C.c_size_t
    assert L.lib.nnb_geometry_frame_workspace_bytes.argtypes == [C.c_int32, C.c_int32, C.c_int32]
    assert L.lib.nnb_geometry_frame.argtypes == [C.POINTER(L.GeometryArgs), C.c_void_p]
    assert [f for f, _ in L.GeometryArgs._fields_] == [
        "weights", "T", "pixels", "frac", "N", "n_steps", "n_secant", "hidden_dim", "near_", "tau", "radius", "flags", "engine",
        "rgb", "rgb_surf", "ray0", "ray_dir", "far_", "depth", "grad", "workspace", "workspace_bytes"]
    assert C.sizeof(L.GeometryArgs) == 144
    assert L.lib.nnb_version() == 105   # the symbol, not the version, marks the capability


def _renderer(**kw):
    import nope_nerf_b200.model as mdl
    cfg = default_cfg()
    return mdl.Renderer(mdl.OfficialStaticNerf(cfg), cfg["rendering"], device=torch.device("cpu"), **kw)


def test_phong_frame_rejects_cpu_tensors_and_batches():
    rend = _renderer()
    eye = torch.eye(4)[None]
    with pytest.raises(RuntimeError, match="CUDA"):
        rend.phong_frame(torch.zeros(1, 4, 2), eye, eye, eye, 0)
    with pytest.raises(NotImplementedError, match="batch_size"):
        rend.phong_frame(torch.zeros(2, 4, 2), eye, eye, eye, 0)
    # routed from forward when the option is on
    rend = _renderer(geometry_frame=True)
    assert rend.geometry_frame is True
    with pytest.raises(RuntimeError, match="CUDA"):
        rend(torch.zeros(1, 4, 2), None, eye, eye, eye, "phong_renderer", it=0)


def test_option_is_off_by_default():
    from nope_nerf_b200 import field
    from nope_nerf_b200.model import rendering
    assert _renderer().geometry_frame is False
    assert rendering.GEOMETRY_CHUNK == 1024
    sig = inspect.signature(field.geometry_frame).parameters
    assert sig["n_secant"].default == 8 and sig["tau"].default == 0.5 and sig["near"].default == 0.0
    assert sig["want_intermediates"].default is False

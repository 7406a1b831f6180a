"""Host side of nnb_render_frame_engine (the volumetric frame with compositing fused into the forward, on either engine): the workspace
query, every documented error code (returned before anything is launched), the ctypes bindings and the Python surface (ops.render_frame_engine,
the Renderer(frame_engine=) option and Extract_Images.render_frame's routing).  Needs no device: rejected calls never reach the GPU."""
import ctypes as C
import inspect
import os

import pytest
import torch

from nope_nerf_b200 import _lib as L
from _cfg import default_cfg
from test_render_frame_host import _args, _Recorder, expected_bytes


def _rc(**over):
    return L.lib.nnb_render_frame_engine(C.byref(_args(**over)), None)


def _rc_tc(**over):
    return L.lib.nnb_render_frame(C.byref(_args(**over)), None)


def _ws(N, S, D, engine):
    return L.lib.nnb_render_frame_workspace_bytes_engine(N, S, D, engine)


def _align(x, a=256):
    return (x + a - 1) // a * a


def test_workspace_query():
    """TC: nnb_render_frame_workspace_bytes; SIMT: the same layout without the weight image, for every S from 2 to 1024"""
    for N in (1, 3, 5, 127, 4096, 1080 * 1920):
        for D in L.HIDDEN_DIMS:
            simt = 256 + 4 * _align(4 * N) + _align(640 * N)
            img = expected_bytes(N, D) - simt
            assert img > 0 and img % 256 == 0
            for S in (16, 17, 128, 1024):
                assert _ws(N, S, D, L.ENGINE_TC) == L.lib.nnb_render_frame_workspace_bytes(N, S, D) == expected_bytes(N, D)
            for S in (2, 3, 8, 15, 16, 31, 33, 128, 512, 1024):
                assert _ws(N, S, D, L.ENGINE_SIMT) == simt == _ws(N, 128, D, L.ENGINE_TC) - img, (N, S, D)
    assert _ws(1000, 8, 0, L.ENGINE_SIMT) == _ws(1000, 8, 256, L.ENGINE_SIMT)   # 0 means 256


def test_workspace_query_rejects_bad_engines_widths_and_sizes():
    for engine in (-1, 2, 7):
        assert _ws(1000, 128, 256, engine) == 0
    for engine in (L.ENGINE_TC, L.ENGINE_SIMT):
        for D in (1, 32, 96, 192, 255, 512, -256):
            assert _ws(1000, 128, D, engine) == 0
        for N, S in ((0, 128), (-1, 128), (1000, 1), (1000, 0), (1000, 1025), (1000, -5)):
            assert _ws(N, S, 256, engine) == 0
    for S in (2, 8, 15):
        assert _ws(1000, S, 256, L.ENGINE_TC) == 0 and _ws(1000, S, 256, L.ENGINE_SIMT) > 0


def test_documented_size_of_a_1080p_frame():
    n = _ws(1080 * 1920, 128, 256, L.ENGINE_SIMT)
    assert n == 1360281856 and n == _ws(1080 * 1920, 2, 64, L.ENGINE_SIMT) == _ws(1080 * 1920, 1024, 128, L.ENGINE_SIMT)
    from _util import ROOT
    hdr = open(os.path.join(ROOT, "include", "nope_nerf_b200.h")).read()
    assert "{:,}".format(n).replace(",", " ") in hdr


@pytest.mark.parametrize("engine", ["tc", "simt"])
def test_every_documented_error_code(engine):
    eng = {"tc": L.ENGINE_TC, "simt": L.ENGINE_SIMT}[engine]
    rc = lambda **over: _rc(**dict(dict(engine=eng), **over))
    assert L.lib.nnb_render_frame_engine(None, None) == -1
    assert _rc(engine=7) == -4 and _rc(engine=-1) == -4 and _rc(engine=2) == -4
    for bit in (512, 1024, 4096, 8192, 1 << 16, 1 << 31):
        assert rc(flags=bit) == -7
    for flag in (L.STASH, L.HVP, L.OCC_ONLY, L.RAW_DENSITY):
        assert rc(flags=flag | L.EVAL) == -6
    for D in (1, 96, 512):
        assert rc(hidden_dim=D) == -8
    assert rc(N=0) == -2 and rc(N=-1) == -2
    for S in (0, 1, 1025, 4096):
        assert rc(S=S) == -2, S
    for S in (2, 3, 8, 15):   # the tensor-core engine's limit; the exact engine takes them (and then wants its workspace)
        assert rc(S=S) == (-4 if engine == "tc" else -5), S
    for k in ("noise", "z_vals", "alpha", "pts", "dirs"):
        assert rc(**{k: 0xa0000}) == -6, k
    for t in (-1e-9, -1.0, float("nan"), float("-inf")):
        assert rc(t_min=t) == -2, t
    for k in ("weights", "c2w", "cam", "rgb", "depth_pred", "depth_gt", "mask"):
        assert rc(**{k: None}) == -3, k
    assert rc(ray_idx=None) == -3 and rc(H=1) == -3 and rc(depth_map=None) == -3
    assert rc(n_eval=0xa0002) == -3 and rc(t_final=0xa0001) == -3
    assert rc() == -5
    need = _ws(1000, 128, 256, eng)
    assert rc(workspace_bytes=need - 1) == -5
    assert rc(workspace=None, workspace_bytes=need) == -5
    assert rc(workspace=0x100080, workspace_bytes=need) == -5
    assert rc(t_min=float("inf")) == -5 and rc(ray_idx=None, pixels=0xb0000, depth=0xc0000, depth_map=None) == -5
    assert "workspace" in L.lib.nnb_last_error().decode()


def test_nnb_render_frame_keeps_its_contract():
    """nnb_render_frame still rejects the exact engine and S < 16 with -4"""
    assert _rc_tc(engine=L.ENGINE_SIMT) == -4 and _rc_tc(engine=7) == -4
    for S in (2, 8, 15):
        assert _rc_tc(S=S) == -4
    assert L.lib.nnb_render_frame_workspace_bytes(1000, 8, 256) == 0


def test_bindings():
    assert L.lib.nnb_render_frame_workspace_bytes_engine.restype is C.c_size_t
    assert L.lib.nnb_render_frame_workspace_bytes_engine.argtypes == [C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    assert L.lib.nnb_render_frame_engine.argtypes == [C.POINTER(L.FrameArgs), C.c_void_p]
    assert L.lib.nnb_version() == 105   # the symbols, not the version, mark the capability


def test_ops_render_frame_engine_surface():
    from nope_nerf_b200 import ops
    assert list(inspect.signature(ops.render_frame_engine).parameters) == list(inspect.signature(ops.render_frame).parameters)
    eye = torch.eye(4)
    with pytest.raises(ValueError, match="noise"):
        ops.render_frame_engine(eye, eye, eye, N=1, S=8, flags=0, engine=None, near=0, far=1, noise=eye)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.render_frame_engine(eye, eye, eye, N=1, S=8, flags=0, engine=L.ENGINE_SIMT, near=0, far=1)


def _renderer(**kw):
    import nope_nerf_b200.model as mdl
    cfg = default_cfg()
    return mdl.Renderer(mdl.OfficialStaticNerf(cfg), cfg["rendering"], device=torch.device("cpu"), **kw)


def test_frame_engine_option_is_checked():
    assert _renderer().frame_engine is None
    assert _renderer(frame_t_min=0, frame_engine="simt").frame_engine == "simt"
    assert _renderer(frame_t_min=1e-3, frame_engine="tc").frame_engine == "tc"
    assert _renderer(frame_engine="tc").frame_engine == "tc"
    with pytest.raises(ValueError, match="frame_t_min"):
        _renderer(frame_engine="simt")                       # would do nothing without frame_t_min
    for bad in ("SIMT", "exact", 0, 1, L.ENGINE_SIMT, True):
        with pytest.raises(ValueError, match="frame_engine"):
            _renderer(frame_t_min=0, frame_engine=bad)


class _EngineRecorder(_Recorder):
    def render_frame_engine(self, *a, **kw):
        self.calls.append(("render_frame_engine", kw))
        n = kw["N"]
        return torch.zeros(n, 3), torch.zeros(n), torch.zeros(n), torch.zeros(n, dtype=torch.uint8)


@pytest.mark.parametrize("frame_engine, opt, engine, S, path", [
    # frame_engine='simt' takes the exact frame at every engine and sample count
    ("simt", 0.0, None, 128, "render_frame_engine"),
    ("simt", 1e-3, None, 8, "render_frame_engine"),
    ("simt", 0.0, "tc", 128, "render_frame_engine"),
    ("simt", 1e-4, "tc", 8, "render_frame_engine"),
    ("simt", 0.0, "simt", 128, "render_frame_engine"),
    ("simt", 0.0, "simt", 8, "render_frame_engine"),
    # None and 'tc' keep the existing routes
    (None, None, None, 128, "RenderCall"),
    (None, 0.0, None, 128, "render_frame"),
    (None, 1e-3, "tc", 64, "render_frame"),
    (None, 0.0, "simt", 128, "RenderCall"),
    (None, 0.0, None, 8, "RenderCall"),
    ("tc", 0.0, None, 128, "render_frame"),
    ("tc", 0.0, "simt", 128, "RenderCall"),
    ("tc", None, None, 128, "RenderCall"),
])
def test_extract_images_routing(monkeypatch, frame_engine, opt, engine, S, path):
    from nope_nerf_b200 import ops
    from nope_nerf_b200.model import extracting_images
    rec = _EngineRecorder(ops)
    monkeypatch.setattr(extracting_images, "ops", rec)
    cfg = default_cfg()
    cfg["rendering"]["num_points"] = S
    cfg["extract_images"] = {"resolution": [6, 5]}
    import nope_nerf_b200.model as mdl
    eng = {None: None, "tc": L.ENGINE_TC, "simt": L.ENGINE_SIMT}[engine]
    rend = mdl.Renderer(mdl.OfficialStaticNerf(cfg), cfg["rendering"], device=torch.device("cpu"), engine=eng, frame_t_min=opt,
                        frame_engine=frame_engine)
    rend.model.flat_weights = lambda: torch.zeros(1)
    ex = extracting_images.Extract_Images(rend, cfg, device=torch.device("cpu"))
    rgb, depth = ex.render_frame(torch.eye(4), torch.eye(4), 6, 5, rows=(2, 5))
    assert [c[0] for c in rec.calls] == [path]
    kw = rec.calls[0][1]
    assert rgb.shape == (3, 5, 3) and depth.shape == (3, 5) and kw["N"] == 15 and kw["S"] == S and kw["stash"] is False
    if path == "render_frame_engine":
        assert kw["engine"] == L.ENGINE_SIMT and kw["t_min"] == opt
    elif path == "render_frame":
        assert kw["t_min"] == opt
    else:
        assert "t_min" not in kw

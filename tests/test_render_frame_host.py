"""Host side of nnb_render_frame (the volumetric view of a frame with compositing fused into the tensor-core forward): the workspace rule,
every documented error code (returned before anything is launched), the ctypes bindings and the Python surface (the default-off
Renderer option and Extract_Images.render_frame's routing).  Needs no device: rejected calls never reach the GPU."""
import ctypes as C
import inspect
import os

import pytest
import torch

from nope_nerf_b200 import _lib as L
from _cfg import default_cfg


def _align(x, a=256):
    return (x + a - 1) // a * a


def expected_bytes(N, D):
    """the documented layout: round counters (256 bytes) | carry, chunks [N] | lane partials [N][5][32] | two ray lists [N] | the forward
    weight image, each 256-byte aligned.  S does not enter."""
    ks = D // 16
    stage = 64 * D
    n_fwd = 4 + 3 * ks + (4 + ks) + 3 * ks + ks + ks
    img = (n_fwd - ks) * stage + ks * stage // 2
    return 256 + 4 * _align(4 * N) + _align(640 * N) + _align(img)


def test_workspace_matches_its_formula():
    for N in (1, 3, 4, 5, 127, 4096, 518400, 1080 * 1920):
        for S in (16, 17, 32, 128, 512, 1024):
            for D in L.HIDDEN_DIMS:
                assert L.lib.nnb_render_frame_workspace_bytes(N, S, D) == expected_bytes(N, D), (N, S, D)
    assert L.lib.nnb_render_frame_workspace_bytes(1000, 128, 0) == expected_bytes(1000, 256)   # 0 means 256


def test_documented_size_of_a_1080p_frame():
    """the byte count the header states for one 1080 x 1920 frame at D = 256 (any S), and the weight image it names"""
    n = L.lib.nnb_render_frame_workspace_bytes(1080 * 1920, 128, 256)
    assert n == 1362641152, n
    assert n == L.lib.nnb_render_frame_workspace_bytes(1080 * 1920, 1024, 256)
    from _util import ROOT
    hdr = open(os.path.join(ROOT, "include", "nope_nerf_b200.h")).read()
    assert "{:,}".format(n).replace(",", " ") in hdr
    assert "2 359 296" in hdr
    # nnb_render_fwd's workspace for the same frame holds 32 N S bytes of records
    assert L.lib.nnb_workspace_bytes_dim(1080 * 1920, 128, 0, L.ENGINE_TC, 256) > 6 * n


def test_workspace_query_rejects_bad_sizes_and_widths():
    for D in (1, 32, 96, 192, 255, 512, -256):
        assert L.lib.nnb_render_frame_workspace_bytes(1000, 128, D) == 0
    for N, S in ((0, 128), (-1, 128), (1000, 15), (1000, 2), (1000, 0), (1000, 1025), (1000, -5)):
        assert L.lib.nnb_render_frame_workspace_bytes(N, S, 256) == 0


def _args(**over):
    """a call whose pointers are fake, aligned device addresses: every call below is rejected before one is dereferenced"""
    f = L.FrameArgs()
    a = f.fwd
    a.weights, a.c2w, a.cam, a.ray_idx, a.depth_map = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000
    a.rgb, a.depth_pred, a.depth_gt, a.mask = 0x60000, 0x70000, 0x80000, 0x90000
    a.N, a.S, a.H, a.W, a.h_d, a.w_d = 1000, 128, 25, 40, 1, 1
    a.near_, a.far_ = 0.0, 1.0
    a.flags = L.EVAL | L.SOFTPLUS; a.engine = L.ENGINE_TC; a.hidden_dim = 256
    a.workspace = 0x100000; a.workspace_bytes = 0      # too small for anything
    f.t_min = 0.0
    for k, v in over.items():
        setattr(f if k in ("t_min", "n_eval", "t_final") else a, k, v)
    return f


def _rc(**over):
    return L.lib.nnb_render_frame(C.byref(_args(**over)), None)


def test_every_documented_error_code():
    assert L.lib.nnb_render_frame(None, None) == -1
    assert _rc(engine=L.ENGINE_SIMT) == -4 and _rc(engine=7) == -4
    for bit in (512, 1024, 4096, 8192, 1 << 16, 1 << 31):
        assert _rc(flags=bit) == -7
    for flag in (L.STASH, L.HVP, L.OCC_ONLY, L.RAW_DENSITY):
        assert _rc(flags=flag | L.EVAL) == -6
    for D in (1, 96, 512):
        assert _rc(hidden_dim=D) == -8
    assert _rc(N=0) == -2 and _rc(N=-1) == -2
    for S in (0, 1, 1025, 4096):
        assert _rc(S=S) == -2, S
    for S in (2, 8, 15):
        assert _rc(S=S) == -4, S                                                    # the tensor-core engine's limit
    for k in ("noise", "z_vals", "alpha", "pts", "dirs"):
        assert _rc(**{k: 0xa0000}) == -6, k
    for t in (-1e-9, -1.0, float("nan"), float("-inf")):
        assert _rc(t_min=t) == -2, t
    for k in ("weights", "c2w", "cam", "rgb", "depth_pred", "depth_gt", "mask"):
        assert _rc(**{k: None}) == -3, k
    assert _rc(ray_idx=None) == -3                                               # no ray_idx, no pixels
    assert _rc(H=1) == -3
    assert _rc(depth_map=None) == -3
    assert _rc(n_eval=0xa0002) == -3 and _rc(t_final=0xa0001) == -3
    assert "n_eval" in L.lib.nnb_last_error().decode()
    assert _rc() == -5                                                           # undersized
    need = L.lib.nnb_render_frame_workspace_bytes(1000, 128, 256)
    assert _rc(workspace_bytes=need - 1) == -5
    assert _rc(workspace=None, workspace_bytes=need) == -5
    assert _rc(workspace=0x100080, workspace_bytes=need) == -5                   # not 256-byte aligned
    # the accepted values of the checks above pass them: t_min = +inf, pixels instead of ray_idx, explicit depth
    assert _rc(t_min=float("inf")) == -5 and _rc(ray_idx=None, pixels=0xb0000, depth=0xc0000, depth_map=None) == -5


def test_bindings():
    assert L.lib.nnb_render_frame_workspace_bytes.restype is C.c_size_t
    assert L.lib.nnb_render_frame_workspace_bytes.argtypes == [C.c_int32, C.c_int32, C.c_int32]
    assert L.lib.nnb_render_frame.argtypes == [C.POINTER(L.FrameArgs), C.c_void_p]
    assert [f for f, _ in L.FrameArgs._fields_] == ["fwd", "t_min", "n_eval", "t_final"]
    assert L.FrameArgs._fields_[0][1] is L.RenderArgs
    assert C.sizeof(L.FrameArgs) == C.sizeof(L.RenderArgs) + 24
    assert L.lib.nnb_version() == 105   # the symbol, not the version, marks the capability


def test_ops_render_frame_surface():
    from nope_nerf_b200 import ops
    sig = inspect.signature(ops.render_frame).parameters
    call = inspect.signature(ops.RenderCall.__init__).parameters
    assert [p for p in call if p != "self"] == list(sig)[:len(call) - 1]           # RenderCall's arguments, then the two new ones
    assert list(sig)[-2:] == ["t_min", "want_stats"]
    assert sig["t_min"].default == 0.0 and sig["want_stats"].default is False
    eye = torch.eye(4)
    with pytest.raises(ValueError, match="noise"):
        ops.render_frame(eye, eye, eye, N=1, S=32, flags=0, engine=None, near=0, far=1, noise=eye)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.render_frame(eye, eye, eye, N=1, S=32, flags=0, engine=None, near=0, far=1)


def _renderer(**kw):
    import nope_nerf_b200.model as mdl
    cfg = default_cfg()
    return mdl.Renderer(mdl.OfficialStaticNerf(cfg), cfg["rendering"], device=torch.device("cpu"), **kw)


def test_option_is_off_by_default_and_checked():
    assert _renderer().frame_t_min is None
    assert _renderer(frame_t_min=0).frame_t_min == 0.0 and _renderer(frame_t_min=1e-3).frame_t_min == 1e-3
    for bad in (-1e-4, float("nan")):
        with pytest.raises(ValueError, match="frame_t_min"):
            _renderer(frame_t_min=bad)


class _Recorder:
    """stands in for ops in extracting_images: records which path render_frame took"""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, k):
        return getattr(self.real, k)

    def RenderCall(self, *a, **kw):
        self.calls.append(("RenderCall", kw))
        n = kw["N"]
        return type("Call", (), dict(rgb=torch.zeros(n, 3), depth_pred=torch.zeros(n)))()

    def render_frame(self, *a, **kw):
        self.calls.append(("render_frame", kw))
        n = kw["N"]
        return torch.zeros(n, 3), torch.zeros(n), torch.zeros(n), torch.zeros(n, dtype=torch.uint8)


@pytest.mark.parametrize("opt, engine, S, path", [
    (None, None, 128, "RenderCall"),          # the default: nnb_render_fwd, as before
    (0.0, None, 128, "render_frame"),
    (1e-3, "tc", 64, "render_frame"),
    (0.0, "simt", 128, "RenderCall"),         # the SIMT engine keeps nnb_render_fwd
    (0.0, None, 8, "RenderCall"),             # S < 16 runs on the SIMT engine
])
def test_extract_images_routing(monkeypatch, opt, engine, S, path):
    from nope_nerf_b200 import ops
    from nope_nerf_b200.model import extracting_images
    rec = _Recorder(ops)
    monkeypatch.setattr(extracting_images, "ops", rec)
    cfg = default_cfg()
    cfg["rendering"]["num_points"] = S
    cfg["extract_images"] = {"resolution": [6, 5]}
    import nope_nerf_b200.model as mdl
    eng = {None: None, "tc": L.ENGINE_TC, "simt": L.ENGINE_SIMT}[engine]
    rend = mdl.Renderer(mdl.OfficialStaticNerf(cfg), cfg["rendering"], device=torch.device("cpu"), engine=eng, frame_t_min=opt)
    rend.model.flat_weights = lambda: torch.zeros(1)
    ex = extracting_images.Extract_Images(rend, cfg, device=torch.device("cpu"))
    rgb, depth = ex.render_frame(torch.eye(4), torch.eye(4), 6, 5, rows=(2, 5))
    assert [c[0] for c in rec.calls] == [path]
    kw = rec.calls[0][1]
    assert rgb.shape == (3, 5, 3) and depth.shape == (3, 5) and kw["N"] == 15 and kw["S"] == S and kw["stash"] is False
    if path == "render_frame":
        assert kw["t_min"] == opt
    else:
        assert "t_min" not in kw

"""Host side of the exact-fp32 fused march and geometry frame (nnb_ray_march_engine / nnb_geometry_frame_engine): the engine
rule and argument checks of both calls (every documented error code, returned before anything is launched), the per-engine workspace
queries, the ctypes bindings, and the keyword routing of field.ray_march / field.geometry_frame / Renderer.  Needs no device."""
import ctypes as C
import inspect

import pytest
import torch

from nope_nerf_b200 import _lib as L
from _cfg import default_cfg


def _align(x, a=256):
    return (x + a - 1) // a * a


def march_bytes(N, n_steps):
    """the exact march's layout: counters | status, first, carry, two lists, hits | brk0, brk1 (no weight image)"""
    rounds = (n_steps + 127) // 128
    return _align(4 * (rounds + 1)) + 6 * _align(4 * N) + 2 * _align(16 * N)


def frame_bytes(N, n_steps, D):
    """the exact frame's documented layout: hit count | rays | compacted rows | the exact march | one pass's records and fp32 stash"""
    npad = (N + 63) // 64 * 64
    c = min(npad, 32768)
    own = _align(4) + 2 * _align(12 * N) + 2 * _align(4 * N) + 2 * _align(12 * N) + _align(4 * N) + _align(16 * N) + _align(16 * npad) + _align(16 * N)
    stash = _align(32 * c) + 9 * _align(4 * c * D) + _align(2 * c * D) + _align(256 * c) + _align(128 * c) + _align(16 * c)
    return own + _align(march_bytes(N, n_steps)) + stash


def test_workspace_queries_match_their_formulas():
    for N in (1, 63, 64, 65, 4096, 129600, 1080 * 1920):
        for n_steps in (2, 128, 129, 512):
            assert L.lib.nnb_ray_march_workspace_bytes_engine(N, n_steps, 256, L.ENGINE_SIMT) == march_bytes(N, n_steps)
            assert (L.lib.nnb_ray_march_workspace_bytes_engine(N, n_steps, 64, L.ENGINE_TC)
                    == L.lib.nnb_ray_march_workspace_bytes(N, n_steps, 64))
            for D in L.HIDDEN_DIMS:
                assert L.lib.nnb_geometry_frame_workspace_bytes_engine(N, n_steps, D, L.ENGINE_SIMT) == frame_bytes(N, n_steps, D), (N, n_steps, D)
                assert (L.lib.nnb_geometry_frame_workspace_bytes_engine(N, n_steps, D, L.ENGINE_TC)
                        == L.lib.nnb_geometry_frame_workspace_bytes(N, n_steps, D))


def test_documented_size_of_a_1080p_exact_frame():
    n = L.lib.nnb_geometry_frame_workspace_bytes_engine(1080 * 1920, 512, 256, L.ENGINE_SIMT)
    assert n == 672993792, n
    import os
    from _util import ROOT
    for doc in ("include/nope_nerf_b200.h", "INTEGRATION.md"):
        assert "{:,}".format(n).replace(",", " ") in open(os.path.join(ROOT, doc)).read(), doc


def test_size_queries_return_zero_on_bad_input():
    for q in (L.lib.nnb_ray_march_workspace_bytes_engine, L.lib.nnb_geometry_frame_workspace_bytes_engine):
        for eng in (L.ENGINE_SIMT, L.ENGINE_TC):
            for D in (1, 32, 96, 255, 512, -256):
                assert q(1000, 512, D, eng) == 0
            for N, n_steps in ((0, 512), (-1, 512), (1000, 1), (1000, 0), (1000, -5)):
                assert q(N, n_steps, 256, eng) == 0
            assert q(1000, 512, 0, eng) == q(1000, 512, 256, eng) > 0   # 0 means 256
        for eng in (2, 7, -1):
            assert q(1000, 512, 256, eng) == 0


def _geo_args(**over):
    """fake, aligned device addresses: every call below is rejected before one is dereferenced"""
    a = L.GeometryArgs()
    a.weights, a.T, a.pixels, a.frac, a.rgb, a.rgb_surf = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
    a.N = 1000; a.n_steps = 512; a.n_secant = 8; a.hidden_dim = 256
    a.near_ = 0.0; a.tau = 0.5; a.radius = 4.0; a.flags = 0; a.engine = L.ENGINE_TC
    a.workspace = 0x100000; a.workspace_bytes = 0
    for k, v in over.items():
        setattr(a, k, v)
    return a


def _geo_rc(**over):
    return L.lib.nnb_geometry_frame_engine(C.byref(_geo_args(**over)), None)


@pytest.mark.parametrize("engine", [L.ENGINE_TC, L.ENGINE_SIMT])
def test_every_documented_error_code_both_engines(engine):
    """nnb_geometry_frame_engine's error codes, in their order, on both engines (the engine check: any other value is -4)"""
    rc = lambda **kw: _geo_rc(engine=engine, **kw)
    for bad in (2, 7, -1):
        assert _geo_rc(engine=bad) == -4
    for bit in (512, 1024, 4096, 8192, 1 << 16, 1 << 31):
        assert rc(flags=bit) == -7
    for flag in (L.NDC, L.STASH, L.RAW_DENSITY, L.OCC_ONLY, L.HVP):
        assert rc(flags=flag) == -6
    for D in (1, 96, 512):
        assert rc(hidden_dim=D) == -8
    assert rc(N=-1) == -2 and rc(n_steps=1) == -2 and rc(n_secant=-1) == -2
    for k in ("weights", "T", "pixels", "frac", "rgb", "rgb_surf"):
        assert rc(**{k: None}) == -3, k
    for k in ("weights", "T", "pixels", "frac", "rgb", "rgb_surf", "ray0", "ray_dir", "far_", "depth"):
        assert rc(**{k: 0x70002}) == -3, k
    assert rc(grad=0x70008) == -3
    assert "grad" in L.lib.nnb_last_error().decode()
    assert rc() == -5
    need = L.lib.nnb_geometry_frame_workspace_bytes_engine(1000, 512, 256, engine)
    assert rc(workspace_bytes=need - 1) == -5
    assert rc(workspace=None, workspace_bytes=need) == -5
    assert rc(workspace=0x100080, workspace_bytes=need) == -5
    assert L.lib.nnb_geometry_frame_engine(None, None) == -1
    assert rc(N=0, weights=None, T=None, workspace=None) == 0


def test_exact_frame_checks_its_own_workspace_size():
    """the exact frame's workspace is smaller than the tensor-core frame's here: a size between the two passes the one and not the other"""
    simt = L.lib.nnb_geometry_frame_workspace_bytes_engine(1000, 512, 256, L.ENGINE_SIMT)
    tc = L.lib.nnb_geometry_frame_workspace_bytes_engine(1000, 512, 256, L.ENGINE_TC)
    assert simt != tc
    small = min(simt, tc)
    bigger_engine = L.ENGINE_SIMT if simt > tc else L.ENGINE_TC
    assert _geo_rc(engine=bigger_engine, workspace_bytes=small) == -5


def _march_rc(**over):
    a = L.RayMarchArgs()
    a.weights, a.ray0, a.ray_dir, a.far_, a.frac, a.depth = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
    a.N = 1000; a.n_steps = 512; a.n_secant = 8; a.hidden_dim = 256; a.near_ = 0.0; a.tau = 0.5; a.flags = 0
    a.engine = L.ENGINE_SIMT; a.workspace = 0x100000; a.workspace_bytes = 0
    for k, v in over.items():
        setattr(a, k, v)
    return L.lib.nnb_ray_march_engine(C.byref(a), None)


def test_tensor_core_calls_keep_rejecting_other_engines():
    """nnb_ray_march and nnb_geometry_frame stay tensor-core calls: the exact engine runs through the _engine forms only"""
    a = _geo_args(engine=L.ENGINE_SIMT)
    assert L.lib.nnb_geometry_frame(C.byref(a), None) == -4
    m = L.RayMarchArgs()
    m.N = 8; m.n_steps = 16; m.engine = L.ENGINE_SIMT
    assert L.lib.nnb_ray_march(C.byref(m), None) == -4
    assert "nnb_ray_march_engine" in L.lib.nnb_last_error().decode()


def test_ray_march_error_codes_on_the_exact_engine():
    for bad in (2, 7, -1):
        assert _march_rc(engine=bad) == -4
    assert _march_rc(hidden_dim=96) == -8
    assert _march_rc(N=-1) == -2 and _march_rc(n_steps=1) == -2 and _march_rc(n_secant=-1) == -2
    for k in ("weights", "ray0", "ray_dir", "far_", "frac", "depth"):
        assert _march_rc(**{k: None}) == -3, k
    need = L.lib.nnb_ray_march_workspace_bytes_engine(1000, 512, 256, L.ENGINE_SIMT)
    assert _march_rc() == -5 and _march_rc(workspace_bytes=need - 1) == -5
    assert _march_rc(workspace=0x100080, workspace_bytes=need) == -5
    assert _march_rc(workspace_bytes=need, bracket=0x70008) == -3
    assert _march_rc(N=0, weights=None, workspace=None) == 0
    assert L.lib.nnb_ray_march_engine(None, None) == -1


def test_bindings():
    for q in (L.lib.nnb_ray_march_workspace_bytes_engine, L.lib.nnb_geometry_frame_workspace_bytes_engine):
        assert q.restype is C.c_size_t and q.argtypes == [C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    assert L.lib.nnb_ray_march_engine.argtypes == [C.POINTER(L.RayMarchArgs), C.c_void_p]
    assert L.lib.nnb_geometry_frame_engine.argtypes == [C.POINTER(L.GeometryArgs), C.c_void_p]
    assert L.lib.nnb_version() == 105   # the symbols, not the version, mark the capability


def _renderer(**kw):
    import nope_nerf_b200.model as mdl
    cfg = default_cfg()
    return mdl.Renderer(mdl.OfficialStaticNerf(cfg), cfg["rendering"], device=torch.device("cpu"), **kw)


def test_keywords_default_to_todays_paths():
    from nope_nerf_b200 import field
    for fn in (field.ray_march, field.geometry_frame):
        assert inspect.signature(fn).parameters["engine"].default == "tc"
    r = _renderer()
    assert r.fused_march is False and r.geometry_frame_engine is None and r.geometry_frame is False


def test_bad_engines_raise_before_any_library_call():
    from nope_nerf_b200 import field
    cfg = default_cfg()
    import nope_nerf_b200.model as mdl
    net = mdl.OfficialStaticNerf(cfg)
    z3, z1 = torch.zeros(4, 3), torch.zeros(4)
    for bad in ("cuda", 2, None, "SIMT"):
        with pytest.raises(ValueError, match="engine"):
            field.ray_march(net, z3, z3, z1, torch.linspace(0, 1, 8), 0.0, 8, 0.5, engine=bad)
        with pytest.raises(ValueError, match="engine"):
            field.geometry_frame(net, torch.eye(4), torch.zeros(4, 2), torch.linspace(0, 1, 8), 1.0, engine=bad)
    with pytest.raises(ValueError, match="engine"):
        _renderer(geometry_frame=True, geometry_frame_engine="cuda")
    for ok in ("simt", "tc", L.ENGINE_SIMT, L.ENGINE_TC):
        assert _renderer(geometry_frame=True, geometry_frame_engine=ok).geometry_frame_engine == ok
    # valid engines still need CUDA tensors
    for ok in ("simt", L.ENGINE_SIMT):
        with pytest.raises(RuntimeError, match="CUDA"):
            field.ray_march(net, z3, z3, z1, torch.linspace(0, 1, 8), 0.0, 8, 0.5, engine=ok)
        with pytest.raises(RuntimeError, match="CUDA"):
            field.geometry_frame(net, torch.eye(4), torch.zeros(4, 2), torch.linspace(0, 1, 8), 1.0, engine=ok)


def test_fused_march_routing(monkeypatch):
    """fused_march=True sends ray_marching on the exact engine (field_engine None or 'simt', no gradient, CUDA rays) to
    field.ray_march(engine='simt') and draws the same torch.randint; without it, or with CPU rays, the torch march runs"""
    from nope_nerf_b200.model import rendering
    calls = []
    monkeypatch.setattr(rendering, "ray_march", lambda *a, **kw: calls.append(kw.get("engine")) or torch.zeros(a[1].shape[0]))
    monkeypatch.setattr(rendering.Renderer, "_ray_marching_torch", lambda self, *a: calls.append("torch") or torch.zeros(1, a[0].shape[1]))

    class FakeCuda(torch.Tensor):
        @property
        def is_cuda(self):
            return True

    ray0 = torch.zeros(1, 4, 3).as_subclass(FakeCuda); rd = torch.ones(1, 4, 3).as_subclass(FakeCuda)
    for kw, want in ((dict(fused_march=True), "simt"), (dict(fused_march=True, field_engine="simt"), "simt"),
                     (dict(), "torch"), (dict(fused_march=True, field_engine="tc"), None)):
        calls.clear()
        r = _renderer(**kw)
        torch.manual_seed(0)
        with torch.no_grad():   # as in phong_renderer: a march that needs no gradient
            r.ray_marching(ray0, rd, r.model, n_steps=[512, 513])
        a = torch.rand(1)
        torch.manual_seed(0); torch.randint(512, 513, (1,)); b = torch.rand(1)
        assert calls == [want], (kw, calls)
        assert torch.equal(a, b)   # one randint drawn, as on every other path
    calls.clear()
    r = _renderer(fused_march=True)
    with torch.no_grad():
        r.ray_marching(torch.zeros(1, 4, 3), torch.ones(1, 4, 3), r.model)   # CPU rays: the torch march
    assert calls == ["torch"]

"""Host side of nnb_field_hvp_tc (the tensor-core second-order field backward): the workspace rule, the argument checks that come before
any device work, the ctypes bindings, and the grad_engine rules of field.field_normal / OfficialStaticNerf.gradient_grad /
Renderer(normal_grad_engine=), with the default routing unchanged and a third derivative refused.  Needs no device: the library's
device calls are replaced by recorders."""
import ctypes as C
import inspect

import pytest
import torch

from nope_nerf_b200 import _lib as L
from test_field_grad_host import _net


def test_workspace_is_the_occupancy_only_grad_layout_plus_a_bf16_image():
    """nnb_field_grad's occupancy-only layout (whose activation stash holds the tangents) plus the bf16 image of the occupancy-only
    forward stages; the flags do not change it"""
    for D in L.HIDDEN_DIMS:
        ks = D // 16
        img_occ = (4 + 3 * ks + (4 + ks) + 3 * ks + ks + ks - 2 * ks) * 64 * D
        for N in (1, 127, 128, 129, 4097, 131072, 200003):
            want = L.lib.nnb_field_grad_workspace_bytes(N, L.OCC_ONLY, D) + (img_occ + 255) // 256 * 256
            for flags in (0, L.RAW_DENSITY, L.OCC_ONLY, L.SOFTPLUS | L.DIST_ALPHA):
                assert L.lib.nnb_field_hvp_tc_workspace_bytes(N, flags, D) == want, (N, D, flags)
        assert L.lib.nnb_field_hvp_tc_workspace_bytes(1000, 0, 0) == L.lib.nnb_field_hvp_tc_workspace_bytes(1000, 0, 256)
    assert L.lib.nnb_field_hvp_tc_workspace_bytes(131072, 0, 256) == 2701648128


def test_workspace_query_rejects_widths_sizes_and_undefined_bits():
    for D in (1, 32, 96, 192, 255, 512, -256):
        assert L.lib.nnb_field_hvp_tc_workspace_bytes(1000, 0, D) == 0
    for N in (0, -1, -131072):
        assert L.lib.nnb_field_hvp_tc_workspace_bytes(N, 0, 256) == 0
    for bit in (512, 1 << 16, 1 << 31):
        assert L.lib.nnb_field_hvp_tc_workspace_bytes(1000, bit, 256) == 0


def test_bindings():
    assert L.lib.nnb_field_hvp_tc_workspace_bytes.restype is C.c_size_t
    assert L.lib.nnb_field_hvp_tc_workspace_bytes.argtypes == [C.c_int32, C.c_uint32, C.c_int32]
    assert L.lib.nnb_field_hvp_tc.argtypes == [C.POINTER(L.RenderArgs)] + [C.c_void_p] * 4


def test_rejections_need_no_device():
    """the checks before any device work, in nnb_field_grad's order: a NULL args, the engine, undefined and rejected flags, the width,
    N < 0; N == 0 succeeds without touching anything"""
    err = lambda: L.lib.nnb_last_error().decode()
    assert L.lib.nnb_field_hvp_tc(None, None, None, None, None) == -3
    cases = [
        (dict(engine=L.ENGINE_SIMT), -4, "engine"),
        (dict(engine=5), -4, "engine"),
        (dict(engine=L.ENGINE_SIMT, flags=1 << 16, hidden_dim=96), -4, "engine"),   # the engine is checked first
        (dict(flags=1 << 16), -7, "not defined"),
        (dict(flags=512, hidden_dim=96), -7, "not defined"),
        (dict(flags=L.STASH), -6, "NNB_STASH"),
        (dict(flags=L.HVP), -6, "NNB_HVP"),
        (dict(flags=L.STASH | L.HVP, N=-1), -6, "NNB_STASH"),
        (dict(hidden_dim=96), -8, "hidden_dim"),
        (dict(hidden_dim=96, N=-1), -8, "hidden_dim"),
        (dict(N=-1), -3, "negative"),
    ]
    for kw, code, word in cases:
        a = L.RenderArgs()
        a.N = 10; a.S = 1; a.flags = 0; a.engine = L.ENGINE_TC; a.hidden_dim = 256
        for k, v in kw.items():
            setattr(a, k, v)
        rc = L.lib.nnb_field_hvp_tc(C.byref(a), None, None, None, None)
        assert rc == code and word in err(), (kw, rc, err())
    a = L.RenderArgs()
    a.N = 0; a.S = 1; a.engine = L.ENGINE_TC
    assert L.lib.nnb_field_hvp_tc(C.byref(a), None, None, None, None) == 0
    # past N == 0: the pointers (pts, weights, u, and at least one of g_pts / g_weights), before the workspace
    buf = (C.c_float * 64)()
    addr = C.addressof(buf)
    a = L.RenderArgs()
    a.N = 4; a.S = 1; a.engine = L.ENGINE_TC; a.hidden_dim = 64; a.pts = addr; a.weights = addr
    assert L.lib.nnb_field_hvp_tc(C.byref(a), None, addr, None, None) == -3 and "u" in err()
    assert L.lib.nnb_field_hvp_tc(C.byref(a), addr, None, None, None) == -3 and "g_pts, g_weights" in err()
    assert L.lib.nnb_field_hvp_tc(C.byref(a), addr, addr + 4, None, None) == -3 and "aligned" in err()
    assert L.lib.nnb_field_hvp_tc(C.byref(a), addr, None, addr + 2, None) == -3 and "g_weights" in err()
    assert L.lib.nnb_field_hvp_tc(C.byref(a), addr, addr, None, None) == -5 and "workspace" in err()


class _Recorder:
    """replaces the ways field_normal can run (the exact engine's autograd function, the detached tensor-core normals, the tensor-core
    autograd function) and records which one a call took"""

    def __init__(self, monkeypatch):
        from nope_nerf_b200 import field, ops
        self.calls = []
        monkeypatch.setattr(ops, "_need_cuda", lambda *a, **k: None)
        monkeypatch.setattr(field._GradFn, "apply", lambda net, flat, p, *ps: (self.calls.append("simt"), p * 0.0)[1])
        monkeypatch.setattr(field._GradTcFn, "apply", lambda net, flat, p, *ps: (self.calls.append("tc_grad"), p * 0.0)[1])
        monkeypatch.setattr(field, "_normal_tc", lambda net, p: (self.calls.append("tc"), torch.zeros(p.shape[0], 3))[1])


def test_grad_engine_routing(monkeypatch):
    from nope_nerf_b200 import field
    rec = _Recorder(monkeypatch)
    net = _net()
    p = torch.zeros(5, 3, requires_grad=True)
    cases = [
        (dict(), "simt"), (dict(engine="tc"), "simt"), (dict(engine="tc", grad_engine=None), "simt"),
        (dict(engine="tc", grad_engine="simt"), "simt"), (dict(engine=L.ENGINE_TC, grad_engine=L.ENGINE_SIMT), "simt"),
        (dict(engine="tc", grad_engine="tc"), "tc_grad"), (dict(engine=L.ENGINE_TC, grad_engine=L.ENGINE_TC), "tc_grad"),
        (dict(engine=None, grad_engine="simt"), "simt"),
    ]
    for kw, want in cases:
        rec.calls.clear()
        field.field_normal(net, p, **kw)
        assert rec.calls == [want], (kw, rec.calls)
        rec.calls.clear()
        net.gradient_grad(p, 0, **kw)
        assert rec.calls == [want], (kw, rec.calls)
    # no graph needed: the detached normals, whatever grad_engine says
    with torch.no_grad():
        for kw in (dict(engine="tc"), dict(engine="tc", grad_engine="tc")):
            rec.calls.clear()
            field.field_normal(net, p, **kw)
            net.gradient_grad(p, 0, **kw)
            assert rec.calls == ["tc", "tc"], (kw, rec.calls)
    # gradient() is gradient_grad with grad_engine=None: a call that needs the graph runs on the exact engine
    rec.calls.clear()
    net.gradient(p, 0, engine="tc")
    net.gradient(p.detach(), 0, engine="tc")
    assert rec.calls == ["simt", "tc"]


def test_grad_engine_tc_needs_engine_tc(monkeypatch):
    from nope_nerf_b200 import field
    rec = _Recorder(monkeypatch)
    net = _net()
    p = torch.zeros(5, 3, requires_grad=True)
    for kw in (dict(grad_engine="tc"), dict(engine=None, grad_engine=L.ENGINE_TC), dict(engine="simt", grad_engine="tc"),
               dict(engine=L.ENGINE_SIMT, grad_engine="tc")):
        with pytest.raises(ValueError, match="grad_engine"):
            field.field_normal(net, p, **kw)
        with pytest.raises(ValueError, match="grad_engine"):
            net.gradient_grad(p, 0, **kw)
        with torch.no_grad(), pytest.raises(ValueError, match="grad_engine"):   # whether or not the call needs the graph
            net.gradient_grad(p, 0, **kw)
        with pytest.raises(ValueError, match="grad_engine"):                    # and for no point at all
            field.field_normal(net, p[:0], **kw)
    for bad in ("cuda", "TC", 2):
        with pytest.raises(ValueError):
            field.field_normal(net, p, engine="tc", grad_engine=bad)
    assert rec.calls == []


def test_renderer_normal_grad_engine(monkeypatch):
    """Renderer(normal_grad_engine='tc') needs normal_engine='tc'; _normal_diff then passes both engines to gradient_grad, and without it
    calls gradient(pp, it) as before"""
    import nope_nerf_b200.model as mdl
    from _fullsize_cases import default_cfg
    cfg = default_cfg()
    net = _net()
    for kw in (dict(normal_grad_engine="tc"), dict(normal_engine="simt", normal_grad_engine="tc")):
        with pytest.raises(ValueError, match="grad_engine"):
            mdl.Renderer(net, cfg["rendering"], **kw)
    seen = []
    monkeypatch.setattr(type(net), "gradient", lambda self, p, it, engine=None: (seen.append(("gradient", engine)), p[:, None] * 0)[1])
    monkeypatch.setattr(type(net), "gradient_grad",
                        lambda self, p, it, engine=None, grad_engine=None: (seen.append(("gradient_grad", engine, grad_engine)), p[:, None] * 0)[1])
    pix = torch.zeros(3, 2); depth = torch.ones(3); c2w = torch.eye(4); cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0]))
    m = torch.ones(3, dtype=torch.bool)
    for kw, want in ((dict(), ("gradient", None)), (dict(normal_engine="tc"), ("gradient", None)),
                     (dict(normal_engine="tc", normal_grad_engine="simt"), ("gradient_grad", "tc", "simt")),
                     (dict(normal_engine="tc", normal_grad_engine="tc"), ("gradient_grad", "tc", "tc"))):
        seen.clear()
        rend = mdl.Renderer(net, cfg["rendering"], **kw)
        rend._normal_diff(pix, depth, c2w, cam, m, 0, torch.zeros(3, 3))
        assert seen == [want], (kw, seen)


def test_third_derivative_raises(monkeypatch):
    """_GradTcFn is differentiable once: its backward calls nnb_field_hvp_tc, and differentiating that backward raises"""
    from nope_nerf_b200 import field, ops
    calls = []
    monkeypatch.setattr(ops, "_need_cuda", lambda *a, **k: None)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    monkeypatch.setattr(field, "_normal_tc", lambda net, p: torch.sin(p))
    monkeypatch.setattr(L.lib, "nnb_field_hvp_tc", lambda *a: (calls.append(a), 0)[1])
    net = _net()
    p = torch.rand(6, 3, requires_grad=True)
    n = field.field_normal(net, p, engine="tc", grad_engine="tc")
    assert type(n.grad_fn).__name__ == "_GradTcFnBackward"
    g, = torch.autograd.grad(n.sum(), p, create_graph=True)
    assert len(calls) == 1 and g.shape == (6, 3)
    with pytest.raises(RuntimeError):
        g.sum().backward()


def test_defaults_are_none():
    from nope_nerf_b200 import field
    from nope_nerf_b200.model.official_nerf import OfficialStaticNerf
    assert inspect.signature(field.field_normal).parameters["grad_engine"].default is None
    assert inspect.signature(OfficialStaticNerf.gradient_grad).parameters["grad_engine"].default is None
    assert inspect.signature(OfficialStaticNerf.gradient_grad).parameters["engine"].default is None

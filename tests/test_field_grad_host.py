"""Host side of nnb_field_grad (the tensor-core backward of explicit-point field queries, with weight gradients): the workspace rule, the
ctypes bindings, and the grad_engine rules of field_query_grad / OfficialStaticNerf.forward / infer_occ, with the default routing unchanged.
Needs no device: the library calls are replaced by recorders."""
import ctypes as C
import inspect

import pytest
import torch

from nope_nerf_b200 import _lib as L

TILE = 128


def _align(x, a=256):
    return (x + a - 1) // a * a


def expected_bytes(N, occ, D):
    """the documented layout: nnb_render_bwd's stash layout at N x 1 samples on NNB_ENGINE_TC | the forward weight image (the
    occupancy-only prefix when occ) | the transposed weight image (its trunk part when occ), each 256-byte aligned"""
    ks = D // 16
    stage = 64 * D
    n_fwd = 4 + 3 * ks + (4 + ks) + 3 * ks + ks + ks
    img_ray = (n_fwd - ks) * stage + ks * stage // 2                       # the render's forward image
    img_pts = img_ray + 2 * stage // 2                                     # + the two direction stages of the points mode
    img_occ = (n_fwd - 2 * ks) * stage
    img_t = 34 * D * D + 576 * D
    prefix_t = (D // 32) * 32 * 64 + (D // 32 + ks) * stage
    stash = L.lib.nnb_workspace_bytes_dim(N, 1, L.STASH, L.ENGINE_TC, D) - _align(img_ray) - _align(img_t)   # make_layout's part
    return stash + (_align(img_occ) + _align(img_t - prefix_t) if occ else _align(img_pts) + _align(img_t))


def per_point_bytes(D):
    """layout bytes per point: record, three float4 adjoints, the per-ray reductions of the render backward (64 bytes, unused here),
    h0..h7 / feat / hr, enc, denc, their dY, dyc and the gate bits"""
    return 32 + 48 + 64 + 2 * (9 * D + D // 2) * 4 + 64 * 4 + 32 * 4 + 16 + D + D // 16


def test_workspace_matches_its_formula():
    for N in (1, 127, 128, 129, 4096, 16901, 131072, 200003, 3500000):
        for D in L.HIDDEN_DIMS:
            for flags, occ in ((0, False), (L.SOFTPLUS | L.DIST_ALPHA, False), (L.RAW_DENSITY, False), (L.RAW_DENSITY | L.OCC_ONLY, True),
                               (L.OCC_ONLY | L.SOFTPLUS, True)):
                assert L.lib.nnb_field_grad_workspace_bytes(N, flags, D) == expected_bytes(N, occ, D), (N, D, flags)
        assert L.lib.nnb_field_grad_workspace_bytes(N, 0, 0) == expected_bytes(N, False, 256)   # 0 means 256


def test_workspace_grows_by_the_stash_row():
    """the size grows by the stash's bytes per point (20 272 at D = 256) with N; 131 072 points at D = 256 take about 2.7 GB"""
    for D in L.HIDDEN_DIMS:
        for flags in (0, L.OCC_ONLY):
            a, b = L.lib.nnb_field_grad_workspace_bytes(2 * 131072, flags, D), L.lib.nnb_field_grad_workspace_bytes(131072, flags, D)
            assert abs((a - b) - 131072 * per_point_bytes(D)) <= 20 * 256, (D, flags)
    assert per_point_bytes(256) == 20272
    assert 2.6e9 < L.lib.nnb_field_grad_workspace_bytes(131072, 0, 256) < 2.8e9
    assert L.lib.nnb_field_grad_workspace_bytes(131072, 0, 256) == 2700501248


def test_workspace_query_rejects_undefined_bits_widths_and_sizes():
    for bit in (512, 1024, 4096, 8192, 1 << 16, 1 << 31):
        for D in (0,) + L.HIDDEN_DIMS:
            assert L.lib.nnb_field_grad_workspace_bytes(1000, bit, D) == 0
    for D in (1, 32, 96, 192, 255, 512, -256):
        assert L.lib.nnb_field_grad_workspace_bytes(1000, 0, D) == 0
    assert L.lib.nnb_field_grad_workspace_bytes(0, 0, 256) == 0 and L.lib.nnb_field_grad_workspace_bytes(-1, 0, 256) == 0


def test_bindings():
    assert L.lib.nnb_field_grad_workspace_bytes.restype is C.c_size_t
    assert L.lib.nnb_field_grad_workspace_bytes.argtypes == [C.c_int32, C.c_uint32, C.c_int32]
    assert L.lib.nnb_field_grad.argtypes == [C.POINTER(L.RenderArgs)] + [C.c_void_p] * 6


def test_rejections_need_no_device():
    """the argument checks that come before any device work: a NULL args, the engine, undefined and rejected flags, the width, N < 0,
    g_dirs with NNB_OCC_ONLY; N == 0 succeeds without touching anything"""
    err = lambda: L.lib.nnb_last_error().decode()
    assert L.lib.nnb_field_grad(None, None, None, None, None, None, None) == -3
    cases = [
        (dict(engine=L.ENGINE_SIMT), {}, -4, "engine"),
        (dict(engine=5), {}, -4, "engine"),
        (dict(flags=1 << 16), {}, -7, "not defined"),
        (dict(flags=512), {}, -7, "not defined"),
        (dict(flags=L.STASH), {}, -6, "NNB_STASH"),
        (dict(flags=L.HVP), {}, -6, "NNB_HVP"),
        (dict(hidden_dim=96), {}, -8, "hidden_dim"),
        (dict(N=-1), {}, -3, "negative"),
        (dict(flags=L.OCC_ONLY), dict(g_dirs=16), -6, "g_dirs"),
    ]
    for kw, ptrs, code, word in cases:
        a = L.RenderArgs()
        a.N = 10; a.S = 1; a.flags = 0; a.engine = L.ENGINE_TC; a.hidden_dim = 256
        for k, v in kw.items():
            setattr(a, k, v)
        rc = L.lib.nnb_field_grad(C.byref(a), None, None, None, ptrs.get("g_dirs"), None, None)
        assert rc == code and word in err(), (kw, rc, err())
    a = L.RenderArgs()
    a.N = 0; a.S = 1; a.engine = L.ENGINE_TC
    assert L.lib.nnb_field_grad(C.byref(a), None, None, None, None, None, None) == 0


def _net(D=64):
    import nope_nerf_b200.model as mdl
    from _fullsize_cases import default_cfg
    cfg = default_cfg(); cfg["model"]["hidden_dim"] = D
    torch.manual_seed(0)
    return mdl.OfficialStaticNerf(cfg)


class _Recorder:
    """replaces the three ways field_query can run (the exact engine's autograd function, the tensor-core query, the tensor-core autograd
    function) and records which one a call took"""

    def __init__(self, monkeypatch):
        from nope_nerf_b200 import field, ops
        self.calls = []
        out = lambda M: (torch.zeros(M, 3), torch.zeros(M))
        monkeypatch.setattr(ops, "_need_cuda", lambda *a, **k: None)
        monkeypatch.setattr(field._FieldFn, "apply", lambda flags, net, flat, p, d, *ps: (self.calls.append(("simt", flags)), out(p.shape[0]))[1])
        monkeypatch.setattr(field._FieldTcFn, "apply", lambda flags, net, flat, p, d, *ps: (self.calls.append(("tc_grad", flags)), out(p.shape[0]))[1])
        monkeypatch.setattr(field, "_field_tc", lambda net, flags, p, d: (self.calls.append(("tc", flags)), torch.zeros(p.shape[0], 4))[1])


def test_grad_engine_routing(monkeypatch):
    from nope_nerf_b200 import field
    rec = _Recorder(monkeypatch)
    net = _net()
    p = torch.zeros(5, 3); d = torch.ones(5, 3)
    # grad mode on and parameters requiring grad: a call that needs a gradient
    cases = [
        (dict(), "simt"), (dict(engine="tc"), "simt"), (dict(engine="tc", grad_engine=None), "simt"),
        (dict(engine="tc", grad_engine="simt"), "simt"), (dict(engine=L.ENGINE_TC, grad_engine=L.ENGINE_SIMT), "simt"),
        (dict(engine="tc", grad_engine="tc"), "tc_grad"), (dict(engine=L.ENGINE_TC, grad_engine=L.ENGINE_TC), "tc_grad"),
        (dict(engine=None, grad_engine="simt"), "simt"),
    ]
    for kw, want in cases:
        rec.calls.clear()
        field.field_query_grad(net, p, d, **kw)
        assert [c[0] for c in rec.calls] == [want], (kw, rec.calls)
    # occupancy only: the flag reaches the tensor-core backward
    rec.calls.clear()
    field.field_query_grad(net, p, None, raw_density=True, occ_only=True, engine="tc", grad_engine="tc")
    assert [c[0] for c in rec.calls] == ["tc_grad"] and rec.calls[0][1] & L.OCC_ONLY and rec.calls[0][1] & L.RAW_DENSITY, rec.calls
    # no gradient needed: the inference query, whatever grad_engine says
    with torch.no_grad():
        for kw in (dict(engine="tc"), dict(engine="tc", grad_engine="tc")):
            rec.calls.clear()
            field.field_query_grad(net, p, d, **kw)
            assert [c[0] for c in rec.calls] == ["tc"], (kw, rec.calls)
        rec.calls.clear()
        field.field_query_grad(net, p, d)
        assert [c[0] for c in rec.calls] == ["simt"]


def test_grad_engine_tc_needs_engine_tc(monkeypatch):
    from nope_nerf_b200 import field
    rec = _Recorder(monkeypatch)
    net = _net()
    p = torch.zeros(5, 3)
    for kw in (dict(grad_engine="tc"), dict(engine=None, grad_engine=L.ENGINE_TC), dict(engine="simt", grad_engine="tc"),
               dict(engine=L.ENGINE_SIMT, grad_engine="tc")):
        with pytest.raises(ValueError, match="grad_engine"):
            field.field_query_grad(net, p, None, **kw)
        with pytest.raises(ValueError, match="grad_engine"):
            net(p, torch.ones(5, 3), **kw)
        with pytest.raises(ValueError, match="grad_engine"):
            net.infer_occ(p, **kw)
        with torch.no_grad(), pytest.raises(ValueError, match="grad_engine"):   # whether or not the call needs a gradient
            field.field_query_grad(net, p, None, **kw)
        with pytest.raises(ValueError, match="grad_engine"):                    # and for no point at all
            field.field_query_grad(net, p[:0], None, **kw)
    for bad in ("cuda", "TC", 2):
        with pytest.raises(ValueError):
            field.field_query_grad(net, p, None, engine="tc", grad_engine=bad)
    assert rec.calls == []


def test_model_passes_grad_engine(monkeypatch):
    rec = _Recorder(monkeypatch)
    net = _net()
    p = torch.zeros(5, 3)
    net(p, torch.ones(5, 3), return_addocc=True, engine="tc", grad_engine="tc")
    net(p, None, only_occupancy=True, engine="tc", grad_engine="tc")
    net.infer_occ(p, engine="tc", grad_engine="tc")
    assert [c[0] for c in rec.calls] == ["tc_grad"] * 3
    assert rec.calls[1][1] & L.OCC_ONLY and rec.calls[2][1] & L.OCC_ONLY and rec.calls[2][1] & L.RAW_DENSITY
    assert not rec.calls[0][1] & L.OCC_ONLY
    rec.calls.clear()
    net(p, torch.ones(5, 3), engine="tc")
    net.infer_occ(p, engine="tc")
    assert [c[0] for c in rec.calls] == ["simt"] * 2


def test_defaults_are_none():
    from nope_nerf_b200 import field
    from nope_nerf_b200.model.official_nerf import OfficialStaticNerf
    assert inspect.signature(field.field_query_grad).parameters["grad_engine"].default is None
    assert "grad_engine" not in inspect.signature(field.field_query).parameters   # field_query keeps its signature: grad_engine=None
    assert inspect.signature(OfficialStaticNerf.forward).parameters["grad_engine"].default is None
    assert inspect.signature(OfficialStaticNerf.infer_occ).parameters["grad_engine"].default is None
    assert inspect.signature(OfficialStaticNerf.infer_occ).parameters["engine"].default is None
    assert "grad_engine" not in inspect.signature(OfficialStaticNerf.gradient).parameters   # gradient() is unchanged


def test_field_query_is_field_query_grad_without_grad_engine(monkeypatch):
    """field_query routes exactly as field_query_grad with grad_engine=None"""
    from nope_nerf_b200 import field
    rec = _Recorder(monkeypatch)
    net = _net()
    p = torch.zeros(5, 3); d = torch.ones(5, 3)
    for kw in (dict(), dict(engine="tc"), dict(engine="simt"), dict(engine="tc", occ_only=True)):
        rec.calls.clear()
        field.field_query(net, p, d, **kw)
        a = list(rec.calls)
        rec.calls.clear()
        field.field_query_grad(net, p, d, grad_engine=None, **kw)
        assert a == rec.calls and [c[0] for c in a] == ["simt"], (kw, a)

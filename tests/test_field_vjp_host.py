"""Host side of nnb_field_vjp (the tensor-core data gradient of explicit-point field queries): the workspace rule, the ctypes bindings
and the Python defaults.  Needs no device."""
import inspect

from nope_nerf_b200 import _lib as L

TILE = 128


def _align(x, a=256):
    return (x + a - 1) // a * a


def expected_bytes(N, occ, D):
    """the documented layout: records | gate bits | forward weight image | transposed weight image, each 256-byte aligned"""
    npad = (N + TILE - 1) // TILE * TILE
    ks = D // 16
    stage = 64 * D                                                         # D rows x 16 k x (hi + lo) 16-bit
    n_fwd = 4 + 3 * ks + (4 + ks) + 3 * ks + ks + ks                       # ray-mode forward stages; the last KS are D/2 rows wide
    img_fwd = (n_fwd - ks) * stage + ks * stage // 2 + 2 * stage // 2      # + the two direction stages of the points mode
    img_occ = (n_fwd - 2 * ks) * stage                                     # up to the density head
    img_t = 34 * D * D + 576 * D
    prefix_t = (D // 32) * 32 * 64 + (D // 32 + ks) * stage                # g_de, g_feat, W_feat
    gates = npad * D + (0 if occ else npad * D // 16)
    return (_align(32 * npad) + _align(gates) + _align(img_occ if occ else img_fwd)
            + _align(img_t - prefix_t if occ else img_t))


def test_workspace_matches_its_formula():
    for N in (1, 127, 128, 129, 4096, 16901, 200003, 3500000):
        for D in L.HIDDEN_DIMS:
            for flags, occ in ((0, False), (L.SOFTPLUS | L.DIST_ALPHA, False), (L.RAW_DENSITY | L.OCC_ONLY, True), (L.OCC_ONLY, True)):
                assert L.lib.nnb_field_vjp_workspace_bytes(N, flags, D) == expected_bytes(N, occ, D), (N, D, flags)
        assert L.lib.nnb_field_vjp_workspace_bytes(N, 0, 0) == expected_bytes(N, False, 256)   # 0 means 256


def test_occupancy_only_workspace_is_smaller():
    for D in L.HIDDEN_DIMS:
        assert L.lib.nnb_field_vjp_workspace_bytes(65536, L.RAW_DENSITY | L.OCC_ONLY, D) < L.lib.nnb_field_vjp_workspace_bytes(65536, L.RAW_DENSITY, D)
    # the largest call the geometry view makes (65 536 surface points at D = 256) stays far below 1 GB
    assert L.lib.nnb_field_vjp_workspace_bytes(65536, L.RAW_DENSITY | L.OCC_ONLY, 256) < 64 << 20


def test_workspace_query_rejects_undefined_bits_widths_and_sizes():
    for bit in (512, 1024, 4096, 8192, 1 << 16, 1 << 31):
        for D in (0,) + L.HIDDEN_DIMS:
            assert L.lib.nnb_field_vjp_workspace_bytes(1000, bit, D) == 0
            assert L.lib.nnb_field_vjp_workspace_bytes(1000, bit | L.OCC_ONLY, D) == 0
    for D in (1, 32, 96, 192, 255, 512, -256):
        assert L.lib.nnb_field_vjp_workspace_bytes(1000, 0, D) == 0
    assert L.lib.nnb_field_vjp_workspace_bytes(0, 0, 256) == 0 and L.lib.nnb_field_vjp_workspace_bytes(-1, 0, 256) == 0


def test_bindings():
    import ctypes as C
    assert L.lib.nnb_field_vjp_workspace_bytes.restype is C.c_size_t
    assert L.lib.nnb_field_vjp_workspace_bytes.argtypes == [C.c_int32, C.c_uint32, C.c_int32]
    assert L.lib.nnb_field_vjp.argtypes == [C.POINTER(L.RenderArgs), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    assert L.lib.nnb_version() == 105


def test_engine_defaults_are_none():
    from nope_nerf_b200 import field
    from nope_nerf_b200.model.official_nerf import OfficialStaticNerf
    from nope_nerf_b200.model import rendering
    assert inspect.signature(OfficialStaticNerf.gradient).parameters["engine"].default is None
    assert inspect.signature(field.field_normal).parameters["engine"].default is None
    assert rendering.GEOMETRY_CHUNK == 1024   # the reference's chunk; see rendering.py for why no engine raises it

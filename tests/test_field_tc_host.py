"""Host side of the tensor-core field query: the workspace rule of nnb_field_fwd on NNB_ENGINE_TC is nnb_workspace_bytes_dim(N, 1, flags,
NNB_ENGINE_TC, hidden_dim), and adding the engine changed no size that function returns.  The weight image of the points mode is
64 * hidden_dim bytes longer than the render's; it extends into the transposed-image region that already follows it.  Needs no device."""
from nope_nerf_b200 import _lib as L

# (N, S, flags, engine, hidden_dim, bytes) as returned by library version 102
PINNED = [
    (1, 1, 0, 0, 64, 4096),
    (1, 1, 0, 0, 128, 4096),
    (1, 1, 0, 0, 256, 4096),
    (1, 1, 0, 0, 0, 4096),
    (1, 1, 0, 1, 64, 352256),
    (1, 1, 0, 1, 128, 1257472),
    (1, 1, 0, 1, 256, 4739072),
    (1, 1, 0, 1, 0, 4739072),
    (1, 1, 256, 0, 64, 7430912),
    (1, 1, 256, 0, 128, 11985408),
    (1, 1, 256, 0, 256, 21881344),
    (1, 1, 256, 0, 0, 21881344),
    (1, 1, 256, 1, 64, 7787776),
    (1, 1, 256, 1, 128, 13256192),
    (1, 1, 256, 1, 256, 26651136),
    (1, 1, 256, 1, 0, 26651136),
    (1, 1, 16640, 0, 64, 7725824),
    (1, 1, 16640, 0, 128, 12542464),
    (1, 1, 16640, 0, 256, 22962688),
    (1, 1, 16640, 0, 0, 22962688),
    (1, 1, 16640, 1, 64, 7787776),
    (1, 1, 16640, 1, 128, 13256192),
    (1, 1, 16640, 1, 256, 26651136),
    (1, 1, 16640, 1, 0, 26651136),
    (4096, 1, 0, 0, 64, 131072),
    (4096, 1, 0, 0, 128, 131072),
    (4096, 1, 0, 0, 256, 131072),
    (4096, 1, 0, 1, 64, 479232),
    (4096, 1, 0, 1, 128, 1384448),
    (4096, 1, 0, 1, 256, 4866048),
    (4096, 1, 256, 0, 64, 28897792),
    (4096, 1, 256, 0, 128, 52752640),
    (4096, 1, 256, 0, 256, 101249280),
    (4096, 1, 256, 1, 64, 29524480),
    (4096, 1, 256, 1, 128, 54563072),
    (4096, 1, 256, 1, 256, 107098368),
    (4096, 1, 16640, 0, 64, 38334976),
    (4096, 1, 16640, 0, 128, 70578432),
    (4096, 1, 16640, 0, 256, 135852288),
    (4096, 1, 16640, 1, 64, 29524480),
    (4096, 1, 16640, 1, 128, 54563072),
    (4096, 1, 16640, 1, 256, 107098368),
    (3500000, 1, 0, 0, 64, 112001024),
    (3500000, 1, 0, 0, 128, 112001024),
    (3500000, 1, 0, 0, 256, 112001024),
    (3500000, 1, 0, 1, 64, 112349184),
    (3500000, 1, 0, 1, 128, 113254400),
    (3500000, 1, 0, 1, 256, 116736000),
    (3500000, 1, 256, 0, 64, 18934917632),
    (3500000, 1, 256, 0, 128, 35963005184),
    (3500000, 1, 256, 0, 256, 70039296256),
    (3500000, 1, 256, 1, 64, 19173267968),
    (3500000, 1, 256, 1, 128, 36440262912),
    (3500000, 1, 256, 1, 256, 70996039936),
    (3500000, 1, 16640, 0, 64, 26998991360),
    (3500000, 1, 16640, 0, 128, 51195144448),
    (3500000, 1, 16640, 0, 256, 99607566592),
    (3500000, 1, 16640, 1, 64, 19173267968),
    (3500000, 1, 16640, 1, 128, 36440262912),
    (3500000, 1, 16640, 1, 256, 70996039936),
    (1024, 128, 0, 0, 64, 4194304),
    (1024, 128, 0, 0, 128, 4194304),
    (1024, 128, 0, 0, 256, 4194304),
    (1024, 128, 0, 1, 64, 4542464),
    (1024, 128, 0, 1, 128, 5447680),
    (1024, 128, 0, 1, 256, 8929280),
    (1024, 128, 256, 0, 64, 707260928),
    (1024, 128, 256, 0, 128, 1348727040),
    (1024, 128, 256, 0, 256, 2651775232),
    (1024, 128, 256, 1, 64, 716521984),
    (1024, 128, 256, 1, 128, 1367806208),
    (1024, 128, 256, 1, 256, 2692161792),
    (1024, 128, 16640, 0, 64, 1009250816),
    (1024, 128, 16640, 0, 128, 1919152384),
    (1024, 128, 16640, 0, 256, 3759071488),
    (1024, 128, 16640, 1, 64, 716521984),
    (1024, 128, 16640, 1, 128, 1367806208),
    (1024, 128, 16640, 1, 256, 2692161792),
    (64, 1024, 0, 0, 64, 2097152),
    (64, 1024, 0, 0, 128, 2097152),
    (64, 1024, 0, 0, 256, 2097152),
    (64, 1024, 0, 1, 64, 2445312),
    (64, 1024, 0, 1, 128, 3350528),
    (64, 1024, 0, 1, 256, 6832128),
    (64, 1024, 256, 0, 64, 356975104),
    (64, 1024, 256, 0, 128, 679674112),
    (64, 1024, 256, 0, 256, 1345188096),
    (64, 1024, 256, 1, 64, 361779712),
    (64, 1024, 256, 1, 128, 689840384),
    (64, 1024, 256, 1, 256, 1367748864),
    (64, 1024, 16640, 0, 64, 507970048),
    (64, 1024, 16640, 0, 128, 964886784),
    (64, 1024, 16640, 0, 256, 1898836224),
    (64, 1024, 16640, 1, 64, 361779712),
    (64, 1024, 16640, 1, 128, 689840384),
    (64, 1024, 16640, 1, 256, 1367748864),
]


def test_workspace_sizes_are_those_of_version_102():
    for N, S, flags, engine, D, nbytes in PINNED:
        assert L.lib.nnb_workspace_bytes_dim(N, S, flags, engine, D) == nbytes, (N, S, flags, engine, D)
    for N, S, flags, engine, D, nbytes in PINNED:
        if D == 256:
            assert L.lib.nnb_workspace_bytes(N, S, flags, engine) == nbytes


def test_occ_only_does_not_change_the_workspace():
    for N in (1, 4096, 3500000):
        for D in L.HIDDEN_DIMS:
            for engine in (L.ENGINE_SIMT, L.ENGINE_TC):
                assert L.lib.nnb_workspace_bytes_dim(N, 1, L.SOFTPLUS | L.OCC_ONLY, engine, D) == L.lib.nnb_workspace_bytes_dim(N, 1, L.SOFTPLUS, engine, D)


def test_version_and_flag():
    assert L.lib.nnb_version() == 105
    assert L.OCC_ONLY == 32768 and L.OCC_ONLY & (L.HVP | L.RAW_DENSITY | L.STASH) == 0


REMOVED_FLAG_BITS = (512, 1024, 4096, 8192)   # flags defined before version 105


def test_undefined_flag_bits_size_no_workspace():
    for bit in REMOVED_FLAG_BITS + (1 << 16, 1 << 31):
        for flags in (bit, bit | L.STASH, bit | L.STASH | L.SOFTPLUS):
            for engine in (L.ENGINE_SIMT, L.ENGINE_TC):
                for D in (0,) + L.HIDDEN_DIMS:
                    assert L.lib.nnb_workspace_bytes_dim(64, 32, flags, engine, D) == 0, (flags, engine, D)
                assert L.lib.nnb_workspace_bytes(64, 32, flags, engine) == 0, (flags, engine)


def test_field_query_signature():
    import inspect
    from nope_nerf_b200 import field
    from nope_nerf_b200.model.official_nerf import OfficialStaticNerf
    sig = inspect.signature(field.field_query)
    assert list(sig.parameters) == ["net", "p", "ray_d", "raw_density", "occ_only", "engine"]
    assert sig.parameters["engine"].default is None and sig.parameters["occ_only"].default is False
    assert inspect.signature(OfficialStaticNerf.forward).parameters["engine"].default is None
    assert inspect.signature(OfficialStaticNerf.infer_occ).parameters["engine"].default is None
    assert field._engine_id(None) is None and field._engine_id("tc") == L.ENGINE_TC and field._engine_id("simt") == L.ENGINE_SIMT

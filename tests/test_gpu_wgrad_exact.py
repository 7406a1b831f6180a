"""Exact check of the weight-gradient stage of both engines on planted stashes.

nnb_debug_wgrad runs the weight-gradient stage of nnb_render_bwd (tc_wgrad_all on the tensor-core engine, simt_wgrad_all on the SIMT
engine) alone, on whatever the workspace's stash holds.  Here every stash region the stage reads (h0..h7, feat, hr, enc, denc, dy0..dy7,
dfeat, dyr, dyc) holds small integers built on the device from sample and column indices: dY in {-1, 0, 1}, X in {-2, ..., 2}.  They are
exact as bf16 hi halves (lo = 0) and as fp32, every product is exact, and every partial sum stays within 2 M <= 2^19 < 2^24 for
M <= 262 144, so whatever the split, chunk or reduction order, each gradient must equal the float64 dY^T X / sum dY bit for bit.  A
counting variant (dY = X = 1: every dW and db equals M) turns a mismatch into a readable number of samples counted.

The rest of the workspace, the stash rows [M, Mpad), column 63 of enc and columns 27..31 of denc are NaN: the stage must not read a
padded row or column, and every partial it reduces must have been stored (an empty split stores zeros).  g_weights starts from an
integer base (the stage accumulates, +=) and is followed by a guard tail that must stay untouched.

The sizes sit on the edges of the split arithmetic; `edges` mirrors the formulas of nnb_tc.cu (tc_wgrad_all, launch_wgrad),
nnb_simt.cu (launch_head_wgrad, head_wgrad, simt_wgrad) and nnb_workspace.cuh, and the host test asserts that each case hits the edge it
names."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
from test_gpu_relu_mask import layout

DIMS = (64, 128, 256)
# (N, S): M = N * S, and the edge of the split arithmetic it sits on
CASES = {
    (33, 31): "ms_big 1",                  # M = 1023: one split of the D-wide jobs
    (64, 16): "ms_big full",               # M = 1024: 2048 / D splits
    (89, 23): "ms_enc 1, head splits 1",   # M = 2047
    (128, 16): "ms_enc 32, head splits 1",
    (3, 683): "ms_enc 32, head splits 2",  # M = 2049
    (55, 20): "splits 6, 7 empty at D = 256",   # M = 1100
    (301, 17): "ragged",                   # M = 5117
    (288, 128): "encoding after the reduce at D = 256",   # M = 36 864
    (289, 128): "encoding chained at D = 256",            # M = 36 992
    (1000, 37): "last split ends inside a 32-sample chunk",   # M = 37 000
    (1024, 128): "C2 size",
    (8193, 16): "head splits capped at 64, 2064-sample chunk",   # M = 131 088
    (512, 512): "largest",                 # M = 262 144
}
SIMT_CASES = {(256, 16): "simt splits 1", (17, 241): "simt splits 2"}   # M = 4096 / 4097
PARAMS = [("tc", D, N, S) for D in DIMS for (N, S) in CASES] + \
         [("simt", D, N, S) for D in DIMS for (N, S) in list(CASES) + list(SIMT_CASES)]
GUARD = 1024
SENTINEL = -12345.25


# -------------------------------------------------------------------------------------------------------- split arithmetic mirror
def _ceil(a, b):
    return (a + b - 1) // b


def tc_msplit(M, D):
    """ms_big / ms_enc of tc_wgrad_all (nnb_tc.cu: `const int ms_big = L.M >= 8 * 128 ? ...`, tc_wgrad_msplit_big)"""
    return (2048 // D if M >= 8 * 128 else 1), (32 if M >= 32 * 64 else 1)


def tc_split_ranges(M, msplit):
    """sample range of each split of launch_wgrad / wgrad_body: per_cta rounded up to 64-sample blocks, s_end clamped to M"""
    per = _ceil(_ceil(M, msplit), 64) * 64
    return [(min(y * per, M), min(y * per + per, M)) for y in range(msplit)]


def head_msplit(M):
    """jobs_wgrad_msplit (nnb_workspace.cuh), the split count of head_wgrad"""
    return min(max(_ceil(M, 2048), 1), 64)


def head_chunk(M):
    """samples per split of head_wgrad and simt_wgrad: ceil(M / msplit) rounded up to 16"""
    return _ceil(_ceil(M, head_msplit(M)), 16) * 16


def simt_msplit(M):
    """simt_wgrad_msplit (nnb_workspace.cuh)"""
    return min(max(_ceil(M, 4096), 1), 16)


def wpart_floats(M, D):
    """wpart_floats (nnb_workspace.cuh)"""
    from nope_nerf_b200 import _lib as L
    np_ = L.num_params(D)
    return max(simt_msplit(M) * (np_ + 8192), (2048 // D) * (np_ + 8192), head_msplit(M) * 8192)


def enc_chained(M, D):
    """tc_wgrad_all: the encoding jobs chain before the reduce when their partials fit behind the D-wide, rgb and head regions"""
    ms_big, ms_enc = tc_msplit(M, D)
    DR = D // 2
    big_f = 8 * (D * D + 2 * D) * ms_big + (DR * D + 2 * DR) * ms_big
    head_f = ((D + 1) + (DR * 27 + DR) + (3 * DR + 3)) * head_msplit(M)
    enc_f = 2 * (D * 63 + 2 * D) * ms_enc
    return big_f + head_f + enc_f <= wpart_floats(M, D)


def edges(M, D):
    """the facts the case table relies on"""
    ms_big, ms_enc = tc_msplit(M, D)
    rng = tc_split_ranges(M, ms_big)
    return dict(ms_big=ms_big, ms_enc=ms_enc, head_msplit=head_msplit(M), head_chunk=head_chunk(M), simt_msplit=simt_msplit(M),
                empty=[y for y, (b, e) in enumerate(rng) if b >= e], last_len=rng[-1][1] - rng[-1][0], enc_chained=enc_chained(M, D))


def test_case_table_edges():
    e = {(N, S): edges(N * S, 256) for (N, S) in list(CASES) + list(SIMT_CASES)}
    assert e[33, 31]["ms_big"] == 1 and e[64, 16]["ms_big"] == 8
    assert [edges(1024, D)["ms_big"] for D in DIMS] == [32, 16, 8]
    assert e[89, 23]["ms_enc"] == 1 and e[89, 23]["head_msplit"] == 1
    assert e[128, 16]["ms_enc"] == 32 and e[128, 16]["head_msplit"] == 1
    assert e[3, 683]["ms_enc"] == 32 and e[3, 683]["head_msplit"] == 2
    assert e[55, 20]["empty"] == [6, 7]
    assert 5117 % 64 and 5117 % 128
    assert not e[288, 128]["enc_chained"] and e[289, 128]["enc_chained"]
    assert e[1000, 37]["last_len"] % 32 == 8
    assert _ceil(8193 * 16, 2048) > 64 and e[8193, 16]["head_msplit"] == 64 and e[8193, 16]["head_chunk"] == 2064
    assert 2 * 512 * 512 <= 2 ** 19   # largest partial sum of the planted integers: exact in fp32
    assert e[256, 16]["simt_msplit"] == 1 and e[17, 241]["simt_msplit"] == 2
    # the encoding jobs are chained at D = 64 always, and at D = 128 only below the full split counts
    assert all(edges(N * S, 64)["enc_chained"] for (N, S) in CASES)
    assert [edges(N * S, 128)["enc_chained"] for (N, S) in CASES] == [N * S < 2048 for (N, S) in CASES]


@pytest.mark.parametrize("engine,D,N,S", PARAMS)
def test_workspace_mirror(engine, D, N, S):
    """the stash offsets used below are the library's: its workspace size at every case, and nnb_debug_layout at D = 256"""
    from nope_nerf_b200 import _lib as L
    lay = layout(N, S, D)
    eng = L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT
    want = lay["total"] + lay["tc_extra"] if engine == "tc" else lay["gates"]
    assert L.lib.nnb_workspace_bytes_dim(N, S, L.STASH, eng, D) == want
    if D == 256:
        out = (C.c_size_t * 14)()
        assert L.lib.nnb_debug_layout(C.c_int32(N), C.c_int32(S), C.c_uint32(L.STASH), C.c_int32(eng), out) == 0
        assert list(out)[:13] == [lay["rec"]] + lay["h"] + [lay["feat"], lay["hr"], lay["enc"], lay["denc"]]


# --------------------------------------------------------------------------------------------------------------------- planting
def _pattern(M, cols, tag, lo, hi):
    """[M, cols] integers in [lo, hi] from sample and column indices (a multiplicative hash), on the device, float32"""
    m = torch.arange(M, device="cuda", dtype=torch.int64)[:, None]
    c = torch.arange(cols, device="cuda", dtype=torch.int64)[None, :]
    h = (m + 1) * 7919 + (c + 1) * 104729 + tag * 1299709
    h = (((h ^ (h >> 7)) & 0xFFFFFF) * 2246822519) & 0xFFFFFFFF   # < 2^56 before the mask: no int64 overflow
    return ((h >> 13) % (hi - lo + 1) + lo).to(torch.float32)


def _region(ws, off, Mpad, cols):
    return ws[off:off + Mpad * cols * 4].view(torch.float32).view(Mpad, cols)


def plant(ws, lay, counting):
    """fill the stash regions the stage reads; returns {name: float64 [M, valid cols]} of what was planted"""
    M, Mpad, D = lay["M"], lay["Mpad"], lay["D"]
    ws.fill_(0xFF)   # NaN everywhere: the stage reads only the valid stash and the partials it stores itself
    regions = [("h%d" % l, lay["h"][l], D, D, "x") for l in range(8)] + \
              [("feat", lay["feat"], D, D, "x"), ("hr", lay["hr"], D // 2, D // 2, "x"), ("enc", lay["enc"], 64, 63, "x"),
               ("denc", lay["denc"], 32, 27, "x")] + \
              [("dy%d" % l, lay["dy"][l], D, D, "y") for l in range(8)] + \
              [("dfeat", lay["dfeat"], D, D, "y"), ("dyr", lay["dyr"], D // 2, D // 2, "y"), ("dyc", lay["dyc"], 4, 4, "y")]
    out = {}
    for tag, (name, off, cols, valid, kind) in enumerate(regions):
        if counting:
            v = torch.ones(M, valid, device="cuda")
        else:
            v = _pattern(M, valid, tag, -1, 1) if kind == "y" else _pattern(M, valid, tag, -2, 2)
        _region(ws, off, Mpad, cols)[:M, :valid] = v
        out[name] = v.double()
    return out


def expected(P, D):
    """every parameter gradient in float64 from the planted stash (the job list of the stage, by parameter)"""
    G = {}
    tr = [("layers0", 0), ("layers0", 2), ("layers0", 4), ("layers0", 6), ("layers1", 0), ("layers1", 2), ("layers1", 4), ("layers1", 6)]
    for l, (blk, i) in enumerate(tr):
        dy = P["dy%d" % l]
        X = P["enc"] if l == 0 else (torch.cat([P["h3"], P["enc"]], 1) if l == 4 else P["h%d" % (l - 1)])
        G["%s.%d.weight" % (blk, i)] = dy.T @ X; G["%s.%d.bias" % (blk, i)] = dy.sum(0)
    dsig = P["dyc"][:, 3:4]
    G["fc_density.weight"] = dsig.T @ P["h7"]; G["fc_density.bias"] = dsig.sum(0)
    G["fc_feature.weight"] = P["dfeat"].T @ P["h7"]; G["fc_feature.bias"] = P["dfeat"].sum(0)
    G["rgb_layers.0.weight"] = P["dyr"].T @ torch.cat([P["feat"], P["denc"]], 1); G["rgb_layers.0.bias"] = P["dyr"].sum(0)
    G["fc_rgb.weight"] = P["dyc"][:, :3].T @ P["hr"]; G["fc_rgb.bias"] = P["dyc"][:, :3].sum(0)
    return G


def run_stage(ws, engine, D, N, S, base):
    """g_weights = base, then nnb_debug_wgrad; returns the whole buffer (parameters + guard tail)"""
    from nope_nerf_b200 import _lib as L
    a = L.RenderArgs()
    a.N, a.S, a.flags, a.hidden_dim = N, S, L.STASH, D
    a.engine = L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    gw = base.clone()
    L.check(L.lib.nnb_debug_wgrad(C.byref(a), gw.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "nnb_debug_wgrad")
    torch.cuda.synchronize()
    return gw


def _describe(name, got, want, counting, M):
    bad = got != want
    idx = np.argwhere(bad)
    msg = "%s: %d of %d entries differ" % (name, idx.shape[0], got.size)
    if got.ndim == 2:
        msg += "; rows %s; columns %s" % (_span(np.unique(idx[:, 0]).tolist()), _span(np.unique(idx[:, 1]).tolist()))
    else:
        msg += "; entries %s" % _span(np.unique(idx[:, 0]).tolist())
    d = (got - want)[bad]
    if counting:
        msg += "; samples counted %s instead of %d" % (sorted(set((d + M).tolist()))[:8], M)
    else:
        msg += "; differences %s" % sorted(set(d.tolist()))[:8]
    return msg


def _span(v):
    return "%s (%d)" % (v[:6] + (["..", v[-1]] if len(v) > 6 else []), len(v))


@pytest.mark.gpu
@pytest.mark.parametrize("counting", (False, True), ids=("integers", "counting"))
@pytest.mark.parametrize("engine,D,N,S", PARAMS)
def test_wgrad_exact(engine, D, N, S, counting):
    from nope_nerf_b200 import _lib as L
    lay = layout(N, S, D)
    M = lay["M"]
    eng = L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT
    nb = L.lib.nnb_workspace_bytes_dim(N, S, L.STASH, eng, D)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    assert ws.data_ptr() % 256 == 0
    P = plant(ws, lay, counting)
    G = expected(P, D)
    npar = L.num_params(D)
    base = torch.full((npar + GUARD,), SENTINEL, device="cuda")
    base[:npar] = (torch.arange(npar, device="cuda") % 13 - 6).float()
    gw = run_stage(ws, engine, D, N, S, base)
    got = O.unflatten_params(gw[:npar].cpu().numpy(), D)
    b0 = O.unflatten_params(base[:npar].cpu().numpy(), D)
    errs = []
    for name, shape in O.param_shapes(D):
        want = (b0[name].astype(np.float64) + G[name].reshape(shape).cpu().numpy()).astype(np.float32)
        if not np.array_equal(got[name].view(np.int32), want.view(np.int32)):
            errs.append(_describe(name, got[name].astype(np.float64), want.astype(np.float64), counting, M))
    assert not errs, "%s D=%d M=%d (%s): %s" % (engine, D, M, CASES.get((N, S)) or SIMT_CASES[N, S], " | ".join(errs))
    tail = gw[npar:]
    assert torch.equal(tail, torch.full_like(tail, SENTINEL)), "guard tail after g_weights written"
    # the same case again: the same bits (fixed-order reductions)
    gw2 = run_stage(ws, engine, D, N, S, base)
    assert torch.equal(gw.view(torch.int32), gw2.view(torch.int32))
    del ws

"""ReLU gate bits of the tensor-core engine: tc_field_fwd writes one bit (h > 0) per activation of h0..h7 and of the rgb hidden layer
into the workspace, in the order of the wgmma accumulator fragment, and tc_dgrad gates the data-gradient chain with those bits instead of
re-reading the fp32 activation stash.
(1) host: the Python mirror of make_layout below matches the library's workspace sizes and offsets, and the fragment order covers
every (row, column) of a tile once; (2) GPU: the decoded bits equal h > 0 of the fp32 stash at every width, at C2 size and at a ragged
size, including pre-activations that are exactly +-0; (3) GPU: with every h / hr stash value overwritten by 1.0 between forward and
backward, the data gradients are the same bits as an untouched run, so tc_dgrad reads no fp32 activation."""
import ctypes as C
import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O

DIMS = (64, 128, 256)
SIZES = ((1024, 128), (301, 17))   # C2 (1024 rays x 128 samples); ragged: M = 5117 is not a multiple of 128


def _align(x, a):
    return (x + a - 1) // a * a


def layout(N, S, D):
    """byte offsets of make_layout (nnb_workspace.cuh) for the TC engine with NNB_STASH, and tc_workspace_extra"""
    from nope_nerf_b200 import _lib as L
    M = N * S
    Mpad = _align(M, 128)
    o = [0]

    def take(n):
        r = o[0]; o[0] = _align(o[0] + n, 256); return r
    npar = L.num_params(D)
    wpart = max(min(max((M + 4095) // 4096, 1), 16) * (npar + 8192), (2048 // D) * (npar + 8192), min(max((M + 2047) // 2048, 1), 64) * 8192)
    out = dict(M=M, Mpad=Mpad, n_tiles=Mpad // 128, D=D)
    out["rec"] = take(Mpad * 32)
    out["gs"], out["gp"], out["gv"] = take(Mpad * 16), take(Mpad * 16), take(Mpad * 16)
    out["rayred"] = take(N * 64); out["wpart"] = take(wpart * 4)
    out["h"] = [take(Mpad * D * 4) for _ in range(8)]
    out["feat"] = take(Mpad * D * 4); out["hr"] = take(Mpad * D // 2 * 4)
    out["enc"] = take(Mpad * 64 * 4); out["denc"] = take(Mpad * 32 * 4)
    out["dy"] = [take(Mpad * D * 4) for _ in range(8)]
    out["dfeat"] = take(Mpad * D * 4); out["dyr"] = take(Mpad * D // 2 * 4); out["dyc"] = take(Mpad * 16)
    out["gates"] = take(Mpad * D + Mpad * D // 16)
    out["total"] = o[0]
    ks = D // 16
    img = (8 + 9 * ks - ks) * D * 64 + ks * D * 32
    img_t = 34 * D * D + 576 * D
    out["tc_extra"] = _align(img, 256) + _align(img_t, 256)
    return out


def gate_offset(lay, layer):
    """byte offset of one layer's gate bits inside the gates region: [layer][tile][thread][bits]"""
    return layer * lay["Mpad"] * lay["D"] // 8


def fragment_map(cols):
    """tile row and column of bit b (0 .. cols/2 - 1) of consumer thread t (0 .. 255): the m64nNk16 accumulator fragment of the
    thread's warpgroup (warps 0-3: rows 0-63, warps 4-7: rows 64-127), bit 4j + 2r + e = row r0 + 8r, column 8j + c0 + e"""
    t = np.arange(256)[:, None]
    b = np.arange(cols // 2)[None, :]
    w, lane = t // 32, t % 32
    j, r, e = b // 4, (b // 2) % 2, b % 2
    return 64 * (w // 4) + 16 * (w % 4) + lane // 4 + 8 * r, 8 * j + 2 * (lane % 4) + e


def decode(region, n_tiles, cols):
    """one layer's gate bits (uint8 array) -> bool [n_tiles * 128, cols]: a thread's bit b is bit W - 1 - b % W of its little-endian
    W-bit word b / W (W = 32, or 16 when the thread holds only 16 bits)"""
    nb = cols // 2
    W = 32 if nb >= 32 else 16
    words = region.view(np.uint32 if W == 32 else np.uint16).reshape(n_tiles, 256, nb // W).astype(np.int64)
    b = np.arange(nb)
    bits = ((words[:, :, b // W] >> (W - 1 - b % W)) & 1).astype(bool)
    row, col = fragment_map(cols)
    out = np.zeros((n_tiles, 128, cols), bool)
    out[:, row, col] = bits
    return out.reshape(n_tiles * 128, cols)


# ---------------------------------------------------------------------------------------------------------------------------------- host

@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("N,S", SIZES)
def test_layout_mirror(N, S, D):
    """the mirror above matches the library: total size per width, and the stash offsets of nnb_debug_layout (D = 256)"""
    from nope_nerf_b200 import _lib as L
    lay = layout(N, S, D)
    assert L.lib.nnb_workspace_bytes_dim(N, S, L.STASH, L.ENGINE_TC, D) == lay["total"] + lay["tc_extra"]
    assert lay["gates"] + lay["Mpad"] * D * 17 // 16 == lay["total"]
    # the SIMT engine has no gate region
    assert L.lib.nnb_workspace_bytes_dim(N, S, L.STASH, L.ENGINE_SIMT, D) == lay["gates"]
    if D == 256:
        out = (C.c_size_t * 14)()
        assert L.lib.nnb_debug_layout(C.c_int32(N), C.c_int32(S), C.c_uint32(L.STASH), C.c_int32(L.ENGINE_TC), out) == 0
        assert list(out) == [lay["rec"]] + lay["h"] + [lay["feat"], lay["hr"], lay["enc"], lay["denc"], lay["total"]]


@pytest.mark.parametrize("cols", (256, 128, 64, 32))
def test_fragment_map_covers_tile(cols):
    row, col = fragment_map(cols)
    idx = np.sort((row * cols + col).ravel())
    assert np.array_equal(idx, np.arange(128 * cols))


# ----------------------------------------------------------------------------------------------------------------------------------- GPU

def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _render(P, D, N, S, seed, engine=None, flags=None):
    """TC (or `engine`) render forward with NNB_STASH on seeded inputs; returns the call (its workspace holds the stash).  flags:
    the rendering flags (default: those of the default config with the softplus occupancy activation)"""
    from nope_nerf_b200 import ops, _lib as L
    rng = np.random.default_rng(seed)
    H, W = 48, 64
    cfg = dict(O.DEFAULT_CFG); cfg["num_points"] = S
    r = _cuda(rng.normal(0, .05, (2, 3)).astype(np.float32)); t = _cuda(rng.normal(0, .05, (2, 3)).astype(np.float32))
    c2w = torch.empty(4, 4, device="cuda"); ops.pose_fwd_raw(r, t, None, 1, c2w)
    cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0])).cuda()
    ray_idx = rng.permutation(H * W)[:N]
    flags = ops.flags_from_cfg(cfg, "softplus") if flags is None else flags
    return ops.RenderCall(_cuda(O.flatten_params(P)), c2w, cam, N=N, S=S, flags=flags,
                          engine=L.ENGINE_TC if engine is None else engine,
                          near=0.01, far=10.0, ray_idx=_cuda(ray_idx), depth_map=_cuda(rng.uniform(.6, 7.2, (24, 32)).astype(np.float32)),
                          scale=torch.tensor([1.05]).cuda(), shift=torch.tensor([0.02]).cuda(),
                          noise=_cuda(rng.uniform(0, 1, (N, S)).astype(np.float32)), H=H, W=W, stash=True, hidden_dim=D)


def _layer(ws, lay, layer):
    """(fp32 stash [Mpad, cols], decoded gate bits [Mpad, cols]) of trunk layer 0..7 or the rgb hidden layer (8)"""
    Mpad, D = lay["Mpad"], lay["D"]
    off, cols = (lay["h"][layer], D) if layer < 8 else (lay["hr"], D // 2)
    h = ws[off:off + Mpad * cols * 4].cpu().numpy().view(np.float32).reshape(Mpad, cols)
    g0 = lay["gates"] + gate_offset(lay, layer)
    return h, decode(ws[g0:g0 + Mpad * cols // 8].cpu().numpy(), lay["n_tiles"], cols)


def _check_gates(ws, lay):
    M = lay["M"]
    for layer in range(9):
        h, bits = _layer(ws, lay, layer)
        open_ = h[:M] > 0
        assert 0 < open_.sum() < open_.size, (layer, "expected a mix of open and closed gates")
        bad = np.argwhere(bits[:M] != open_)
        assert bad.size == 0, (layer, bad[:5])


@pytest.mark.gpu
@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("N,S", SIZES)
def test_gate_bits_match_stash(N, S, D):
    call = _render(O.init_params(seed=5, D=D), D, N, S, seed=11)
    torch.cuda.synchronize()
    _check_gates(call.ws, layout(N, S, D))
    call.release()


@pytest.mark.gpu
@pytest.mark.parametrize("D", (64, 256))
def test_gate_bits_exact_zero(D):
    """pre-activations of exactly +0 (layer 2, rgb hidden layer) and of a -0 weight row and bias (layer 6) close the gate: the
    predicate is h > 0, as the fp32 stash gave it"""
    N, S = 301, 17
    P = O.init_params(seed=5, D=D)
    cz, cn, cr = 7, 11, 3
    P["layers0.4.weight"][cz] = 0.0; P["layers0.4.bias"][cz] = 0.0
    P["layers1.4.weight"][cn] = -0.0; P["layers1.4.bias"][cn] = -0.0
    P["rgb_layers.0.weight"][cr] = 0.0; P["rgb_layers.0.bias"][cr] = 0.0
    call = _render(P, D, N, S, seed=11)
    torch.cuda.synchronize()
    lay = layout(N, S, D)
    _check_gates(call.ws, lay)
    M = lay["M"]
    for layer, col in ((2, cz), (6, cn), (8, cr)):
        h, bits = _layer(call.ws, lay, layer)
        assert np.all(h[:M, col] == 0.0), layer
        assert not bits[:M, col].any(), layer
    call.release()


def _backward(D, N, S, clobber):
    """pose / depth-distortion gradients (no weight gradients) and tc_dgrad's d p, d viewdir; clobber: every h0..h7 / hr stash value
    set to 1.0 between forward and backward"""
    rng = np.random.default_rng(7)
    call = _render(O.init_params(seed=5, D=D), D, N, S, seed=11)
    lay = layout(N, S, D)
    ws = call.ws
    if clobber:
        Mpad = lay["Mpad"]
        for off, cols in [(o, D) for o in lay["h"]] + [(lay["hr"], D // 2)]:
            ws[off:off + Mpad * cols * 4].view(torch.float32).fill_(1.0)
    g_rgb = _cuda(rng.normal(0, 1, (N, 3)).astype(np.float32))
    g_dp = _cuda(rng.normal(0, 1, N).astype(np.float32)); g_dg = _cuda(rng.normal(0, 1, N).astype(np.float32))
    g_c2w = torch.zeros(4, 4, device="cuda"); g_cam = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
    call.backward(g_rgb, g_dp, g_dg, None, g_c2w, g_cam, None, g_ss)
    M = lay["M"]
    out = dict(c2w=g_c2w, cam=g_cam, ss=g_ss, gp=ws[lay["gp"]:lay["gp"] + M * 16].view(torch.float32),
               gv=ws[lay["gv"]:lay["gv"] + M * 16].view(torch.float32))
    out = {k: v.cpu() for k, v in out.items()}
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("D,N,S", [(64, 301, 17), (128, 301, 17), (256, 301, 17), (256, 1024, 128)])
def test_dgrad_reads_no_fp32_stash(D, N, S):
    ref = _backward(D, N, S, clobber=False)
    got = _backward(D, N, S, clobber=True)
    assert ref["gp"].abs().max() > 0 and ref["c2w"].abs().max() > 0
    for k in ref:
        assert torch.equal(ref[k], got[k]), k

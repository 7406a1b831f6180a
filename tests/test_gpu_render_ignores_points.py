"""GPU: nnb_render_fwd and nnb_render_bwd never read nnb_render_args.pts / dirs, which belong to the explicit-point field calls.  A render
whose args still carry the pointers of an earlier field query (here: a buffer of N * S NaN points, large enough for the render to read
in full) gives the same bits as one with NULL pointers, forward and backward, on both engines."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("engine", ["simt", "tc"])
def test_render_ignores_explicit_point_pointers(engine):
    from nope_nerf_b200 import _lib as L, ops
    eng = {"simt": L.ENGINE_SIMT, "tc": L.ENGINE_TC}[engine]
    N, S, D = 64, 32, 64
    dev = "cuda"
    w = torch.from_numpy(O.flatten_params(O.init_params(seed=5, D=D))).to(dev)
    c2w = torch.eye(4, device=dev); cam = torch.diag(torch.tensor([1.2, -1.5, -1.0, 1.0])).to(dev)
    g = torch.Generator().manual_seed(3)
    pix = (torch.rand(N, 2, generator=g) * 2 - 1).to(dev); dep = (torch.rand(N, generator=g) * 3 + 1).to(dev)
    g_rgb = torch.randn(N, 3, generator=g).to(dev)
    nan_pts = torch.full((N * S, 3), float("nan"), device=dev)

    def run(with_pts):
        outs = [torch.empty(N, 3, device=dev), torch.empty(N, device=dev), torch.empty(N, device=dev), torch.empty(N, dtype=torch.uint8, device=dev)]
        ws = torch.zeros(L.lib.nnb_workspace_bytes_dim(N, S, L.STASH, eng, D), dtype=torch.uint8, device=dev)
        a = L.RenderArgs()
        a.weights, a.c2w, a.cam, a.pixels, a.depth = L.ptr(w), L.ptr(c2w), L.ptr(cam), L.ptr(pix), L.ptr(dep)
        a.N, a.S, a.near_, a.far_, a.flags, a.engine, a.hidden_dim = N, S, 0.1, 5.0, L.STASH | L.SOFTPLUS, eng, D
        a.rgb, a.depth_pred, a.depth_gt, a.mask = (L.ptr(o) for o in outs)
        a.workspace, a.workspace_bytes = L.ptr(ws), ws.numel()
        if with_pts:
            a.pts = L.ptr(nan_pts); a.dirs = L.ptr(nan_pts)
        L.check(L.lib.nnb_render_fwd(C.byref(a), ops._stream()), "nnb_render_fwd")
        b = L.RenderBwdArgs()
        b.fwd = a
        g_w = torch.zeros(L.num_params(D), device=dev); g_c = torch.zeros(4, 4, device=dev)
        b.g_rgb, b.g_weights, b.g_c2w = L.ptr(g_rgb), L.ptr(g_w), L.ptr(g_c)
        L.check(L.lib.nnb_render_bwd(C.byref(b), ops._stream()), "nnb_render_bwd")
        torch.cuda.synchronize()
        return [o.cpu().numpy() for o in outs] + [g_w.cpu().numpy(), g_c.cpu().numpy()]

    ref, got = run(False), run(True)
    assert np.isfinite(ref[0]).all()
    for x, y in zip(ref, got):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))

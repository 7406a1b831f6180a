"""Bits of the one-wave weight-gradient stage of the tensor-core engine (tc_wgrad_all): the D-wide grid holds only the trunk and
fc_feature jobs, rgb_layers.0 runs as 64-column pieces (tc_wgrad_piece<64>) that stage X through a tensor map, and the head jobs run
on head_wgrad instead of simt_wgrad.  None of this may move a bit, so every weight and bias gradient is compared with SHA-256 digests
recorded from the build before the change:
- D = 128 at C2 size (1024 x 128): two column pieces of rgb_layers.0 per split instead of one 128-column CTA;
- a ragged D = 256 size, 1000 x 37 = 37 000 samples: the last of the 8 sample splits ends 8 samples into a 32-sample chunk, the last
  head split 8 samples into a 16-sample chunk, and the encoding jobs are chained;
- 60 x 25 = 1 500 samples at D = 256: fewer than one head split (2 048 samples), so each head job is a single split;
- the SIMT engine at C2 size and at a ragged 301 x 17, whose weight gradients share the partial buffer and wgrad_reduce.

The digests were generated with
    python tests/test_gpu_wgrad_one_wave.py
(NNB_LIB_PATH selects the library), which rewrites tests/golden/wgrad_one_wave_bits.npz."""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)   # run as a script
from oracle import nerf_oracle as O
from test_gpu_relu_mask import _cuda

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wgrad_one_wave_bits.npz")
CASES = {"tc_c2_d128": ("tc", 128, 1024, 128), "tc_ragged_d256": ("tc", 256, 1000, 37),
         "tc_below_head_split_d256": ("tc", 256, 60, 25), "simt_c2_d256": ("simt", 256, 1024, 128),
         "simt_ragged_d256": ("simt", 256, 301, 17)}


def all_grads(engine, D, N, S):
    """{parameter name: gradient} of one seeded render forward (NNB_STASH) + backward on the given engine"""
    from nope_nerf_b200 import ops, _lib as L
    rng = np.random.default_rng(11)
    H, W = 48, 64
    cfg = dict(O.DEFAULT_CFG); cfg["num_points"] = S
    r = _cuda(rng.normal(0, .05, (2, 3)).astype(np.float32)); t = _cuda(rng.normal(0, .05, (2, 3)).astype(np.float32))
    c2w = torch.empty(4, 4, device="cuda"); ops.pose_fwd_raw(r, t, None, 1, c2w)
    cam = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0])).cuda()
    ray_idx = rng.permutation(H * W)[:N] if N <= H * W else rng.integers(0, H * W, N)
    call = ops.RenderCall(_cuda(O.flatten_params(O.init_params(seed=5, D=D))), c2w, cam, N=N, S=S,
                          flags=ops.flags_from_cfg(cfg, "softplus"), engine=L.ENGINE_TC if engine == "tc" else L.ENGINE_SIMT,
                          near=0.01, far=10.0, ray_idx=_cuda(ray_idx), depth_map=_cuda(rng.uniform(.6, 7.2, (24, 32)).astype(np.float32)),
                          scale=torch.tensor([1.05]).cuda(), shift=torch.tensor([0.02]).cuda(),
                          noise=_cuda(rng.uniform(0, 1, (N, S)).astype(np.float32)), H=H, W=W, stash=True, hidden_dim=D)
    g = np.random.default_rng(7)
    g_rgb = _cuda(g.normal(0, 1, (N, 3)).astype(np.float32))
    g_dp = _cuda(g.normal(0, 1, N).astype(np.float32)); g_dg = _cuda(g.normal(0, 1, N).astype(np.float32))
    g_w = torch.zeros(L.num_params(D), device="cuda")
    g_c2w = torch.zeros(4, 4, device="cuda"); g_cam = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
    call.backward(g_rgb, g_dp, g_dg, g_w, g_c2w, g_cam, None, g_ss)
    torch.cuda.synchronize()
    return O.unflatten_params(g_w.cpu().numpy(), D)


def digests(grads):
    return np.array([hashlib.sha256(np.ascontiguousarray(grads[n], dtype=np.float32).tobytes()).hexdigest() for n in O.PARAM_NAMES])


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_weight_grad_bits(case):
    ref = np.load(GOLDEN)
    assert list(ref["params"]) == list(O.PARAM_NAMES)
    grads = all_grads(*CASES[case])
    for n in O.PARAM_NAMES:
        assert np.isfinite(grads[n]).all(), (case, n)
        assert np.abs(grads[n]).max() > 0, (case, n)
    bad = [n for n, a, b in zip(O.PARAM_NAMES, digests(grads), ref[case]) if a != b]
    assert not bad, (case, bad)


if __name__ == "__main__":
    out = {"params": np.array(list(O.PARAM_NAMES))}
    for case, args in CASES.items():
        out[case] = digests(all_grads(*args))
    np.savez(sys.argv[1] if len(sys.argv) > 1 else GOLDEN, **out)
    print("wrote %d cases" % len(CASES))

"""Bits of the overlapped weight-gradient stage of the tensor-core engine (tc_wgrad_all).  The encoding jobs (tc_wgrad<64>) and the
head jobs (simt_wgrad) run beside the second wave of the D-wide tc_wgrad grid, write their own regions of the partial buffer, and one
wgrad_reduce sums all of them.  Where the encoding region does not fit into the partial buffer (at D = 256, M <= 36 864 samples) the
encoding jobs run after that reduce, with their own.  Moving work in time must not move a bit, so the gradients are compared with
SHA-256 digests recorded from the build before the overlap:
- fc_density and fc_rgb (the head jobs; test_gpu_wgrad_pipeline.py pins every other parameter) in its five cases;
- every parameter at D = 256 on both sides of the fit predicate: 288 x 128 = 36 864 samples (encoding jobs after the reduce) and
  289 x 128 = 36 992 (encoding jobs chained).

The digests were generated with
    python tests/test_gpu_wgrad_overlap.py
(NNB_LIB_PATH selects the library), which rewrites tests/golden/wgrad_head_bits.npz."""
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
from test_gpu_relu_mask import _cuda, _render
from test_gpu_wgrad_pipeline import CASES as PIPELINE_CASES

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wgrad_head_bits.npz")
HEAD_PARAMS = [n for n in O.PARAM_NAMES if n.startswith(("fc_density.", "fc_rgb."))]
FIT_CASES = {"unchained_d256": (256, 288, 128), "chained_d256": (256, 289, 128)}


def all_grads(D, N, S):
    """{parameter name: gradient} of the seeded forward + backward of test_gpu_wgrad_pipeline.weight_grads"""
    from nope_nerf_b200 import _lib as L
    rng = np.random.default_rng(7)
    call = _render(O.init_params(seed=5, D=D), D, N, S, seed=11)
    g_rgb = _cuda(rng.normal(0, 1, (N, 3)).astype(np.float32))
    g_dp = _cuda(rng.normal(0, 1, N).astype(np.float32)); g_dg = _cuda(rng.normal(0, 1, N).astype(np.float32))
    g_w = torch.zeros(L.num_params(D), device="cuda")
    g_c2w = torch.zeros(4, 4, device="cuda"); g_cam = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
    call.backward(g_rgb, g_dp, g_dg, g_w, g_c2w, g_cam, None, g_ss)
    torch.cuda.synchronize()
    return O.unflatten_params(g_w.cpu().numpy(), D)


def digests(grads, names):
    return np.array([hashlib.sha256(np.ascontiguousarray(grads[n], dtype=np.float32).tobytes()).hexdigest() for n in names])


def _check(key, grads, names):
    ref = np.load(GOLDEN)
    for n in names:
        assert np.isfinite(grads[n]).all(), (key, n)
        assert np.abs(grads[n]).max() > 0, (key, n)
    bad = [n for n, a, b in zip(names, digests(grads, names), ref[key]) if a != b]
    assert not bad, (key, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(PIPELINE_CASES))
def test_head_bits(case):
    assert list(np.load(GOLDEN)["head_params"]) == HEAD_PARAMS
    _check("head_" + case, all_grads(*PIPELINE_CASES[case]), HEAD_PARAMS)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FIT_CASES))
def test_all_bits_at_fit_edge(case):
    assert list(np.load(GOLDEN)["params"]) == list(O.PARAM_NAMES)
    _check("all_" + case, all_grads(*FIT_CASES[case]), list(O.PARAM_NAMES))


if __name__ == "__main__":
    out = {"head_params": np.array(HEAD_PARAMS), "params": np.array(list(O.PARAM_NAMES))}
    for case, args in PIPELINE_CASES.items():
        out["head_" + case] = digests(all_grads(*args), HEAD_PARAMS)
    for case, args in FIT_CASES.items():
        out["all_" + case] = digests(all_grads(*args), list(O.PARAM_NAMES))
    np.savez(sys.argv[1] if len(sys.argv) > 1 else GOLDEN, **out)
    print("wrote %d head cases and %d fit-edge cases" % (len(PIPELINE_CASES), len(FIT_CASES)))

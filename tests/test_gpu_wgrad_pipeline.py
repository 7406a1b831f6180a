"""Bits of the tensor-core weight-gradient stage (tc_wgrad, then wgrad_reduce): the weight and bias gradients of seeded render backward
calls on the tensor-core engine are compared, parameter by parameter, with SHA-256 digests recorded from a known-good build.  The stage
keeps its sample splits and its MMA sequence per output element, so any change to its pipelining must leave these bits unchanged.

Cases: C2 size (1024 rays x 128 samples) at every width; a ragged 301 x 17 (M = 5117: the last sample split ends inside a 32-sample
chunk, and stash rows [M, Mpad) filled with NaN must not reach the gradients); 55 x 20 = 1100 samples at D = 256, where the 8 sample
splits of 192 samples leave splits 6 and 7 empty (they store zero partials).

The digests were generated with
    python tests/test_gpu_wgrad_pipeline.py
(NNB_LIB_PATH selects the library), which rewrites tests/golden/wgrad_tc_bits.npz."""
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
from test_gpu_relu_mask import _cuda, _render, layout

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wgrad_tc_bits.npz")
CASES = {"c2_d256": (256, 1024, 128), "c2_d128": (128, 1024, 128), "c2_d64": (64, 1024, 128),
         "ragged_d256": (256, 301, 17), "empty_splits_d256": (256, 55, 20)}
# parameters whose gradient comes from tc_wgrad (fc_density and fc_rgb are SIMT head jobs)
TC_PARAMS = [n for n in O.PARAM_NAMES if not n.startswith(("fc_density.", "fc_rgb."))]


def _stash_regions(lay):
    """(byte offset, floats per row) of every fp32 stash region the backward reads"""
    D = lay["D"]
    return ([(o, D) for o in lay["h"]] + [(lay["feat"], D), (lay["hr"], D // 2), (lay["enc"], 64), (lay["denc"], 32)]
            + [(o, D) for o in lay["dy"]] + [(lay["dfeat"], D), (lay["dyr"], D // 2)])


def weight_grads(D, N, S, nan_pad=False):
    """{parameter name: gradient} of one seeded forward + backward on the tensor-core engine; nan_pad: stash rows [M, Mpad) set to NaN
    between forward and backward"""
    from nope_nerf_b200 import _lib as L
    rng = np.random.default_rng(7)
    call = _render(O.init_params(seed=5, D=D), D, N, S, seed=11)
    lay = layout(N, S, D)
    if nan_pad:
        M, Mpad = lay["M"], lay["Mpad"]
        assert Mpad > M
        for off, cols in _stash_regions(lay):
            call.ws[off + M * cols * 4:off + Mpad * cols * 4].view(torch.float32).fill_(float("nan"))
    g_rgb = _cuda(rng.normal(0, 1, (N, 3)).astype(np.float32))
    g_dp = _cuda(rng.normal(0, 1, N).astype(np.float32)); g_dg = _cuda(rng.normal(0, 1, N).astype(np.float32))
    g_w = torch.zeros(L.num_params(D), device="cuda")
    g_c2w = torch.zeros(4, 4, device="cuda"); g_cam = torch.zeros(4, 4, device="cuda"); g_ss = torch.zeros(2, device="cuda")
    call.backward(g_rgb, g_dp, g_dg, g_w, g_c2w, g_cam, None, g_ss)
    torch.cuda.synchronize()
    P = O.unflatten_params(g_w.cpu().numpy(), D)
    return {n: P[n] for n in TC_PARAMS}


def digests(grads):
    return np.array([hashlib.sha256(np.ascontiguousarray(grads[n], dtype=np.float32).tobytes()).hexdigest() for n in TC_PARAMS])


def _check(case, grads):
    ref = np.load(GOLDEN)
    assert list(ref["params"]) == TC_PARAMS
    for n in TC_PARAMS:
        assert np.isfinite(grads[n]).all(), (case, n)
        assert np.abs(grads[n]).max() > 0, (case, n)
    bad = [n for n, a, b in zip(TC_PARAMS, digests(grads), ref[case]) if a != b]
    assert not bad, (case, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_wgrad_bits(case):
    _check(case, weight_grads(*CASES[case]))


@pytest.mark.gpu
def test_wgrad_ignores_padding_rows():
    """NaN in stash rows [M, Mpad) leaves every weight gradient finite and bit-identical"""
    _check("ragged_d256", weight_grads(*CASES["ragged_d256"], nan_pad=True))


if __name__ == "__main__":
    out ={"params": np.array(TC_PARAMS)}
    for case, args in CASES.items():
        out[case] = digests(weight_grads(*args))
    padded = digests(weight_grads(*CASES["ragged_d256"], nan_pad=True))
    print("ragged_d256 with NaN padding rows: %s" % ("same bits" if (padded == out["ragged_d256"]).all() else "DIFFERENT"))
    np.savez(sys.argv[1] if len(sys.argv) > 1 else GOLDEN, **out)
    print("wrote %d cases" % len(CASES))

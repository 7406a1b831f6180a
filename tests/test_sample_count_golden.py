"""CPU: pin the numpy oracle at rendering.num_points outside {32, 64, 128, 256} against fixtures written by the unmodified reference
(tools/make_golden.py samples): S = 48 and 96 (rays that straddle the tensor-core engine's 64-row blocks), 200 and 300 (more than 256
samples per ray, the compositing adjoint's former limit).  Same gates as tests/test_oracle_golden.py."""
import re
import numpy as np
import pytest
from _util import load_golden, relmax, check_param_digest
import test_oracle_golden as T

RENDER = ["render_tanks_noise_s48", "render_ndc_distalpha_s96", "render_eval_ones_s200", "render_tanks_noise_s300"]
RENDER_ALL = RENDER + [n + "_damped" for n in RENDER]


@pytest.mark.parametrize("name", RENDER_ALL)
def test_render(name):
    """outputs <= 2e-5 of the reference; gradients <= max(2e-4, 3 x |reference - fp64 oracle|)"""
    g = load_golden(name)
    S = int(re.search(r"_s(\d+)", name).group(1))
    assert int(g["S"]) == S and g["alpha"].shape == (int(g["N"]), S) and int(g["hidden_dim"]) == 256
    T.test_render(name)


def test_train_step_full_losses_s48():
    """two reference Trainer.train_step calls with the default loss set at 48 samples per ray vs oracle.train_step"""
    assert int(load_golden("train_full_losses_s48")["S"]) == 48
    T.test_train_step_full_losses("train_full_losses_s48")


def test_train_step_render_only_s300():
    """two render-only reference Trainer.train_step calls at 300 samples per ray vs oracle.train_step: losses, pose / distortion / MLP
    gradients of both steps, and the pose / distortion updates"""
    g = load_golden("train_render_only_s300")
    assert int(g["S"]) == 300 and g["noise_0"].shape == (int(g["N"]), 300)
    idx = int(g["idx"])
    st32, h32 = T._oracle_train(g, np.float32)
    _, h64 = T._oracle_train(g, np.float64)
    for it in range(int(g["steps"])):
        ld, gr = h32[it]; _, gr64 = h64[it]
        for k in ("loss", "loss_rgb", "loss_depth", "l2_mean"):
            ref = float(g["loss_%d.%s" % (it, k)])
            assert abs(float(ld[k]) - ref) / abs(ref) < 2e-5, (it, k, float(ld[k]), ref)
        for name, key in (("r", "grad_r_%d"), ("t", "grad_t_%d")):
            ref = g[key % it][idx]
            assert relmax(gr[name], ref) < max(2e-4, 3 * relmax(gr64[name], ref)), (it, name)
        ref_ss = np.array([g["grad_scales_%d" % it][idx, 0], g["grad_shifts_%d" % it][idx, 0]])
        env = relmax(np.array([gr64["scale"], gr64["shift"]]), ref_ss)
        assert relmax(np.array([gr["scale"], gr["shift"]]), ref_ss) < max(2e-4, 3 * env)
        env = check_param_digest(g, gr64["P"], prefix="pg_%d." % it)
        assert check_param_digest(g, gr["P"], prefix="pg_%d." % it) < max(5e-4, 3 * env), it
    for key in ("r", "t", "scales", "shifts"):
        assert relmax(st32[key] - g[key + "0"], g[key + "_end"] - g[key + "0"]) < 2e-3, key

"""CPU: a float64 torch restatement of the reference's normal_loss term (surface points, jittered neighbours, OfficialStaticNerf.gradient
with create_graph) reproduces the fixtures that the unmodified reference wrote in fp64 (tools/make_golden.py normals), values and
gradients with respect to the MLP, r, t, the camera matrix's kx / ky, scale and shift; and the reference's own fp32 run lies within the
gate the GPU test applies."""
import numpy as np
import pytest

from _util import load_golden
import _normals_ref as NR


@pytest.mark.parametrize("name", NR.NAMES)
def test_restatement_reproduces_reference_fp64(name):
    g = load_golden(name)
    assert g["diff_norm.f64"].shape[0] == int(g["N"]) and g["nbr"].shape == (int(g["N"]), 3)
    out = NR.diff_norm64(g)
    for key in [k[:-4] for k in g if k.endswith(".f64")]:
        got = NR.sel(g, key, out[key])
        ref = g[key + ".f64"]
        err = np.abs(np.asarray(got, np.float64).reshape(ref.shape) - ref).max()
        assert err <= 1e-6 * max(np.abs(ref).max(), 1e-30), (key, err)


@pytest.mark.parametrize("name", NR.NAMES)
def test_fixture_has_gradients_through_every_input(name):
    """the weighting reaches the pose, the camera matrix, the distortion and the trunk; biases and the rgb branch get exactly zero"""
    g = load_golden(name)
    for key in ("grad_r", "grad_t", "grad_kxy", "grad_scale", "grad_shift", "pg.layers0.0.weight", "pg.layers1.6.weight",
                "pg.fc_density.weight"):
        assert np.abs(g[key + ".f64"]).max() > 0, key
    for key in ("pg.layers0.0.bias", "pg.fc_density.bias", "pg.fc_feature.weight", "pg.rgb_layers.0.weight", "pg.fc_rgb.bias"):
        assert np.abs(g[key + ".f64"]).max() == 0 and np.abs(g[key + ".f32"]).max() == 0, key

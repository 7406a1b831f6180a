"""The reference logic the fused ray march is checked against, pinned without a device: Renderer._ray_marching_torch (the torch march,
run here on the CPU over an analytic occupancy) against the numpy restatement of tests/_ray_march_ref.py, bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import _ray_march_ref as R
from _cfg import default_cfg


class Blob(nn.Module):
    """occupancy of a ball of radius 0.5 around c with a soft edge, plus a ripple so that rays see several crossings"""

    def __init__(self, c):
        super().__init__()
        self.c = torch.tensor(c, dtype=torch.float32)

    def forward(self, p, ray_d=None, only_occupancy=False, **kw):
        r = (p - self.c).norm(2, -1)
        return torch.sigmoid(20 * (0.5 - r) + 3 * torch.sin(25 * r)).unsqueeze(-1)


def _renderer(model):
    import nope_nerf_b200.model as mdl
    return mdl.Renderer(model, default_cfg()["rendering"], device=torch.device("cpu"))


@pytest.mark.parametrize("n_steps", [2, 64, 129, 512])
@pytest.mark.parametrize("n_secant", [0, 1, 8])
def test_numpy_march_equals_torch_march(n_steps, n_secant):
    g = torch.Generator().manual_seed(5 + n_steps)
    N = 600
    model = Blob([0.1, -0.05, 0.2])
    rend = _renderer(model)
    # one origin outside the ball (most rays enter it), one inside (first sample occupied)
    for origin in ([0.0, 0.0, -1.5], [0.1, -0.05, 0.25]):
        ray0 = torch.tensor(origin).repeat(1, N, 1)
        d = torch.randn(1, N, 3, generator=g) * 0.35 + torch.tensor([0.0, 0.0, 1.0])
        d = d / d.norm(2, -1, keepdim=True)
        ref = rend._ray_marching_torch(ray0, d, model, n_steps, n_secant, [0.0, 2.4], 3500000, 2.0, None)[0].numpy()
        far = rend._sphere_far(ray0[:, 0], d, 2.0)[0].numpy()
        frac = torch.linspace(0, 1, n_steps).numpy()
        t = R.depths(0.0, far, frac)
        o, dn = ray0[0].numpy(), d[0].numpy()
        occ = lambda p: model(torch.from_numpy(p))[..., 0].numpy()
        val = occ(o[:, None, :] + dn[:, None, :] * t[:, :, None]) - np.float32(0.5)
        first, hit, v0neg, br = R.first_and_bracket(val, t)
        d_hit = R.secant(br[hit], n_secant, lambda dd: occ(o[hit] + dd[:, None] * dn[hit]) - np.float32(0.5))
        out = R.depth_out(hit, v0neg, d_hit)
        assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))
        if origin[2] < -1 and n_steps > 2:
            assert hit.any() and (~hit).any()
        if origin[2] > 0:
            assert (~v0neg).all() and (out == 0).all()


def test_planted_values():
    """first sign change, products that underflow, pos -> neg first, last pair, occupied first sample"""
    tiny = np.float32(1e-30)
    val = np.array([[-1, -1, 1, -1, 1],        # first = 1, hit
                    [-1, 1, 1, 1, 1],          # first pair
                    [-1, -1, -1, -1, 1],       # last pair
                    [-1, -1, -1, -1, -1],      # no crossing
                    [1, -1, 1, 1, 1],          # first sample occupied, crossings later
                    [-tiny, tiny, 1, -1, 1],   # the product of the first pair underflows to -0: no sign change; the first one is pos -> neg
                    [-1, 0, 1, 1, 1]],         # through an exact zero: no negative product
                   np.float32)
    t = np.tile(np.linspace(0, 1, 5, dtype=np.float32), (7, 1))
    first, hit, v0neg, br = R.first_and_bracket(val, t)
    assert first.tolist() == [1, 0, 3, -1, 0, 2, -1]
    assert hit.tolist() == [True, True, True, False, False, False, False]
    assert v0neg.tolist() == [True, True, True, True, False, True, True]
    assert br[0].tolist() == [0.25, 0.5, -1, 1] and br[2].tolist() == [0.75, 1.0, -1, 1]
    out = R.depth_out(hit, v0neg, R.secant(br[hit], 0, None))
    assert out[0] == np.float32(0.375) and np.isinf(out[3]) and out[4] == 0 and np.isinf(out[5]) and np.isinf(out[6])

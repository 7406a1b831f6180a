"""OfficialStaticNerf — parameter container + field evaluation (reference:
model/official_nerf.py:8-119).  Same nn.Linear submodules / state_dict keys as the
reference so checkpoints and train.py's reset_parameters() loop work unchanged; the
arithmetic runs in the CUDA library on a FLAT fp32 view of all 24 tensors."""
import math
import torch
import torch.nn as nn
from .. import _lib as L

_PIN, _DIN = 63, 27


def param_shapes(D=256):
    """(state_dict key, shape) of every parameter of a width-D field, in parameters() order (official_nerf.py:20-37)"""
    shapes = []
    for blk, ins in (("layers0", [_PIN, D, D, D]), ("layers1", [D + _PIN, D, D, D])):
        for j, i in enumerate((0, 2, 4, 6)):
            shapes += [("%s.%d.weight" % (blk, i), (D, ins[j])), ("%s.%d.bias" % (blk, i), (D,))]
    shapes += [("fc_density.weight", (1, D)), ("fc_density.bias", (1,)), ("fc_feature.weight", (D, D)),
               ("fc_feature.bias", (D,)), ("rgb_layers.0.weight", (D // 2, D + _DIN)), ("rgb_layers.0.bias", (D // 2,)),
               ("fc_rgb.weight", (3, D // 2)), ("fc_rgb.bias", (3,))]
    return shapes


def param_slices(D=256):
    """(offset, numel, shape) of every parameter in the flat vector of a width-D field (flat order == parameters() order)"""
    out, o = [], 0
    for _, s in param_shapes(D):
        k = int(math.prod(s)); out.append((o, k, s)); o += k
    assert o == L.num_params(D)
    return out


PARAM_NAMES = [n for n, _ in param_shapes()]
PARAM_SLICES = param_slices(256)  # the default width; a module's own layout is OfficialStaticNerf.param_slices
assert PARAM_SLICES[-1][0] + 3 == L.NUM_PARAMS


class OfficialStaticNerf(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        D = cfg['model']['hidden_dim']
        if D not in L.HIDDEN_DIMS:
            raise NotImplementedError("the CUDA field supports model.hidden_dim in {%s} (got %r)" % (", ".join(map(str, L.HIDDEN_DIMS)), D))
        if cfg['model']['pos_enc_levels'] != 10 or cfg['model']['dir_enc_levels'] != 4:
            raise NotImplementedError("the CUDA field is specialised for pos/dir encoding levels 10/4 "
                                      "(the reference hard-codes the levels, official_nerf.py:61,87)")
        self.hidden_dim = D
        self.num_params = L.num_params(D)
        self.param_slices = param_slices(D)
        pos_in, dir_in = 63, 27
        self.white_bkgd = cfg['rendering']['white_background']
        self.dist_alpha = cfg['rendering']['dist_alpha']
        self.occ_activation = cfg['model']['occ_activation']
        self.layers0 = nn.Sequential(nn.Linear(pos_in, D), nn.ReLU(), nn.Linear(D, D), nn.ReLU(),
                                     nn.Linear(D, D), nn.ReLU(), nn.Linear(D, D), nn.ReLU())
        self.layers1 = nn.Sequential(nn.Linear(D + pos_in, D), nn.ReLU(), nn.Linear(D, D), nn.ReLU(),
                                     nn.Linear(D, D), nn.ReLU(), nn.Linear(D, D), nn.ReLU())
        self.fc_density = nn.Linear(D, 1)
        self.fc_feature = nn.Linear(D, D)
        self.rgb_layers = nn.Sequential(nn.Linear(D + dir_in, D // 2), nn.ReLU())
        self.fc_rgb = nn.Linear(D // 2, 3)
        self.fc_density.bias.data = torch.tensor([0.1]).float()          # official_nerf.py:39
        self.sigmoid = nn.Sigmoid()
        self.fc_rgb.bias.data = torch.tensor([0.8 if self.white_bkgd else 0.02] * 3).float()   # :41-44
        self._flat = None
        self._flat_grad = None

    # ---- flat parameter view -------------------------------------------------------------
    def _plist(self):
        ps = list(self.parameters())
        assert len(ps) == len(self.param_slices)
        return ps

    def flat_weights(self):
        """Flat fp32 tensor aliasing all parameters (re-packed if a .to()/load broke the aliasing)."""
        ps = self._plist()
        f = self._flat
        ok = f is not None and f.device == ps[0].device
        if ok:
            base = f.data_ptr()
            for p, (o, n, s) in zip(ps, self.param_slices):
                if p.data_ptr() != base + 4 * o:
                    ok = False; break
        if not ok:
            f = torch.empty(self.num_params, dtype=torch.float32, device=ps[0].device)
            with torch.no_grad():
                for p, (o, n, s) in zip(ps, self.param_slices):
                    f[o:o + n].copy_(p.detach().reshape(-1).float())
                    p.data = f[o:o + n].view(s)
            self._flat = f
        return f

    def flat_grad(self, zero=True, alias=None):
        """Flat gradient buffer whose slices are installed as every parameter's .grad.
        `alias` lets a caller (data-parallel trainer) provide the storage."""
        ps = self._plist()
        g = alias if alias is not None else self._flat_grad
        if g is None or g.device != ps[0].device:
            g = torch.zeros(self.num_params, dtype=torch.float32, device=ps[0].device)
            zero = False
        self._flat_grad = g
        if zero:
            g.zero_()
        for p, (o, n, s) in zip(ps, self.param_slices):
            if p.requires_grad:
                p.grad = g[o:o + n].view(s)
        return g

    # ---- reference API -------------------------------------------------------------------
    def infer_occ(self, p, engine=None, grad_engine=None):
        """official_nerf.py:60-67: (trunk features, density logit).  The trunk features never leave the kernel here; callers in the
        reference (gradient(), forward()) only use the logit, so the first element is None.  engine, grad_engine: see forward(); with
        engine='tc', grad_engine='tc' a logit under autograd differentiates the occupancy alone on tensor cores."""
        from ..field import field_query_grad
        _, s = field_query_grad(self, p, None, raw_density=True, occ_only=True, engine=engine, grad_engine=grad_engine)
        return None, s

    def gradient(self, p, it, engine=None):
        """official_nerf.py:46-58: -d(density logit)/d p, shape (N, 1, 3) (surface normals of the geometry view).  The reference
        differentiates infer_occ with autograd (create_graph=True); here it is the data-gradient chain of the field kernel with cotangent
        1 on the logit.  With grad mode on and p requiring grad the result has a grad_fn: its backward is the second-order field kernel
        (nnb_field_hvp) and reaches p and the MLP parameters, so normal regularisers train the field.  The reference sets requires_grad
        on the caller's p itself; here the caller does (p.requires_grad_(True) for a regulariser on fixed points), and otherwise the
        normals come back detached, as plain values that callers may read directly (.numpy()).  Renderer.nope_nerf's normal term sets
        requires_grad on its own surface points, as the reference does, so it reaches the MLP with a fixed pose, camera and depth too.
        engine: None = the exact-fp32 engine; 'tc' = the tensor-core data gradient (nnb_field_vjp) for detached normals.  A call that
        returns a grad_fn (grad mode on and p requiring grad) runs on the exact engine whatever engine it names (field.field_normal).
        gradient_grad(p, it, engine='tc', grad_engine='tc') keeps such a call on tensor cores."""
        return self.gradient_grad(p, it, engine)

    def gradient_grad(self, p, it, engine=None, grad_engine=None):
        """gradient() with the engine of a call that returns a grad_fn.  grad_engine: None or 'simt' = the exact engine (gradient()'s
        rule); 'tc' (with engine='tc' only, ValueError otherwise, whether or not the call needs the graph) = the normals keep the bits of
        the detached tensor-core normals and their backward is the tensor-core second-order backward nnb_field_hvp_tc
        (field.field_normal)."""
        from ..field import field_normal
        q = p.reshape(-1, 3)
        if torch.is_grad_enabled() and p.requires_grad:
            n = field_normal(self, q) if grad_engine is None else field_normal(self, q, engine=engine, grad_engine=grad_engine)
        else:
            with torch.no_grad():
                n = field_normal(self, q, engine=engine, grad_engine=grad_engine)
        return -n.reshape(p.shape).unsqueeze(1)

    def forward(self, p, ray_d=None, only_occupancy=False, return_logits=False, return_addocc=False,
                noise=False, it=100000, engine=None, grad_engine=None, **kwargs):
        """Field query on explicit points (official_nerf.py:69-96); `noise`, `it`, `return_logits`
        are accepted and ignored exactly like the reference.
        engine: None = the exact-fp32 engine; 'tc' = the tensor-core engine for a call that needs no gradient (a call that does runs
        on the exact engine), skipping the colour branch when only_occupancy (field.field_query_grad).
        grad_engine: None = a call that needs a gradient runs on the exact engine; 'tc' (with engine='tc' only, ValueError otherwise) =
        it runs on tensor cores too, with the tensor-core backward nnb_field_grad (gradients to p, ray_d and every parameter)."""
        from ..field import field_query_grad
        rgb, a = field_query_grad(self, p, ray_d, occ_only=only_occupancy, engine=engine, grad_engine=grad_engine)
        if only_occupancy:
            return a
        if ray_d is not None:
            return (rgb, a) if return_addocc else rgb
        return None

"""float64 torch restatement of the reference's normal_loss term (model/rendering.py:53-94,133-141 with OfficialStaticNerf.gradient,
official_nerf.py:46-67) for the fixtures tools/make_golden.py normals writes (test infrastructure)."""
import numpy as np
import torch

from oracle import nerf_oracle as O

TRUNK = [("layers0", 0), ("layers0", 2), ("layers0", 4), ("layers0", 6), ("layers1", 0), ("layers1", 2), ("layers1", 4), ("layers1", 6)]


def exp_so3(r):
    K = torch.zeros(3, 3, dtype=r.dtype)
    K[0, 1], K[0, 2], K[1, 0], K[1, 2], K[2, 0], K[2, 1] = -r[2], r[1], r[2], -r[0], -r[1], r[0]
    th = r.norm() + 1e-15
    return torch.eye(3, dtype=r.dtype) + (torch.sin(th) / th) * K + ((1 - torch.cos(th)) / th ** 2) * (K @ K)


def logit(W, p):
    e = [p]
    for i in range(10):
        e += [torch.sin(2.0 ** i * p), torch.cos(2.0 ** i * p)]
    e = torch.cat(e, -1)
    x = e
    for l, (blk, i) in enumerate(TRUNK):
        if l == 4:
            x = torch.cat([x, e], -1)
        x = torch.relu(x @ W["%s.%d.weight" % (blk, i)].T + W["%s.%d.bias" % (blk, i)])
    return x @ W["fc_density.weight"].T + W["fc_density.bias"]


def inputs(g):
    """(pixels [N,2], raw prior depth [N]) of a fixture"""
    H, W = int(g["H"]), int(g["W"])
    raw, _ = O.gather_prior_depth(g["dpt"], g["ray_idx"], H, W)
    return g["pixels"].astype(np.float64), raw.astype(np.float64)


def diff_norm64(g, normalise=True):
    """float64 diff_norm and its gradients for the fixture's weighting: dict like the fixture's .f64 entries (param gradients full)"""
    D = int(g["hidden_dim"])
    P = O.init_params(seed=int(g["seed"]), D=D, hf_damp=True)
    W = {k: torch.from_numpy(np.asarray(v, np.float64)).requires_grad_(True) for k, v in P.items()}
    cam = int(g["cam_id"])
    r = torch.from_numpy(g["r"][cam].astype(np.float64)).requires_grad_(True)
    t = torch.from_numpy(g["t"][cam].astype(np.float64)).requires_grad_(True)
    kxy = torch.tensor([float(g["kx"]), float(g["ky"])], dtype=torch.float64, requires_grad=True)
    scale = torch.tensor(float(g["scale"]), dtype=torch.float64, requires_grad=True)
    shift = torch.tensor(float(g["shift"]), dtype=torch.float64, requires_grad=True)
    pix, raw = inputs(g)
    pix = torch.from_numpy(pix); depth = torch.from_numpy(raw) * scale + shift
    R = exp_so3(r)
    dc = torch.stack([pix[:, 0] / kxy[0], pix[:, 1] / kxy[1], -torch.ones(pix.shape[0], dtype=torch.float64)], -1)
    dt = dc @ R.T
    d_i = (depth.unsqueeze(-1) * dt).norm(dim=-1)
    m = torch.isfinite(d_i) & (d_i != 0)
    nrm = dt.norm(dim=-1)
    pts = (t + dt / nrm.unsqueeze(-1) * d_i.unsqueeze(-1)) if normalise else (t + dt * (d_i / nrm).unsqueeze(-1))
    pts = pts[m]
    N = pts.shape[0]
    pp = torch.cat([pts, pts + (torch.from_numpy(g["nbr"].astype(np.float64)) - 0.5) * 0.01])
    s = logit(W, pp)
    n, = torch.autograd.grad(s.sum(), pp, create_graph=True)
    gr = -n
    nn_ = gr / (gr.norm(dim=1, keepdim=True) + 1e-5)
    dn = (nn_[:N] - nn_[N:]).norm(dim=-1)
    (dn * torch.from_numpy(g["wts"].astype(np.float64))).sum().backward()
    out = {"diff_norm": dn.detach().numpy(), "grad_r": r.grad.numpy(), "grad_t": t.grad.numpy(), "grad_kxy": kxy.grad.numpy(),
           "grad_scale": scale.grad.numpy(), "grad_shift": shift.grad.numpy()}
    for k, v in W.items():
        out["pg." + k] = (np.zeros(v.numel()) if v.grad is None else v.grad.numpy().reshape(-1))
    return out


def sel(g, key, full):
    """the fixture's entries of a full parameter gradient"""
    return full[g[key + ".idx"]] if key + ".idx" in g else full


def gate(g, key, got):
    """max |got - fp64| and the project's rule max(1e-4 max|fp64|, 3 max|fp32 - fp64|) for one stored quantity"""
    a32, a64 = g[key + ".f32"].astype(np.float64), g[key + ".f64"]
    got = np.asarray(got, np.float64).reshape(a64.shape)
    return float(np.abs(got - a64).max()), max(1e-4 * float(np.abs(a64).max()), 3 * float(np.abs(a32 - a64).max()))


NAMES = ["normals_uniform_d64", "normals_ndc_d64", "normals_uniform_d256", "normals_ndc_d256"]

#!/usr/bin/env python
"""Eager-PyTorch statement of the same C2 training step (autograd, torch.optim.Adam x3), timed on the device it is run on.

Where no reference checkout is available, this is the stand-in for "the reference's single-GPU PyTorch path" that
BASELINE.md section 3 asks to time next to the product: the SAME op structure as the reference's step (SURVEY.md 8a: whole-map
nearest interpolation + gather, randperm(H*W), pixel grid rebuilt per step, exp-map pose, per-level sin/cos + cat encoding,
nn.Linear MLP, cumprod compositing, L1 losses, loss.backward(), three Adam optimizers), written from the equations of
oracle/nerf_oracle.py.  A measurement tool only: nothing in the product imports it.

    python tools/torch_step_baseline.py [--device cuda|cpu] [--steps 10] [--check]
--check: one small step against oracle.train_step on the CPU (same inputs), prints the relative differences."""
import argparse, json, os, sys, time
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class Field(nn.Module):   # official_nerf.py:20-96 layer list
    def __init__(self, D=256):
        super().__init__()
        self.layers0 = nn.Sequential(nn.Linear(63, D), nn.ReLU(), nn.Linear(D, D), nn.ReLU(), nn.Linear(D, D), nn.ReLU(), nn.Linear(D, D), nn.ReLU())
        self.layers1 = nn.Sequential(nn.Linear(D + 63, D), nn.ReLU(), nn.Linear(D, D), nn.ReLU(), nn.Linear(D, D), nn.ReLU(), nn.Linear(D, D), nn.ReLU())
        self.fc_density = nn.Linear(D, 1); self.fc_feature = nn.Linear(D, D)
        self.rgb_layers = nn.Sequential(nn.Linear(D + 27, D // 2), nn.ReLU()); self.fc_rgb = nn.Linear(D // 2, 3)

    @staticmethod
    def encode(x, L):
        out = [x]
        for l in range(L):
            out += [torch.sin(2.0 ** l * x), torch.cos(2.0 ** l * x)]
        return torch.cat(out, -1)

    def forward(self, p, d):
        e = self.encode(p, 10)
        h = self.layers0(e)
        h = self.layers1(torch.cat([h, e], -1))
        sigma = F.softplus(self.fc_density(h))
        alpha = 1.0 - torch.exp(-sigma)
        feat = self.fc_feature(h)
        hr = self.rgb_layers(torch.cat([feat, self.encode(d, 4)], -1))
        return torch.sigmoid(self.fc_rgb(hr)), alpha


def exp_so3(r):   # common.py:277-330
    n = r.norm() + 1e-15
    K = torch.zeros(3, 3, device=r.device, dtype=r.dtype)
    K[0, 1], K[0, 2], K[1, 0], K[1, 2], K[2, 0], K[2, 1] = -r[2], r[1], r[2], -r[0], -r[1], r[0]
    return torch.eye(3, device=r.device, dtype=r.dtype) + (torch.sin(n) / n) * K + ((1 - torch.cos(n)) / n ** 2) * (K @ K)


def c2w_of(r, t, cam_id):
    R = exp_so3(r[cam_id])
    return torch.cat([torch.cat([R, t[cam_id][:, None]], 1), torch.tensor([[0., 0, 0, 1]], device=r.device)], 0)


def render_eval(net, c2w, H, W, kx, ky, S, near, far, chunk=8192):
    """all pixels of one view, no jitter, eval-mode outputs (rgb (H,W,3), distance along the normalised ray / |d~| = depth)"""
    dev = c2w.device
    ys, xs = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    pix = torch.stack([2.0 * xs.reshape(-1) / (W - 1) - 1.0, 2.0 * ys.reshape(-1) / (H - 1) - 1.0], -1)
    out_rgb, out_d = [], []
    with torch.no_grad():
        for i in range(0, H * W, chunk):
            p = pix[i:i + chunk]; n = p.shape[0]
            dcam = torch.stack([p[:, 0] / kx, p[:, 1] / ky, -torch.ones(n, device=dev)], -1)
            dt = dcam @ c2w[:3, :3].t(); nrm = dt.norm(dim=-1, keepdim=True); d = dt / nrm
            u = torch.linspace(0, 1, S, device=dev); z = (near * (1 - u) + far * u).expand(n, S)
            pts = (c2w[:3, 3].expand(n, 3)[:, None] + d[:, None] * z[..., None]).reshape(-1, 3)
            rgb_s, alpha = net(pts, (-d)[:, None].expand(n, S, 3).reshape(-1, 3))
            alpha = alpha.reshape(n, S)
            w = alpha * torch.cumprod(torch.cat([torch.ones(n, 1, device=dev), 1 - alpha + 1e-6], -1), -1)[:, :-1]
            out_rgb.append((w[..., None] * rgb_s.reshape(n, S, 3)).sum(1)); out_d.append((w * z).sum(1) / nrm[:, 0])
    return torch.cat(out_rgb).reshape(H, W, 3), torch.cat(out_d).reshape(H, W)


def step(net, r, t, scales, shifts, opts, img, dpt, cam_id, kx, ky, N, S, near, far, ray_idx=None, noise=None):
    H, W = img.shape[-2:]; dev = img.device
    for o in opts: o.zero_grad()
    R = exp_so3(r[cam_id]); c2w = torch.cat([torch.cat([R, t[cam_id][:, None]], 1), torch.tensor([[0., 0, 0, 1]], device=dev)], 0)
    if ray_idx is None: ray_idx = torch.randperm(H * W, device=dev)[:N]
    ys, xs = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")        # common.py:22-45
    grid = torch.stack([2.0 * xs.reshape(-1) / (W - 1) - 1.0, 2.0 * ys.reshape(-1) / (H - 1) - 1.0], -1)
    pix = grid[ray_idx]
    rgb_gt = img.reshape(3, -1)[:, ray_idx].t()
    depth_full = F.interpolate(dpt[None, None], (H, W), mode="nearest").reshape(-1)                           # network.py:19-33
    depth = depth_full[ray_idx] * scales[cam_id, 0] + shifts[cam_id, 0]
    dcam = torch.stack([pix[:, 0] / kx, pix[:, 1] / ky, -torch.ones(N, device=dev)], -1)                    # rendering.py:57-69
    dt = dcam @ c2w[:3, :3].t()
    nrm = dt.norm(dim=-1, keepdim=True); d = dt / nrm
    o = c2w[:3, 3].expand(N, 3)
    depth_gt = depth * nrm[:, 0]
    u = torch.linspace(0, 1, S, device=dev); z = (near * (1 - u) + far * u).expand(N, S)
    mids = 0.5 * (z[:, 1:] + z[:, :-1]); hi = torch.cat([mids, z[:, -1:]], -1); lo = torch.cat([z[:, :1], mids], -1)
    if noise is None: noise = torch.rand(N, S, device=dev)
    z = lo + (hi - lo) * noise
    pts = (o[:, None] + d[:, None] * z[..., None]).reshape(-1, 3)
    dirs = (-d)[:, None].expand(N, S, 3).reshape(-1, 3)
    rgb_s, alpha = net(pts, dirs)
    alpha = alpha.reshape(N, S)
    w = alpha * torch.cumprod(torch.cat([torch.ones(N, 1, device=dev), 1 - alpha + 1e-6], -1), -1)[:, :-1]
    rgb = (w[..., None] * rgb_s.reshape(N, S, 3)).sum(1); dist = (w * z).sum(1)
    loss_rgb = (rgb - rgb_gt).abs().sum() / N; loss_depth = (dist - depth_gt).abs().mean()
    loss = loss_rgb + 0.04 * loss_depth
    loss.backward()
    for o_ in opts: o_.step()
    return loss.detach(), loss_rgb.detach(), loss_depth.detach()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", default="cuda" if torch.cuda.is_available() else "cpu")
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    if a.check:
        from oracle import nerf_oracle as O
        torch.manual_seed(0); rng = np.random.default_rng(0)
        H, W, hd, wd, V, N, S = 48, 64, 24, 32, 4, 64, 32
        P = O.init_params(seed=42)
        net = Field()
        with torch.no_grad():
            for k, v in net.state_dict().items(): v.copy_(torch.from_numpy(P[k]))
        img = rng.uniform(0, 1, (3, H, W)).astype(np.float32); dpt = rng.uniform(0.6, 7.2, (hd, wd)).astype(np.float32)
        r0 = (0.05 * rng.standard_normal((V, 3))).astype(np.float32); t0 = (0.05 * rng.standard_normal((V, 3))).astype(np.float32)
        ray_idx = rng.permutation(H * W)[:N]; noise = rng.uniform(0, 1, (N, S)).astype(np.float32)
        kx, ky = 1.2, -1.2 * W / H
        cfg = dict(O.DEFAULT_CFG); cfg["num_points"] = S
        state = dict(P=P, r=r0.copy(), t=t0.copy(), scales=np.ones((V, 1), np.float32), shifts=np.zeros((V, 1), np.float32))
        ld, grads, _ = O.train_step(state, img, dpt, ray_idx, noise, 1, kx, ky, cfg, apply_update=False)
        r = nn.Parameter(torch.from_numpy(r0)); t = nn.Parameter(torch.from_numpy(t0))
        sc = nn.Parameter(torch.ones(V, 1)); sh = nn.Parameter(torch.zeros(V, 1))
        opts = [torch.optim.SGD(net.parameters(), lr=0.0), torch.optim.SGD([r, t], lr=0.0), torch.optim.SGD([sc, sh], lr=0.0)]
        loss, lr_, ld_ = step(net, r, t, sc, sh, opts, torch.from_numpy(img), torch.from_numpy(dpt), 1, kx, ky, N, S, 0.01, 10.0,
                              ray_idx=torch.from_numpy(ray_idx), noise=torch.from_numpy(noise))
        rel = lambda x, y: float(np.abs(np.asarray(x) - np.asarray(y)).max() / (np.abs(np.asarray(y)).max() + 1e-30))
        print("loss", float(loss), float(ld["loss"]), "| rel g_r", rel(r.grad[1].numpy(), grads["r"]), "g_t", rel(t.grad[1].numpy(), grads["t"]),
              "g_W(layers1.6)", rel(net.layers1[6].weight.grad.numpy(), grads["P"]["layers1.6.weight"]))
        return
    dev = torch.device(a.device)
    torch.manual_seed(42)
    H, W, hd, wd, V, N, S = 1080, 1920, 384, 672, 200, 1024, 128
    net = Field().to(dev)
    r = nn.Parameter(torch.zeros(V, 3, device=dev)); t = nn.Parameter(torch.zeros(V, 3, device=dev))
    sc = nn.Parameter(torch.ones(V, 1, device=dev)); sh = nn.Parameter(torch.zeros(V, 1, device=dev))
    opts = [torch.optim.Adam(net.parameters(), lr=1e-3), torch.optim.Adam([r, t], lr=5e-4), torch.optim.Adam([sc, sh], lr=5e-4)]
    frames = [(torch.rand(3, H, W, device=dev), torch.rand(hd, wd, device=dev) * 6.6 + 0.6) for _ in range(4)]
    kx, ky = 1.2, -1.2 * W / H
    sync = (lambda: torch.cuda.synchronize()) if dev.type == "cuda" else (lambda: None)
    for i in range(a.warmup): step(net, r, t, sc, sh, opts, *frames[i % 4], i % V, kx, ky, N, S, 0.01, 10.0)
    sync(); t0 = time.perf_counter()
    for i in range(a.steps): loss = step(net, r, t, sc, sh, opts, *frames[i % 4], i % V, kx, ky, N, S, 0.01, 10.0)[0]
    sync(); dt = (time.perf_counter() - t0) / a.steps
    print(json.dumps({"impl": "eager PyTorch statement of the reference step (autograd + torch.optim.Adam x3)", "device": str(dev),
                      "gpu": torch.cuda.get_device_name(0) if dev.type == "cuda" else None, "ms_per_step": round(dt * 1e3, 3),
                      "value": round(N * S / dt, 1), "unit": "ray-samples/s", "steps": a.steps, "loss": float(loss),
                      "tf32": bool(torch.backends.cuda.matmul.allow_tf32)}))


if __name__ == "__main__":
    main()

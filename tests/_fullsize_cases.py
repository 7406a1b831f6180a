"""Inputs of tests/test_gpu_fullsize_ref.py and of the generator of its stored reference results (tools/make_golden_fullsize.py):
configurations, seeded frames, seeded starting states.  Everything here is reproducible from seeds alone."""
import copy

import torch

from _cfg import default_cfg

CASES = {
    "C2_render": dict(H=1080, W=1920, hd=384, wd=672, V=200, N=1024, S=128, over={"training.pc_weight": [0.0, 0.0], "training.rgb_s_weight": [0.0, 0.0]}),
    "C2_full": dict(H=1080, W=1920, hd=384, wd=672, V=200, N=1024, S=128, over={}),
    "C3_ndc": dict(H=756, W=1008, hd=384, wd=512, V=20, N=1024, S=128,
                   over={"rendering.sample_option": "ndc", "rendering.dist_alpha": True, "rendering.depth_range": [0.0, 1.0],
                         "training.pc_weight": [0.0, 0.0], "training.rgb_s_weight": [0.0, 0.0]}),
    "C5_full": dict(H=1080, W=1920, hd=384, wd=672, V=200, N=4096, S=128, over={}),
    # the same C2 step with the high-frequency columns of the two encoding-fed layers damped by 2^-l (oracle.init_params(hf_damp)):
    # no ReLU-gate switches and no 2^9-amplified rounding in the encoding adjoint -> the strict 1e-4 gate on every pose gradient
    "C2_render_damped": dict(H=1080, W=1920, hd=384, wd=672, V=200, N=1024, S=128, damp=True,
                             over={"training.pc_weight": [0.0, 0.0], "training.rgb_s_weight": [0.0, 0.0]}),
}
N_PARAM_SAMPLE = 8192   # MLP-gradient entries stored per case (fixed, seeded draw): the full vector would not fit a small fixture


def set_cfg(cfg, overrides):
    """overrides: {'section.key': value}"""
    for k, v in (overrides or {}).items():
        sec, key = k.split(".")
        cfg[sec][key] = v
    return cfg


def case_cfg(c, base=None):
    cfg = copy.deepcopy(base) if base is not None else default_cfg()
    set_cfg(cfg, c["over"])
    cfg["training"]["n_training_points"] = c["N"]; cfg["rendering"]["num_points"] = c["S"]
    cfg["training"]["vis_reprojection_every"] = 10 ** 9
    return cfg


def frames(c, idx, seed):
    g = torch.Generator().manual_seed(seed)
    H, W, hd, wd = c["H"], c["W"], c["hd"], c["wd"]
    fx = 0.6 * W
    cam = torch.tensor([[2 * fx / W, 0, 0, 0], [0, -2 * fx / H, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
    # smooth frames / depth maps (low-res noise, bilinearly upsampled) so that the warped-RGB term sees image structure
    up = lambda t, size: torch.nn.functional.interpolate(t, size, mode="bilinear", align_corners=False)
    img = up(torch.rand(1, 3, 27, 48, generator=g), (H, W)).contiguous()
    ref = up(torch.rand(1, 3, 27, 48, generator=g), (H, W)).contiguous()
    dpt = (up(torch.rand(1, 1, 12, 21, generator=g), (hd, wd))[0] * 3.0 + 2.0).contiguous()
    rdpt = (dpt * (1 + 0.05 * up(torch.rand(1, 1, 6, 8, generator=g), (hd, wd))[0])).contiguous()
    return {"img": img, "img.idx": torch.tensor([idx]), "img.dpt": dpt, "img.camera_mat": cam, "img.scale_mat": torch.eye(4)[None],
            "img.ref_imgs": ref, "img.ref_dpts": rdpt, "img.ref_idxs": torch.tensor([idx + 1])}


def small_scene(H=48, W=64, hd=24, wd=32, V=4, seed=11):
    g = torch.Generator().manual_seed(seed)
    up = lambda t, size: torch.nn.functional.interpolate(t, size, mode="bilinear", align_corners=False)
    fx = 0.6 * W
    cam = torch.tensor([[2 * fx / W, 0, 0, 0], [0, -2 * fx / H, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
    img = up(torch.rand(1, 3, 6, 8, generator=g), (H, W)).contiguous()
    dpt = (up(torch.rand(1, 1, 6, 8, generator=g), (hd, wd))[0] * 3.0 + 2.0).contiguous()
    return {"img": img, "img.idx": torch.tensor([1]), "img.dpt": dpt, "img.camera_mat": cam, "img.scale_mat": torch.eye(4)[None],
            "img.depth": torch.rand(1, H, W, generator=g) * 5 + 0.5}


def start_state(cfg, V, net_seed, pose_seed, damp=False, geo=False):
    """parameters of the OfficialStaticNerf built under torch.manual_seed(net_seed) (the reference's torch init gives the same
    tensors), optionally damped (high-frequency encoding columns) or turned into a geometry field; seeded poses / distortions"""
    import nope_nerf_b200.model as mdl
    torch.manual_seed(net_seed)
    net = mdl.OfficialStaticNerf(cfg)
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    if damp:
        d = torch.ones(63)
        for l in range(10):
            d[3 + 6 * l:9 + 6 * l] = 2.0 ** (-l)
        sd["layers0.0.weight"] = sd["layers0.0.weight"] * d[None, :]
        w = sd["layers1.0.weight"].clone(); w[:, 256:] *= d[None, :]; sd["layers1.0.weight"] = w
    if geo:   # occupancy crosses the ray-marching threshold (alpha = 0.5 <=> density logit = 0) inside the sphere
        sd["fc_density.weight"] = sd["fc_density.weight"] * 10.0; sd["fc_density.bias"] = torch.zeros_like(sd["fc_density.bias"])
    g = torch.Generator().manual_seed(pose_seed)
    r = torch.randn(V, 3, generator=g) * 0.05; t = torch.randn(V, 3, generator=g) * 0.05
    scales = 1 + 0.1 * (torch.rand(V, 1, generator=g) - 0.5); shifts = 0.1 * (torch.rand(V, 1, generator=g) - 0.5)
    return dict(net=sd, r=r, t=t, scales=scales, shifts=shifts)


def state_digest(state):
    return float(sum(v.double().sum() for v in state["net"].values()) + state["r"].double().sum() + state["t"].double().sum()
                 + state["scales"].double().sum() + state["shifts"].double().sum())


def param_sample_idx(n):
    return torch.randperm(n, generator=torch.Generator().manual_seed(2024))[:N_PARAM_SAMPLE]

"""CPU: pin the numpy oracle at model.hidden_dim 128 and 64 against fixtures written by the unmodified reference with the width
overridden (tools/make_golden.py hidden).  Same gates as tests/test_oracle_golden.py; the field's trunk is D wide and its rgb hidden
layer D/2 wide, everything else is unchanged."""
import numpy as np
import pytest
from oracle import nerf_oracle as O
from _util import load_golden, relmax, cfg_from_golden, check_param_digest

DIMS = (128, 64)
RENDER = ["render_tanks_noise", "render_ndc_distalpha", "render_tanks_noise_damped", "render_ndc_distalpha_damped"]


def golden_name(base, D):
    return base.replace("_damped", "_d%d_damped" % D) if base.endswith("_damped") else "%s_d%d" % (base, D)


def oracle_render(g, dtype):
    """fp32 / fp64 oracle of one render golden at its width: (outputs, gradients, d r, d t, raw prior depth)"""
    cfg = cfg_from_golden(g)
    D = int(g["hidden_dim"])
    P = {k: v.astype(dtype) for k, v in O.init_params(seed=int(g["seed"]), D=D, white_bkgd=cfg["white_background"],
                                                      hf_damp=bool(g["hf_damp"])).items()}
    H, W, cam, N = int(g["H"]), int(g["W"]), int(g["cam_id"]), int(g["N"])
    r, t = g["r"][cam].astype(dtype), g["t"][cam].astype(dtype)
    c2w = O.make_c2w(r, t, None)
    raw, _ = O.gather_prior_depth(g["dpt"], g["ray_idx"], H, W)
    depth = (raw.astype(dtype) * dtype(g["scale"]) + dtype(g["shift"])).astype(dtype)
    pix = O.pixels_from_idx(g["ray_idx"], H, W, dtype)
    out, cache = O.render_forward(P, pix, depth, c2w, dtype(g["kx"]), dtype(g["ky"]), cfg, noise=g["noise"].astype(dtype),
                                  eval_=bool(g["eval_mode"]))
    m = out["mask"]
    gdp = np.zeros(N, dtype); gdg = np.zeros(N, dtype)
    gdp[m] = g["g_dp"]; gdg[m] = g["g_dg"]
    gr = O.render_backward(P, cache, g["g_rgb"].astype(dtype), gdp, gdg)
    g_r, g_t = O.make_c2w_bwd(r, t, None, gr["c2w"])
    return out, gr, g_r, g_t, raw


@pytest.mark.parametrize("D", DIMS)
def test_mlp(D):
    g = load_golden("mlp_alpha_softplus_d%d" % D)
    assert int(g["hidden_dim"]) == D
    P = O.init_params(seed=int(g["seed"]), D=D)
    assert P["fc_feature.weight"].shape == (D, D) and P["rgb_layers.0.weight"].shape == (D // 2, D + 27)
    rgb, a, cache = O.mlp_forward(P, g["pts"], g["dirs"], dist_alpha=bool(g["dist_alpha"]), occ_activation=str(g["occ"]))
    assert relmax(rgb, g["rgb"]) < 2e-6
    assert relmax(a, g["a"]) < 2e-5
    G, gp, gd = O.mlp_backward(P, cache, g["g_rgb"], g["g_a"])
    assert relmax(gp, g["g_pts"]) < 1e-4
    assert relmax(gd, g["g_dirs"]) < 1e-4
    assert check_param_digest(g, G) < 1e-4


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("base", RENDER)
def test_render(base, D):
    """outputs <= 2e-5 of the reference; gradients <= max(2e-4, 3 x |reference - fp64 oracle|) (test_oracle_golden.test_render)"""
    g = load_golden(golden_name(base, D))
    assert int(g["hidden_dim"]) == D and int(g["S"]) == 128
    cam = int(g["cam_id"])
    out, gr, g_r, g_t, raw = oracle_render(g, np.float32)
    out64, gr64, g_r64, g_t64, _ = oracle_render(g, np.float64)
    for o in (out, out64):
        assert relmax(o["rgb"], g["rgb"]) < 2e-5
        assert relmax(o["depth_pred"], g["depth_pred"]) < 2e-5
        assert relmax(o["depth_gt"], g["depth_gt"]) < 2e-5
        assert relmax(o["alpha"], g["alpha"]) < 5e-5

    def gate(a32, a64, ref):
        env = relmax(a64, ref)
        assert env < 2e-2, env
        assert relmax(a32, ref) < max(2e-4, 3 * env), (relmax(a32, ref), env)
    gate(gr["c2w"], gr64["c2w"], g["grad_c2w"])
    gate(g_r, g_r64, g["grad_r"][cam])
    gate(g_t, g_t64, g["grad_t"][cam])
    gate(np.array([(gr["depth"] * raw).sum(), gr["depth"].sum()]), np.array([(gr64["depth"] * raw).sum(), gr64["depth"].sum()]),
         np.array([g["grad_scale"], g["grad_shift"]]))
    env = check_param_digest(g, gr64["params"])
    assert check_param_digest(g, gr["params"]) < max(5e-4, 3 * env)


@pytest.mark.parametrize("D", DIMS)
def test_train_step_full_losses(D):
    """two reference Trainer.train_step calls with the default loss set at width D vs oracle.train_step"""
    g = load_golden("train_full_losses_d%d" % D)
    assert int(g["hidden_dim"]) == D
    idx = int(g["idx"])

    def run(dtype):
        cfg = dict(O.DEFAULT_CFG); cfg["num_points"] = int(g["S"])
        state = dict(P={k: v.astype(dtype) for k, v in O.init_params(seed=int(g["seed"]), D=D).items()},
                     r=g["r0"].astype(dtype).copy(), t=g["t0"].astype(dtype).copy(),
                     scales=g["scales0"].astype(dtype).copy(), shifts=g["shifts0"].astype(dtype).copy())
        hist = []
        for it in range(int(g["steps"])):
            ref = dict(img=g["ref"].astype(dtype), dpt=g["rdpt"].astype(dtype), idx=int(g["ref_idx"]), w_pc=1.0, w_rgb_s=1.0)
            hist.append(O.train_step(state, g["img"].astype(dtype), g["dpt"].astype(dtype), g["ray_idx_%d" % it], g["noise_%d" % it].astype(dtype),
                                     idx, dtype(g["kx"]), dtype(g["ky"]), cfg, w_rgb=1.0, w_depth=0.04, rgb_loss_type="l1", ref=ref)[:2])
        return state, hist
    st32, h32 = run(np.float32)
    st64, h64 = run(np.float64)
    for it in range(int(g["steps"])):
        ld, gr = h32[it]; _, gr64 = h64[it]
        for k in ("loss", "loss_rgb", "loss_depth", "loss_pc", "loss_rgb_s"):
            ref = float(np.ravel(g["loss_%d.%s" % (it, k)])[0])
            assert abs(float(ld[k]) - ref) / abs(ref) < 5e-5, (it, k, float(ld[k]), ref)
        for nm, key in (("r", "grad_r_%d"), ("t", "grad_t_%d")):
            ref = g[key % it][idx]
            assert relmax(gr[nm], ref) < max(2e-4, 3 * relmax(gr64[nm], ref)), (it, nm)
        if it == 0:   # after one Adam update (~ lr * sign(g)) fp32 and the reference differ by Adam noise on near-zero gradients
            env = check_param_digest(g, gr64["P"], prefix="pg_0.")
            assert check_param_digest(g, gr["P"], prefix="pg_0.") < max(5e-4, 3 * env)
    for key in ("r", "t", "scales", "shifts"):
        assert relmax(st32[key] - g[key + "0"], g[key + "_end"] - g[key + "0"]) < 2e-3, key


@pytest.mark.parametrize("D", (64, 128, 256))
def test_module_layout_matches_reference_shapes(D):
    """OfficialStaticNerf at width D: the reference's state_dict keys and shapes, and a flat layout of nnb_num_params(D) floats"""
    from nope_nerf_b200 import _lib as L
    from nope_nerf_b200.model.official_nerf import OfficialStaticNerf
    from _cfg import default_cfg
    cfg = default_cfg(); cfg["model"]["hidden_dim"] = D
    net = OfficialStaticNerf(cfg)
    sd = net.state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [(n, tuple(s)) for n, s in O.param_shapes(D)]
    assert net.num_params == L.num_params(D) == O.flatten_params(O.init_params(seed=1, D=D)).size
    assert {64: 44516, 128: 158660, 256: L.NUM_PARAMS}[D] == net.num_params
    fresh = OfficialStaticNerf(cfg)
    fresh.load_state_dict(sd)
    assert all(np.array_equal(fresh.state_dict()[k].numpy(), v.numpy()) for k, v in sd.items())


def test_unsupported_width_rejected():
    from nope_nerf_b200 import _lib as L
    from nope_nerf_b200.model.official_nerf import OfficialStaticNerf
    from _cfg import default_cfg
    cfg = default_cfg(); cfg["model"]["hidden_dim"] = 96
    with pytest.raises(NotImplementedError, match="64, 128, 256"):
        OfficialStaticNerf(cfg)
    assert L.lib.nnb_num_params(96) == 0 and L.lib.nnb_num_params(512) == 0
    assert L.lib.nnb_workspace_bytes_dim(64, 32, L.STASH, L.ENGINE_TC, 96) == 0
    assert L.lib.nnb_num_params(0) == L.NUM_PARAMS
    for eng in (L.ENGINE_SIMT, L.ENGINE_TC):
        assert L.lib.nnb_workspace_bytes_dim(64, 32, L.STASH, eng, 0) == L.lib.nnb_workspace_bytes(64, 32, L.STASH, eng)
        assert L.lib.nnb_workspace_bytes_dim(64, 32, L.STASH, eng, 64) < L.lib.nnb_workspace_bytes_dim(64, 32, L.STASH, eng, 128) < \
            L.lib.nnb_workspace_bytes(64, 32, L.STASH, eng)

"""GPU: the reference-image stage with `training.with_ssim: True` and `training.detach_ref_img: False`.
(1) Trainer steps against the reference Trainer (tests/golden/train_full_{ssim,undetached}*.npz) on the SIMT and tensor-core engines;
(2) ops.refstage against the fp64 oracle (tests/_refopts_oracle.py) at the golden size and at C2 size, reference-view gradients
included; (3) the CUDA-graph step equals the eager step with both options on."""
import numpy as np
import pytest
import torch

from _util import load_golden, relmax
from oracle import nerf_oracle as O
import _refopts_oracle as RO
from test_gpu_parity import _build_trainer, _report, cuda, engines
from test_refopts_golden import CASES, _refcfg, _stage_inputs

pytestmark = pytest.mark.gpu


def _apply_cfg(trainer, g):
    c = _refcfg(g)
    trainer.detach_ref_img = c["detach_ref_img"]; trainer.shift_first = c["shift_first"]
    trainer.loss.cfg["with_ssim"] = c["with_ssim"]


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("eng,fused", [("simt", True), ("tc", True), ("simt", False)])
def test_trainer_refopts_step_vs_reference_golden(name, eng, fused, monkeypatch):
    """gates of test_gpu_parity.test_trainer_step_vs_reference_golden ('exact' weight gradients); the r / t / scales / shifts gradients
    are compared over every row, so the reference view's rows are checked too.  fused=False takes Trainer.compute_loss (the general
    path, torch.optim.Adam) instead of the fixed kernel sequence of the graph step"""
    if dict(engines()).get(eng) is None:
        pytest.skip("engine disabled")
    g = load_golden(name)
    trainer, net, pose, dist = _build_trainer(g, eng, True)
    _apply_cfg(trainer, g)
    trainer.fused_adam = fused
    from _util import check_param_digest
    kx, ky = float(g["kx"]), float(g["ky"])
    cam = np.array([[kx, 0, 0, 0], [0, ky, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], np.float32)
    data = {"img": torch.from_numpy(g["img"])[None], "img.idx": torch.tensor([int(g["idx"])]),
            "img.dpt": torch.from_numpy(g["dpt"])[None], "img.camera_mat": torch.from_numpy(cam)[None],
            "img.scale_mat": torch.eye(4)[None], "img.ref_imgs": torch.from_numpy(g["ref"])[None],
            "img.ref_dpts": torch.from_numpy(g["rdpt"])[None], "img.ref_idxs": torch.tensor([int(g["ref_idx"])])}
    state = {"it": 0}
    monkeypatch.setattr(torch, "randperm", lambda n, device=None: cuda(g["ray_idx_%d" % state["it"]]))
    monkeypatch.setattr(torch, "rand", lambda *a, **k: cuda(g["noise_%d" % state["it"]])[None])
    worst = {}
    ri = int(g["ref_idx"])
    for it in range(int(g["steps"])):
        state["it"] = it
        ld = trainer.train_step(data, it=it + 1, epoch=0, scheduling_start=10000, render_path="/tmp")
        torch.cuda.synchronize()
        for k in ("loss", "loss_rgb", "loss_depth", "l2_mean", "loss_pc", "loss_rgb_s"):
            ref = float(g["loss_%d.%s" % (it, k)].reshape(-1)[0]); got = float(ld[k].reshape(-1)[0])
            worst["loss_%d_%s" % (it, k)] = abs(got - ref) / max(abs(ref), 1e-3)
        for nm, p in (("r", pose.r), ("t", pose.t), ("scales", dist.global_scales), ("shifts", dist.global_shifts)):
            got, ref = p.grad.cpu().numpy(), g["grad_%s_%d" % (nm, it)]
            worst["g_%s_%d" % (nm, it)] = relmax(got, ref)
            if np.abs(ref[ri]).max() > 0:                                   # the reference view's row on its own
                worst["g_%s_ref_%d" % (nm, it)] = relmax(got[ri], ref[ri])
        worst["g_params_%d" % it] = check_param_digest(g, {n: p.grad.cpu().numpy() for n, p in net.named_parameters()}, prefix="pg_%d." % it)
    worst["r_end"] = relmax(pose.r.detach().cpu().numpy() - g["r0"], g["r_end"] - g["r0"])
    worst["t_end"] = relmax(pose.t.detach().cpu().numpy() - g["t0"], g["t_end"] - g["t0"])
    worst["params_end"] = check_param_digest(g, {n: p.detach().cpu().numpy() for n, p in net.named_parameters()}, prefix="pend.")
    _report("refopts/%s/%s%s" % (name, eng, "" if fused else "-general"), **worst)
    if not _refcfg(g)["detach_ref_img"]:
        assert any(k.startswith("g_r_ref") for k in worst)
    for k, v in worst.items():
        if k.startswith("loss"):
            assert v < 2e-4, (k, v)
        elif k.startswith("g_params"):
            assert v < 5e-3, (k, v)
        elif k.startswith("g_"):
            assert v < 2e-3, (k, v)
        elif k in ("r_end", "t_end"):
            assert v < 5e-2, (k, v)
        else:
            assert v < 1e-3, (k, v)


def _native_vs_oracle(img, ref, dpt, rdpt, c2w, c2wr, dc, dr, is_last, kx, ky, with_ssim, tag):
    from nope_nerf_b200 import ops
    cfg = dict(O.REF_CFG, with_ssim=with_ssim, detach_ref_img=False)
    f64 = lambda a: np.asarray(a, np.float64)
    l, gr = RO.ref_stage(f64(img), f64(ref), f64(dpt), f64(rdpt), f64(c2w), f64(c2wr), dc[0], dc[1], dr[0], dr[1], is_last, kx, ky, cfg=cfg)
    c2w_t = cuda(c2w).float().requires_grad_(True); dist = torch.tensor(dc, device="cuda", requires_grad=True)
    c2wr_t = cuda(c2wr).float().requires_grad_(True); distr = torch.tensor(dr, device="cuda", requires_grad=True)
    total, losses = ops.refstage(c2w_t, dist, c2wr_t, distr, cuda(img).float(), cuda(ref).float(), cuda(dpt).float(), cuda(rdpt).float(),
                                 is_last, kx, ky, with_ssim=with_ssim)
    total.backward()
    e = dict(loss_pc=abs(losses[0].item() - l["loss_pc"]) / l["loss_pc"], loss_rgb_s=abs(losses[1].item() - l["loss_rgb_s"]) / l["loss_rgb_s"],
             g_c2w=relmax(c2w_t.grad.cpu().numpy()[:3], gr["c2w"][:3]),
             g_dist=relmax(dist.grad.cpu().numpy(), np.array([gr["scale"], gr["shift"]])),
             g_c2w_ref=relmax(c2wr_t.grad.cpu().numpy()[:3], gr["c2w_ref"][:3]),
             g_dist_ref=relmax(distr.grad.cpu().numpy(), np.array([gr["scale_ref"], gr["shift_ref"]])))
    _report("native_refopts/%s" % tag, **e)
    assert all(v <= 1e-4 for v in e.values()), e


@pytest.mark.parametrize("name", ["train_full_ssim", "train_full_undetached_lastview"])
@pytest.mark.parametrize("with_ssim", [False, True])
def test_native_refstage_refopts_vs_oracle(name, with_ssim):
    """golden inputs (8 x 12 grid); is_last False / True"""
    g, c2w, c2wr, dc, dr, is_last = _stage_inputs(name)
    _native_vs_oracle(g["img"], g["ref"], g["dpt"], g["rdpt"], c2w, c2wr, dc, dr, is_last, float(g["kx"]), float(g["ky"]), with_ssim,
                      "%s/ssim%d" % (name, with_ssim))


@pytest.mark.parametrize("is_last", [False, True])
def test_native_refstage_refopts_c2_size_vs_oracle(is_last):
    """C2 size: 384 x 672 DPT maps, 96 x 168 low-resolution grid, both options on"""
    rng = np.random.default_rng(17)
    H, W, hd, wd = 216, 384, 384, 672
    up = lambda t, size: torch.nn.functional.interpolate(torch.from_numpy(t)[None], size, mode="bilinear", align_corners=False)[0].numpy()
    img = up(rng.uniform(0, 1, (3, 18, 32)).astype(np.float32), (H, W)); ref = up(rng.uniform(0, 1, (3, 18, 32)).astype(np.float32), (H, W))
    dpt = up(rng.uniform(1.5, 6, (1, 12, 21)).astype(np.float32), (hd, wd))[0]; rdpt = up(rng.uniform(1.5, 6, (1, 12, 21)).astype(np.float32), (hd, wd))[0]
    c2w = O.make_c2w(rng.normal(0, 0.03, 3).astype(np.float32), rng.normal(0, 0.05, 3).astype(np.float32)).astype(np.float32)
    c2wr = O.make_c2w(rng.normal(0, 0.03, 3).astype(np.float32), rng.normal(0, 0.05, 3).astype(np.float32)).astype(np.float32)
    _native_vs_oracle(img, ref, dpt, rdpt, c2w, c2wr, (1.03, 0.02), (0.97, -0.04), is_last, 1.2, -1.6, True, "c2/last%d" % is_last)


def test_refstage_grad_ref_needs_output_pointers():
    """flag 16 without g_c2w_ref / g_dist_ref is a checked error (return code), nothing is launched"""
    from nope_nerf_b200 import ops, _lib as L
    import ctypes as C
    g, c2w, c2wr, dc, dr, is_last = _stage_inputs("train_full_undetached")
    a = L.RefStageArgs()
    t = {k: cuda(v).float() for k, v in dict(img=g["img"], ref=g["ref"], dpt=g["dpt"], rdpt=g["rdpt"], c2w=c2w, c2wr=c2wr).items()}
    d1, d2, losses = torch.tensor(dc, device="cuda"), torch.tensor(dr, device="cuda"), torch.zeros(2, device="cuda")
    hd, wd = g["dpt"].shape
    ws = torch.empty(L.lib.nnb_refstage_workspace_bytes_flags(hd, wd, 4, 1 | 16), dtype=torch.uint8, device="cuda")
    a.img_cur, a.img_ref, a.dpt_cur, a.dpt_ref = t["img"].data_ptr(), t["ref"].data_ptr(), t["dpt"].data_ptr(), t["rdpt"].data_ptr()
    a.c2w_cur, a.c2w_ref, a.dist_cur, a.dist_ref = t["c2w"].data_ptr(), t["c2wr"].data_ptr(), d1.data_ptr(), d2.data_ptr()
    a.H, a.W, a.h_d, a.w_d, a.pc_ratio, a.is_last, a.flags = g["img"].shape[1], g["img"].shape[2], hd, wd, 4, 0, 1 | 16
    a.kx, a.ky, a.nearest_limit, a.w_pc, a.w_rgb_s = float(g["kx"]), float(g["ky"]), 0.01, 1.0, 1.0
    a.losses, a.workspace, a.workspace_bytes = losses.data_ptr(), ws.data_ptr(), ws.numel()
    assert L.lib.nnb_refstage(C.byref(a), ops._stream()) != 0
    assert b"g_c2w_ref" in L.lib.nnb_last_error()
    a.flags = 1 | 8                                          # SSIM needs the larger workspace of the flag-aware query
    ws_small = torch.empty(L.lib.nnb_refstage_workspace_bytes(hd, wd, 4), dtype=torch.uint8, device="cuda")
    a.workspace, a.workspace_bytes = ws_small.data_ptr(), ws_small.numel()
    assert L.lib.nnb_refstage(C.byref(a), ops._stream()) != 0
    assert L.lib.nnb_refstage_workspace_bytes_flags(hd, wd, 4, 1) == L.lib.nnb_refstage_workspace_bytes(hd, wd, 4)


def test_graph_replay_equals_eager_refopts(monkeypatch):
    """test_gpu_parity.test_graph_replay_equals_eager_on_injected_draws(full=True) with with_ssim and detach_ref_img False, same gates;
    the reference views' rows of r / t / shifts are part of the compared parameters"""
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200 import ops
    from _cfg import default_cfg
    ops.set_default_engine("tc")
    H, W, V, N, S, hd, wd = 96, 128, 6, 256, 64, 24, 32
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(3)
    up = lambda t, size: torch.nn.functional.interpolate(t, size, mode="bilinear", align_corners=False)
    frames = [dict(img=up(torch.rand(1, 3, 12, 16, generator=g), (H, W)).cuda(), dpt=(up(torch.rand(1, 1, 6, 8, generator=g), (hd, wd))[0] * 3 + 2).cuda())
              for _ in range(V)]
    draws = [(torch.randperm(H * W, generator=g)[:N].cuda(), torch.rand(N, S, generator=g).cuda()) for _ in range(8)]
    ray_buf = torch.zeros(N, dtype=torch.int64, device=dev); noise_buf = torch.zeros(1, N, S, device=dev)
    monkeypatch.setattr(torch, "randperm", lambda n, device=None: ray_buf)
    monkeypatch.setattr(torch, "rand", lambda *a, **k: noise_buf)
    cam = torch.tensor([[1.2, 0, 0, 0], [0, -1.6, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], dtype=torch.float32)[None]
    res = {}
    for mode in (False, True):
        cfg = default_cfg()
        cfg["training"]["n_training_points"] = N; cfg["rendering"]["num_points"] = S
        cfg["training"]["annealing_epochs"] = 10
        cfg["training"]["with_ssim"] = True; cfg["training"]["detach_ref_img"] = False
        net = mdl.OfficialStaticNerf(cfg)
        net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in O.init_params(seed=9, hf_damp=True).items()})
        model = mdl.get_model(mdl.Renderer(net, cfg["rendering"], device=dev), cfg, device=dev)
        pose = mdl.LearnPose(V, True, True, cfg).to(dev); dist = mdl.Learn_Distortion(V, True, True, cfg).to(dev)
        with torch.no_grad():
            pose.r.copy_(torch.randn(V, 3, generator=torch.Generator().manual_seed(5)) * 0.03); pose.t.copy_(torch.randn(V, 3, generator=torch.Generator().manual_seed(6)) * 0.03)
        opt = torch.optim.Adam(model.parameters(), lr=1e-3); opt_p = torch.optim.Adam(pose.parameters(), lr=5e-4)
        opt_d = torch.optim.Adam(dist.parameters(), lr=5e-4)
        tr = mdl.Trainer(model, opt, cfg["training"], device=dev, optimizer_pose=opt_p, pose_param_net=pose, optimizer_distortion=opt_d,
                         distortion_net=dist, use_cuda_graph=mode, pixel_sampler="randperm")
        losses = []
        for it in range(8):
            ray_buf.copy_(draws[it][0]); noise_buf[0].copy_(draws[it][1])
            i = (it * 2 + 1) % (V - 1)
            data = {"img": frames[i]["img"], "img.idx": torch.tensor([i]), "img.dpt": frames[i]["dpt"], "img.camera_mat": cam,
                    "img.scale_mat": torch.eye(4)[None], "img.ref_imgs": frames[i + 1]["img"], "img.ref_dpts": frames[i + 1]["dpt"],
                    "img.ref_idxs": torch.tensor([i + 1])}
            ld = tr.train_step(data, it=it, epoch=it, scheduling_start=3, render_path=None)
            losses.append([ld[k].item() for k in ("loss", "loss_rgb", "loss_depth", "loss_pc", "loss_rgb_s")])
        if mode:
            gsteps = [v for v in tr._gsteps.values() if v]
            assert len(gsteps) == 1 and gsteps[0].graph is not None and gsteps[0].calls == 8
        res[mode] = (np.array(losses), net.flat_weights().detach().cpu().numpy().copy(), pose.r.detach().cpu().numpy().copy(),
                     pose.t.detach().cpu().numpy().copy(), dist.global_shifts.detach().cpu().numpy().copy())
    le, lg = res[False][0], res[True][0]
    w0 = O.flatten_params(O.init_params(seed=9, hf_damp=True)).astype(np.float64)
    ug, ue = res[True][1] - w0, res[False][1] - w0
    r0 = (torch.randn(V, 3, generator=torch.Generator().manual_seed(5)) * 0.03).numpy().astype(np.float64)
    t0 = (torch.randn(V, 3, generator=torch.Generator().manual_seed(6)) * 0.03).numpy().astype(np.float64)
    upd = lambda k, p0: np.linalg.norm((res[True][k] - p0) - (res[False][k] - p0)) / max(np.linalg.norm(res[False][k] - p0), 1e-30)
    e = dict(loss=np.abs(le - lg).max() / np.abs(le).max(), w=np.linalg.norm(ug - ue) / np.linalg.norm(ue), w_max=relmax(ug, ue),
             r=upd(2, r0), t=upd(3, t0), r_abs=np.abs(res[True][2] - res[False][2]).max(), t_abs=np.abs(res[True][3] - res[False][3]).max(),
             shifts=relmax(res[True][4], res[False][4]))
    _report("graph_vs_eager/refopts", **e)
    assert le[:, 3].min() > 0 and le[:, 4].min() > 0, le
    # view 5 is only ever a reference view: its shift moved through the reference-view gradients
    assert abs(res[False][4][5, 0]) > 0 and abs(res[True][4][5, 0]) > 0, res[False][4]
    assert e["loss"] < 1e-5, (e, le, lg)
    assert e["w"] < 2e-2 and e["r"] < 0.1 and e["t"] < 0.1 and e["r_abs"] < 5e-4 and e["t_abs"] < 5e-4 and e["shifts"] < 1e-3, e

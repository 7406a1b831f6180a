"""CPU: the reference-image stage with `training.with_ssim: True` and `training.detach_ref_img: False`.
(1) tests/_refopts_oracle.py against reference Trainer steps (tests/golden/train_full_{ssim,undetached}*.npz, tools/make_golden.py refopts),
including the reference view's rows of the pose and distortion gradients; (2) with both options at their defaults it equals
oracle.ref_stage; (3) nnb_refstage.cuh's __host__ __device__ functions, run on the CPU by tools/refstage_host_check.cu, against it."""
import itertools
import os
import subprocess
import numpy as np
import pytest
from oracle import nerf_oracle as O
from _util import ROOT, load_golden, relmax
import _refopts_oracle as RO

CASES = ["train_full_ssim", "train_full_undetached", "train_full_undetached_lastview", "train_full_ssim_undetached_shiftfirst"]


def _refcfg(g):
    cfg = dict(O.REF_CFG)
    cfg["with_ssim"] = bool(g.get("cfg.training.with_ssim", False))
    cfg["detach_ref_img"] = bool(g.get("cfg.training.detach_ref_img", True))
    cfg["shift_first"] = bool(g.get("cfg.training.shift_first", False))
    return cfg


def _run(g, dtype):
    cfg = dict(O.DEFAULT_CFG); cfg["num_points"] = int(g["S"])
    state = dict(P={k: v.astype(dtype) for k, v in O.init_params(seed=int(g["seed"])).items()},
                 r=g["r0"].astype(dtype).copy(), t=g["t0"].astype(dtype).copy(),
                 scales=g["scales0"].astype(dtype).copy(), shifts=g["shifts0"].astype(dtype).copy())
    hist = []
    for it in range(int(g["steps"])):
        ref = dict(img=g["ref"].astype(dtype), dpt=g["rdpt"].astype(dtype), idx=int(g["ref_idx"]), w_pc=1.0, w_rgb_s=1.0)
        hist.append(RO.train_step(state, g["img"].astype(dtype), g["dpt"].astype(dtype), g["ray_idx_%d" % it], g["noise_%d" % it].astype(dtype),
                                  int(g["idx"]), dtype(g["kx"]), dtype(g["ky"]), cfg, ref, _refcfg(g)))
    return state, hist


@pytest.mark.parametrize("name", CASES)
def test_refopts_oracle_vs_reference_steps(name):
    """losses and the r / t / scales / shifts gradients of every row (the reference view's rows are non-zero exactly when
    detach_ref_img is False), then the parameters after the Adam updates; gates of test_oracle_golden.test_train_step_full_losses"""
    g = load_golden(name)
    idx, ri = int(g["idx"]), int(g["ref_idx"])
    undetached = not bool(g.get("cfg.training.detach_ref_img", True))
    st32, h32 = _run(g, np.float32)
    st64, h64 = _run(g, np.float64)
    for it in range(int(g["steps"])):
        (ld, gr), (_, gr64) = h32[it], h64[it]
        for k in ("loss", "loss_rgb", "loss_depth", "loss_pc", "loss_rgb_s"):
            ref = float(np.ravel(g["loss_%d.%s" % (it, k)])[0])
            assert abs(float(ld[k]) - ref) / abs(ref) < 5e-5, (it, k, float(ld[k]), ref)
        rows = [idx, ri] if undetached else [idx]
        for nm in ("r", "t", "scales", "shifts"):
            ref = g["grad_%s_%d" % (nm, it)]
            for row in rows:
                if nm == "scales" and row == int(g["V"]) - 1:
                    assert ref[row].max() == 0.0 and gr[nm][row].max() == 0.0          # fixed scale of the last view
                    continue
                env = relmax(gr64[nm][row], ref[row])
                assert relmax(gr[nm][row], ref[row]) < max(2e-4, 3 * env), (it, nm, row, relmax(gr[nm][row], ref[row]), env)
                assert np.abs(ref[row]).max() > 0.0, (it, nm, row)
            others = np.delete(ref, rows, 0)
            assert np.abs(others).max() == 0.0 and np.abs(np.delete(gr[nm], rows, 0)).max() == 0.0
    for key in ("r", "t", "scales", "shifts"):
        upd_ref = g[key + "_end"] - g[key + "0"]
        assert relmax(st32[key] - g[key + "0"], upd_ref) < 2e-3, key


def _stage_inputs(name, dtype=np.float32):
    g = load_golden(name)
    idx, ri, V = int(g["idx"]), int(g["ref_idx"]), int(g["V"])
    state = dict(r=g["r0"], t=g["t0"], scales=g["scales0"], shifts=g["shifts0"])
    c2w = O.make_c2w(g["r0"][idx], g["t0"][idx]).astype(dtype); c2wr = O.make_c2w(g["r0"][ri], g["t0"][ri]).astype(dtype)
    s_c, h_c, _ = O._distortion(state, idx, np.float32, {}); s_r, h_r, _ = O._distortion(state, ri, np.float32, {})
    return g, c2w, c2wr, (float(s_c), float(h_c)), (float(s_r), float(h_r)), idx == V - 1


@pytest.mark.parametrize("name", ["train_full_losses", "train_full_lastview"])
def test_refopts_oracle_defaults_equal_oracle(name):
    g, c2w, c2wr, dc, dr, is_last = _stage_inputs(name, np.float64)
    args = (g["img"].astype(np.float64), g["ref"].astype(np.float64), g["dpt"], g["rdpt"], c2w, c2wr, dc[0], dc[1], dr[0], dr[1], is_last,
            float(g["kx"]), float(g["ky"]))
    l0, g0 = O.ref_stage(*args)
    l1, g1 = RO.ref_stage(*args)
    for k in l0:
        assert abs(l0[k] - l1[k]) <= 1e-12 * abs(l0[k])
    for k in g0:
        assert np.abs(np.asarray(g0[k]) - np.asarray(g1[k])).max() <= 1e-10 * max(np.abs(np.asarray(g0[k])).max(), 1.0), k
    assert "c2w_ref" not in g1


def test_ssim_map_adjoint_matches_finite_differences():
    rng = np.random.default_rng(4)
    x = rng.uniform(0, 1, (3, 5, 3)); y = np.clip(x + rng.normal(0, 0.2, x.shape), 0, 1)
    w = rng.normal(0, 1, x.shape)
    _, gy = RO.ssim_map(x, y, w)
    eps = 1e-6
    for k in rng.choice(x.size, 12, replace=False):
        d = np.zeros(x.size); d[k] = eps; d = d.reshape(x.shape)
        fd = ((RO.ssim_map(x, y + d) - RO.ssim_map(x, y - d)) * w).sum() / (2 * eps)
        assert abs(fd - gy.reshape(-1)[k]) < 1e-6 * max(1.0, abs(fd)), (k, fd, gy.reshape(-1)[k])


def _host_exe():
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = os.path.join(ROOT, "nope_nerf_b200", "build", "refstage_host_check")
    src = os.path.join(ROOT, "tools", "refstage_host_check.cu"); hdr = os.path.join(ROOT, "nope_nerf_b200", "csrc", "nnb_refstage.cuh")
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(exe), exist_ok=True)
        subprocess.check_call([nvcc, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", exe, src])
    return exe


_GRID = list(itertools.product([False, True], repeat=5))    # scale_pcs, shift_first, detach_rgbs_scale, with_ssim, detach_ref_img


@pytest.mark.parametrize("name", ["train_full_ssim", "train_full_undetached_lastview"])     # is_last = False / True
@pytest.mark.parametrize("scale_pcs,shift_first,detach,with_ssim,detach_ref", _GRID)
def test_refstage_refopts_device_math_on_host(name, scale_pcs, shift_first, detach, with_ssim, detach_ref, tmp_path):
    """the .cuh functions on the CPU vs _refopts_oracle.ref_stage over every combination of the stage's flags; gates of
    test_host.test_refstage_device_math_on_host, the reference view's gradients gated like the current view's"""
    exe = _host_exe()
    g, c2w, c2wr, dc, dr, is_last = _stage_inputs(name)
    H, W = g["img"].shape[1:]; hd, wd = g["dpt"].shape
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as fo:
        np.array([H, W, hd, wd, 4, int(is_last), int(scale_pcs), int(detach)], np.int32).tofile(fo)
        np.array([g["kx"], g["ky"], 0.01, dc[0], dc[1], dr[0], dr[1], 1.0, 1.0], np.float32).tofile(fo)
        for arr in (c2w, c2wr, g["img"], g["ref"], g["dpt"], g["rdpt"]):
            np.ascontiguousarray(arr, np.float32).tofile(fo)
    subprocess.check_call([exe, fin, fout, "1" if shift_first else "0", str((8 if with_ssim else 0) | (0 if detach_ref else 16))])
    o = np.fromfile(fout, np.float32)
    cfg = dict(O.REF_CFG, scale_pcs=scale_pcs, detach_rgbs_scale=detach, shift_first=shift_first, with_ssim=with_ssim, detach_ref_img=detach_ref)
    l, gr = RO.ref_stage(g["img"], g["ref"], g["dpt"], g["rdpt"], c2w, c2wr, dc[0], dc[1], dr[0], dr[1], is_last,
                         np.float32(g["kx"]), np.float32(g["ky"]), cfg=cfg)
    assert abs(o[0] - l["loss_pc"]) < 2e-6 * abs(l["loss_pc"]) and abs(o[1] - l["loss_rgb_s"]) < 2e-6 * abs(l["loss_rgb_s"])
    assert relmax(o[2:18].reshape(4, 4)[:3], gr["c2w"][:3]) < 2e-5
    assert abs(o[18] - gr["scale"]) < 2e-5 * max(abs(gr["scale"]), 1.0) and abs(o[19] - gr["shift"]) < 2e-5 * max(abs(gr["shift"]), 1.0)
    assert relmax(o[20:22], gr["kxy"]) < 5e-5, (o[20:22], gr["kxy"])
    if detach_ref:
        assert o.size == 22
    else:
        assert o.size == 40
        assert relmax(o[22:38].reshape(4, 4)[:3], gr["c2w_ref"][:3]) < 2e-5
        assert abs(o[38] - gr["scale_ref"]) < 2e-5 * max(abs(gr["scale_ref"]), 1.0)
        assert abs(o[39] - gr["shift_ref"]) < 2e-5 * max(abs(gr["shift_ref"]), 1.0)

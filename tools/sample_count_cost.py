#!/usr/bin/env python
"""Train-step time of the C2 workload (1080x1920, V = 200, 1024 rays, uniform + jitter, rgb L1 + depth L1, Adam x3, whole-step CUDA graph;
bench.py's headline configuration) at rendering.num_points S = 96, 128, 192, 256 and 512 on the tensor-core engine, and at S = 96 and 192
also on the exact-fp32 SIMT engine (which served every S outside {32, 64, 128, 256} before the tensor-core engine took any S in
[16, 1024]).  One trainer per (engine, S), timed in alternating windows of K steps (CUDA events), median over the windows.
    python tools/sample_count_cost.py [K] [windows]

--dump DIR [--lib-root ROOT]: instead of timing, write the outputs and every gradient of one seeded render call (forward + backward,
1024 rays) at S = 32, 64, 256 on the tensor-core engine and S = 100, 256 on the SIMT engine as .npy files, using the nope_nerf_b200
package found under ROOT (default: this tree), so that two builds can be compared file by file."""
import json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMP = sys.argv[sys.argv.index("--dump") + 1] if "--dump" in sys.argv else None
LIB_ROOT = os.path.abspath(sys.argv[sys.argv.index("--lib-root") + 1]) if "--lib-root" in sys.argv else ROOT
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, LIB_ROOT)
import numpy as np
import torch

TIMED = [("tc", 96), ("tc", 128), ("tc", 192), ("tc", 256), ("tc", 512), ("simt", 96), ("simt", 192)]
DUMPED = [("tc", 32), ("tc", 64), ("tc", 256), ("simt", 100), ("simt", 256)]


def dump(out_dir):
    from nope_nerf_b200 import ops, _lib as L
    from oracle import nerf_oracle as O
    assert os.path.dirname(os.path.abspath(ops.__file__)) == os.path.join(LIB_ROOT, "nope_nerf_b200"), ops.__file__
    os.makedirs(out_dir, exist_ok=True)
    N, H, W = 1024, 1080, 1920
    flat = torch.from_numpy(O.flatten_params(O.init_params(seed=5))).cuda()
    for eng, S in DUMPED:
        rng = np.random.default_rng(S)
        cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
        c2w = cu(O.make_c2w(rng.normal(0, 0.05, 3).astype(np.float32), rng.normal(0, 0.05, 3).astype(np.float32)))
        cam = torch.diag(torch.tensor([1.2, -2.1, -1.0, 1.0])).cuda()
        ray_idx = cu(rng.permutation(H * W)[:N].astype(np.int64)); noise = cu(rng.uniform(0, 1, (N, S)).astype(np.float32))
        dpt = cu(rng.uniform(0.6, 7.2, (384, 672)).astype(np.float32))
        g_rgb = cu(rng.normal(0, 1, (N, 3)).astype(np.float32)); g_dp = cu(rng.normal(0, 1, N).astype(np.float32))
        g_dg = cu(rng.normal(0, 1, N).astype(np.float32))
        engine = {"tc": L.ENGINE_TC, "simt": L.ENGINE_SIMT}[eng]
        call = ops.RenderCall(flat, c2w, cam, N=N, S=S, flags=ops.flags_from_cfg(dict(O.DEFAULT_CFG), "softplus"), engine=engine, near=0.01,
                              far=10.0, ray_idx=ray_idx, depth_map=dpt, scale=torch.tensor([1.05]).cuda(), shift=torch.tensor([0.02]).cuda(),
                              noise=noise, H=H, W=W, want_z_alpha=True, stash=True)
        assert call.args.engine == engine
        out = dict(rgb=call.rgb, depth_pred=call.depth_pred, depth_gt=call.depth_gt, mask=call.mask, z_vals=call.z_vals, alpha=call.alpha)
        out = {k: v.clone() for k, v in out.items()}
        g = dict(g_w=torch.zeros(L.NUM_PARAMS, device="cuda"), g_c2w=torch.zeros(4, 4, device="cuda"), g_cam=torch.zeros(4, 4, device="cuda"),
                 g_depth=torch.zeros(N, device="cuda"), g_ss=torch.zeros(2, device="cuda"))
        call.backward(g_rgb, g_dp, g_dg, g["g_w"], g["g_c2w"], g["g_cam"], g["g_depth"], g["g_ss"])
        torch.cuda.synchronize()
        call.release()
        for k, v in list(out.items()) + list(g.items()):
            np.save(os.path.join(out_dir, "%s_s%d.%s.npy" % (eng, S, k)), v.cpu().numpy())
    print("dumped %d cases to %s" % (len(DUMPED), out_dir))


def timed(K, NWIN):
    import bench
    from nope_nerf_b200 import _lib as L
    dev = torch.device("cuda", 0); torch.cuda.set_device(0)
    _, frames = bench.synth_frames(bench.H, bench.W, bench.HD, bench.WD, bench.N_FRAMES, bench.V, dev, with_ref=False)
    trainers = {}
    for eng, S in TIMED:
        cfg = bench.make_cfg(bench.NRAYS)
        cfg["rendering"]["num_points"] = S
        tr = bench.build_trainer(cfg, dev, bench.V)
        tr.model.renderer.engine = {"tc": L.ENGINE_TC, "simt": L.ENGINE_SIMT}[eng]
        trainers[(eng, S)] = tr

    def run(key, n, start):
        for i in range(start, start + n):
            trainers[key].train_step(frames[i % len(frames)], it=i, epoch=0, scheduling_start=10000, render_path=None)

    for key in trainers:
        run(key, 30, 0)                              # eager first step, capture, clocks settle
    torch.cuda.synchronize()
    times = {key: [] for key in trainers}
    for w in range(NWIN):
        for key in trainers:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); run(key, K, 30 + w * K); e1.record(); torch.cuda.synchronize()
            times[key].append(e0.elapsed_time(e1) / K)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {}
    for (eng, S), v in times.items():
        med = float(np.median(v))
        out["%s_s%d" % (eng, S)] = {"ms_per_step_median": round(med, 4), "ms_per_step_min": round(min(v), 4), "ms_per_step_max": round(max(v), 4),
                                    "ray_samples_per_s": round(bench.NRAYS * S / (med / 1e3), 1)}
    for S in sorted({S for eng, S in TIMED if eng == "simt"}):
        out["simt_over_tc_s%d" % S] = round(out["simt_s%d" % S]["ms_per_step_median"] / out["tc_s%d" % S]["ms_per_step_median"], 3)
    out.update(steps_per_window=K, windows=NWIN, gpu=q.splitlines()[0] if q else torch.cuda.get_device_name(0))
    print(json.dumps(out))


if __name__ == "__main__":
    if DUMP:
        dump(DUMP)
    else:
        args = [a for a in sys.argv[1:] if not a.startswith("--")]
        timed(int(args[0]) if args else 20, int(args[1]) if len(args) > 1 else 5)

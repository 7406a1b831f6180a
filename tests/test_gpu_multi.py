"""Data-parallel correctness on REAL GPUs (needs >= 2 devices; `gpurun --gpus 2`): the 2-rank Trainer against the 1-rank Trainer on
identical pixel / jitter draws.
  dp_mode='rays'  : both ranks see the same view and take rays rank::2 -> the summed gradient buffer must equal the single-GPU one
  dp_mode='views' : each rank trains its own view (config 5) -> the summed buffer must equal the mean of the two single-view buffers
for the NCCL exchange (two graphs around torch.distributed.all_reduce) and for the peer-memory exchange (nnb_allreduce_adam: P2P
all-reduce fused with Adam inside ONE graph).  The worker also asserts that the ranks' parameters stay bit-identical."""
import os
import subprocess
import sys
import numpy as np
import pytest
import torch

from _util import ROOT, relmax

pytestmark = pytest.mark.gpu
WORKER = os.path.join(ROOT, "tests", "_dp_worker.py")


def _run(tmp, name, mode, graph, peer, world):
    out = os.path.join(tmp, name + ".npz")
    env = dict(os.environ); env.pop("RANK", None); env.pop("WORLD_SIZE", None); env.pop("LOCAL_RANK", None)
    if world == 1:
        cmd = [sys.executable, WORKER, out, mode, str(graph), str(peer)]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
               "--master-port", str(29500 + (os.getpid() % 500)), WORKER, out, mode, str(graph), str(peer)]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    z = np.load(out)
    return {k: z[k] for k in z.files}


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("graph,peer", [(0, 0), (1, 0), (0, 1), (1, 1)])
def test_dp_rays_equals_single_gpu(graph, peer, tmp_path):
    one = _run(str(tmp_path), "one", "rays", 0, 0, 1)
    two = _run(str(tmp_path), "two", "rays", graph, peer, 2)
    assert int(two["peer"]) == peer and int(two["graph"]) == graph
    n = one["g_first"].size
    e = dict(g=relmax(two["g_first"][:n - 4], one["g_first"][:n - 4]), loss=abs(float(two["loss0"]) - float(one["loss0"])) / abs(float(one["loss0"])),
             r=relmax(two["r"], one["r"]), t=relmax(two["t"], one["t"]), shifts=relmax(two["shifts"], one["shifts"]),
             w=np.linalg.norm(two["w"] - one["w"]) / np.linalg.norm(one["w"]))
    print("dp rays graph=%d peer=%d" % (graph, peer), e)
    assert e["g"] < 1e-5 and e["loss"] < 1e-6, e                 # summed gradient buffer == single-GPU buffer (fp32 atomics order)
    assert e["r"] < 1e-3 and e["t"] < 1e-3 and e["shifts"] < 1e-3 and e["w"] < 1e-4, e


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("peer", [0, 1])
def test_dp_views_equals_mean_of_single_views(peer, tmp_path):
    a = _run(str(tmp_path), "v1", "single:1", 0, 0, 1)
    b = _run(str(tmp_path), "v3", "single:3", 0, 0, 1)
    two = _run(str(tmp_path), "two", "views", 1, peer, 2)
    n = a["g_first"].size
    ref = 0.5 * (a["g_first"] + b["g_first"])
    e = dict(g=relmax(two["g_first"][:n - 4], ref[:n - 4]), loss=abs(float(two["loss0"]) - 0.5 * (float(a["loss0"]) + float(b["loss0"]))))
    print("dp views peer=%d" % peer, e)
    assert e["g"] < 1e-5, e

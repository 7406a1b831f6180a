"""BASELINE.json configs[0] / SURVEY.md 8(d) "C1": the reference's train.py, UNCHANGED (oracle/_ref/train.py), driven end to end
against the drop-in through the INTEGRATION.md binding on a fixture scene in the loader's on-disk layout (tools/run_ref_train.py):
DataLoader / OurDataset batches with pin_memory, three torch.optim.Adam instances, CheckpointIO save, scale / shift logging per view,
render_visdata, the auto-scheduler and `reset_parameters()` at scheduling_start.  The same harness then runs the reference's own
Trainer; both runs must produce the same artefacts and scalar tags, and comparable losses (the RNG streams differ: whole-step CUDA
graph + hash pixel sampler on our side)."""
import json
import os
import subprocess
import sys
import pytest

from _util import ROOT

pytestmark = pytest.mark.gpu
sys.path.insert(0, ROOT)
from oracle import ref_harness as RH  # noqa: E402

if not RH.available():
    pytest.skip("oracle/_ref missing (oracle/vendor_ref.py needs a reference checkout)", allow_module_level=True)


def _run(tmp, impl):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_ref_train.py"), os.path.join(tmp, impl), "--impl", impl],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    return json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1]), r.stdout


def test_reference_train_py_runs_unchanged_on_the_dropin(tmp_path):
    ours, log = _run(str(tmp_path), "ours")
    ref, _ = _run(str(tmp_path), "reference")
    assert ours["trainer_class"] == "nope_nerf_b200.model.training.Trainer" and ref["trainer_class"] == "model.training.Trainer"
    assert ours["train_steps"] == ref["train_steps"] == 27 and ours["render_visdata_calls"] == ref["render_visdata_calls"] == 4
    assert ours["losses_finite"] and ours["n_loss_logs"] == 27
    assert ours["scalar_tags"] == ref["scalar_tags"]                       # every loss_dict key train.py logs, per-view scale / shift, lr, psnr
    assert ours["vis_dirs"] == ref["vis_dirs"] and ours["vis_files"] == ref["vis_files"]
    assert set(ours["checkpoints"]) == {"model.pt", "model_pose.pt", "model_distortion.pt"}
    # CheckpointIO wrote the reference's format: same parameter names / shapes, same optimizer state entries and step count (file
    # sizes differ by a few KB: our parameters and Adam moments are views of flat buffers, which torch.save stores once)
    assert ours["model_keys_shapes"] == ref["model_keys_shapes"] and ours["optimizer_state_entries"] == ref["optimizer_state_entries"] == 24
    assert ours["optimizer_state_keys"] == ref["optimizer_state_keys"] and ours["optimizer_step"] == ref["optimizer_step"] == ours["checkpoint_it"] + 1
    assert ours["checkpoint_keys"] == ref["checkpoint_keys"] and ours["n_model_tensors"] == ref["n_model_tensors"] == 24
    assert abs(ours["loss_first"] - ref["loss_first"]) < 0.1 * ref["loss_first"], (ours["loss_first"], ref["loss_first"])
    assert all(abs(a - b) < 1.0 for a, b in zip(ours["train_psnr_per_epoch"], ref["train_psnr_per_epoch"])), (ours, ref)
    assert "[Epoch 02]" in log and "Saving checkpoint" in log

"""GPU: the reference's unmodified train.py runs on the drop-in with rendering.normal_loss: True (tools/run_ref_train.py
--normal-loss, the plumbing run of tests/test_gpu_train_plumbing.py); only where a reference copy exists under oracle/_ref."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
sys.path.insert(0, ROOT)
from oracle import ref_harness as RH  # noqa: E402

if not RH.available():
    pytest.skip("oracle/_ref missing (oracle/vendor_ref.py needs a reference checkout)", allow_module_level=True)


def test_reference_train_py_runs_with_normal_loss(tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_ref_train.py"), str(tmp_path / "ours"), "--impl", "ours",
                        "--normal-loss"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    assert out["trainer_class"] == "nope_nerf_b200.model.training.Trainer"
    assert out["train_steps"] == 27 and out["losses_finite"] and out["n_loss_logs"] == 27

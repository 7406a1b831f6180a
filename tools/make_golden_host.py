#!/usr/bin/env python
"""Stored reference results of tests/test_host.py::test_rgb_s_loss_with_ssim_vs_live_reference: the UNMODIFIED reference's
Loss.get_rgb_s_loss (value, gradients with respect to both images) and compute_ssim_loss on the CPU, on the test's seeded inputs.

    python tools/make_golden_host.py          # needs oracle/_ref; writes tests/golden/rgb_s_loss.npz"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_harness as RH  # noqa: E402
from test_host import rgb_s_inputs  # noqa: E402

if __name__ == "__main__":
    RH.import_reference("cpu")
    import model.losses as ref_losses                              # the reference's module (oracle/_ref on sys.path)
    a, b, valid = rgb_s_inputs()
    out = {"ssim_map": ref_losses.compute_ssim_loss(a, b).numpy()}
    for with_ssim in (False, True):
        cfg = {"depth_loss_type": "l1", "with_ssim": with_ssim, "with_auto_mask": False, "match_method": "dense"}
        x, y = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        v = ref_losses.Loss(cfg).get_rgb_s_loss(x, y, valid)
        v.backward()
        out.update({"value_%d" % with_ssim: float(v.detach()), "gx_%d" % with_ssim: x.grad.numpy(), "gy_%d" % with_ssim: y.grad.numpy()})
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "rgb_s_loss.npz"), **out)

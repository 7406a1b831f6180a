#!/usr/bin/env python
"""Stored reference results of tests/test_host.py::test_resident_dataset_equals_reference_dataloader_items: the UNMODIFIED
reference loader (dataloading.get_dataloader -> OurDataset -> DataLoader(batch_size=1)) reads the fixture scene of
tools/run_ref_train.write_scene; this writes tests/golden/dataloader_items.npz with

  * the loaded DataField as ResidentDataset.from_reference_field reads it (imgs as their 8-bit codes when code / 255 rebuilds
    every float exactly, DPT maps, K, ref_img, random_ref),
  * every item the DataLoader yields under random.seed(11): per key the shape, the dtype and either the value (small tensors) or the
    field frame it equals exactly (checked here, bit for bit).

    python tools/make_golden_dataloader.py          # needs oracle/_ref"""
import os
import random
import sys
import tempfile
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
from oracle import ref_harness as RH  # noqa: E402
from run_ref_train import write_scene  # noqa: E402

if __name__ == "__main__":
    tmp = tempfile.mkdtemp()
    write_scene(os.path.join(tmp, "data", "Test", "images"), V=10)
    RH.install_stubs()
    sys.path.insert(0, RH.REF)
    import dataloading as dl                                      # the reference's package, unchanged
    cfg = dl.load_config(os.path.join(RH.REF, "configs", "Test", "images.yaml"), os.path.join(RH.REF, "configs", "default.yaml"))
    cfg["dataloading"].update(path=os.path.join(tmp, "data", "Test"), n_workers=0, resize_factor=None, random_ref=2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                           # pin_memory=True without a GPU
        loader, fields = dl.get_dataloader(cfg, mode="train", shuffle=False)
        random.seed(11)
        items = list(loader)
    f = fields["img"]
    imgs = np.asarray(f.imgs, np.float32); dpts = np.asarray(f.dpt_depth, np.float32)
    codes = np.rint(imgs.astype(np.float64) * 255.0).astype(np.uint8)
    assert np.array_equal((codes / 255.0).astype(np.float32), imgs), "8-bit codes do not rebuild the frames exactly"
    out = dict(imgs_u8=codes, dpt_depth=dpts, K=np.asarray(f.K), ref_img=int(bool(f.ref_img)), random_ref=int(f.random_ref),
               N_imgs=int(f.N_imgs), n_items=len(items))
    frames = {"imgs": torch.from_numpy(imgs), "dpt_depth": torch.from_numpy(dpts)}
    for i, it in enumerate(items):
        out["item%d_keys" % i] = np.array(sorted(it))
        for k, v in it.items():
            pre = "item%d_%s" % (i, k)
            out[pre + "_shape"] = np.asarray(tuple(v.shape)); out[pre + "_dtype"] = np.array(str(v.dtype))
            if v.numel() <= 64:
                out[pre + "_value"] = v.numpy()
                continue
            src = [(name, j) for name, t in frames.items() for j in range(t.shape[0])
                   if tuple(t[j].shape) == tuple(v.shape[1:]) and torch.equal(t[j], v[0])]
            assert src, (i, k)
            out[pre + "_src"] = np.array(src[0][0]); out[pre + "_frame"] = src[0][1]
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "dataloader_items.npz"), **out)

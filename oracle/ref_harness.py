"""TEST INFRASTRUCTURE — imports the UNMODIFIED reference from oracle/_ref/ (oracle/vendor_ref.py) and builds its own
Trainer so that tests/, bench.py's reference arm and tools/psnr_parity.py can run the reference itself (CPU or cuda)
beside the CUDA path.  Nothing under nope_nerf_b200/ imports this module.

Harness-side shims, none of which carries arithmetic (SURVEY.md 8(c)); reference files are never edited:
  * stub modules for imageio / matplotlib / timm / lpips / skimage (imported at module scope by model/training.py:7,
    model/common.py:4, DPT/dpt/vit.py:3, model/eval_images.py); `imageio` gets PIL-backed imread / imwrite / mimwrite so
    train.py can load a fixture scene,
  * device == cpu only: torch.Tensor.cuda -> identity (hard-coded .cuda() in model/losses.py:84,162-194) and
    model.common.transform_to_world default device -> cpu (model/common.py:113).  On cuda the reference runs as is.
"""
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(HERE, "_ref")
_state = {"mdl": None, "cpu_patched": False}


def available():
    return os.path.isfile(os.path.join(REF, "model", "training.py"))


def _imageio_shim():
    import numpy as np
    m = types.ModuleType("imageio")

    def imread(path, *a, **k):
        from PIL import Image
        return np.asarray(Image.open(path))

    def imwrite(path, arr, *a, **k):
        from PIL import Image
        arr = np.asarray(arr)
        if arr.dtype != np.uint8:
            arr = np.clip(arr, 0, 255).astype(np.uint8) if arr.max() > 1.5 else (np.clip(arr, 0, 1) * 255).astype(np.uint8)
        Image.fromarray(arr).save(path)

    def mimwrite(path, frames, *a, **k):        # video writing is outside the hot path: keep the first frame as evidence
        imwrite(os.path.splitext(path)[0] + "_frame0.png", frames[0])
    m.imread = imread; m.imwrite = imwrite; m.mimwrite = mimwrite
    m.v2 = m
    return m


def install_stubs():
    if "imageio" not in sys.modules:
        sys.modules["imageio"] = _imageio_shim()
    for name in ("matplotlib", "matplotlib.pyplot", "timm", "lpips", "skimage", "skimage.metrics"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.modules["skimage"].metrics = sys.modules["skimage.metrics"]


def import_reference(device="cpu"):
    """returns the reference's `model` package (imported from oracle/_ref)"""
    import torch
    if not available():
        raise RuntimeError("oracle/_ref is missing: run `python oracle/vendor_ref.py` beside a reference checkout")
    install_stubs()
    if REF not in sys.path:
        sys.path.insert(0, REF)
    if _state["mdl"] is None:
        import model as mdl                       # noqa: the REFERENCE's package (ours is nope_nerf_b200.model)
        assert os.path.abspath(mdl.__file__).startswith(REF), mdl.__file__
        _state["mdl"] = mdl
    if str(device).startswith("cpu") and not _state["cpu_patched"]:
        import model.common as mc
        import model.training as mt
        torch.Tensor.cuda = lambda self, *a, **k: self
        _orig = mc.transform_to_world

        def ttw(pixels, depth, camera_mat, world_mat=None, scale_mat=None, invert=True, device=torch.device("cpu")):
            return _orig(pixels, depth, camera_mat, world_mat, scale_mat, invert, device)
        mc.transform_to_world = ttw
        mt.transform_to_world = ttw
        _state["cpu_patched"] = True
    return _state["mdl"]


class fp64_mode:
    """Run the unmodified reference in float64 (its rounding-free twin, used as the envelope of the parity tests): torch's default
    dtype becomes float64 and the two places that hard-code float32 are bridged WITHOUT changing a value -- `arange_pixels` casts
    its (float32-computed) pixel grid up, and modules built inside the context are cast with .double() by RefRig."""
    active = False

    def __enter__(self):
        import torch
        import model.common as mc
        import model.training as mt
        self._dt = torch.get_default_dtype(); torch.set_default_dtype(torch.float64)
        self._orig = mc.arange_pixels
        orig = self._orig

        def arange_pixels64(*a, **k):
            loc, scaled = orig(*a, **k)
            return loc, scaled.double()
        self._mods = [m for m in (mc, mt, sys.modules.get("model.extracting_images"), sys.modules.get("model.eval_images"),
                                  sys.modules.get("model.eval_pose_one_epoch")) if m is not None and hasattr(m, "arange_pixels")]
        for m in self._mods:
            m.arange_pixels = arange_pixels64
        # transform_to_world builds float32 identity matrices when world_mat / scale_mat are omitted (common.py:125-128): hand it the
        # same identities in the working dtype
        self._ttw = (mc.transform_to_world, mt.transform_to_world)
        inner = mt.transform_to_world

        def ttw64(pixels, depth, camera_mat, world_mat=None, scale_mat=None, invert=True, device=None):
            eye = torch.eye(4, dtype=camera_mat.dtype, device=camera_mat.device)[None]
            kw = {} if device is None else {"device": device}
            return inner(pixels, depth, camera_mat, eye if world_mat is None else world_mat, eye if scale_mat is None else scale_mat, invert, **kw)
        mc.transform_to_world = ttw64; mt.transform_to_world = ttw64
        fp64_mode.active = True
        return self

    def __exit__(self, *exc):
        import torch
        import model.common as mc
        import model.training as mt
        for m in self._mods:
            m.arange_pixels = self._orig
        mc.transform_to_world, mt.transform_to_world = self._ttw
        torch.set_default_dtype(self._dt)
        fp64_mode.active = False


def load_default_cfg():
    import yaml
    with open(os.path.join(REF, "configs", "default.yaml")) as f:
        return yaml.safe_load(f)


def set_cfg(cfg, overrides):
    """overrides: {'section.key': value}"""
    for k, v in (overrides or {}).items():
        sec, key = k.split(".")
        cfg[sec][key] = v
    return cfg


class RefRig:
    """the reference's modules + optimizers + Trainer, wired the way train.py:49-160 wires them"""

    def __init__(self, cfg, V, device, state=None, learn_focal=False, init_c2w=None):
        import torch
        mdl = import_reference(device)
        self.mdl = mdl; self.cfg = cfg; self.device = torch.device(device)
        dev = self.device
        self.net = mdl.OfficialStaticNerf(cfg)
        self.rend = mdl.Renderer(self.net, cfg["rendering"], device=dev)
        self.model = mdl.nope_nerf(cfg, self.rend, None, device=dev)          # what get_model returns for depth.type None (config.py:4-17)
        self.pose = mdl.LearnPose(V, cfg["pose"]["learn_R"], cfg["pose"]["learn_t"], cfg, init_c2w=init_c2w).to(dev)
        self.dist = mdl.Learn_Distortion(V, cfg["distortion"]["learn_scale"], cfg["distortion"]["learn_shift"], cfg).to(dev)
        self.focal = mdl.LearnFocal(True, False, order=2).to(dev) if learn_focal else None
        if fp64_mode.active:
            for m in (self.net, self.pose, self.dist, self.focal):
                if m is not None: m.double()
        if state is not None:
            self.load_state(state)
        tr = cfg["training"]
        self.opt = torch.optim.Adam(self.model.parameters(), lr=tr["learning_rate"], weight_decay=tr.get("weight_decay", 0.0))
        self.opt_pose = torch.optim.Adam(self.pose.parameters(), lr=tr["pose_lr"])
        self.opt_dist = torch.optim.Adam(self.dist.parameters(), lr=tr["distortion_lr"])
        self.opt_focal = torch.optim.Adam(self.focal.parameters(), lr=tr.get("focal_lr", 1e-3)) if learn_focal else None
        self.trainer = mdl.Trainer(self.model, self.opt, tr, device=dev, optimizer_pose=self.opt_pose, pose_param_net=self.pose,
                                   optimizer_focal=self.opt_focal, focal_net=self.focal, optimizer_distortion=self.opt_dist,
                                   distortion_net=self.dist, cfg_all=cfg)

    def load_state(self, st):
        """st: dict(net=state_dict of OfficialStaticNerf, r, t, scales, shifts[, fx, fy]) as tensors / arrays"""
        import torch
        as_t = lambda x: x if isinstance(x, torch.Tensor) else torch.as_tensor(x)
        with torch.no_grad():
            if "net" in st:
                self.net.load_state_dict({k: as_t(v).to(self.device) for k, v in st["net"].items()})
            for name, prm in (("r", self.pose.r), ("t", self.pose.t), ("scales", self.dist.global_scales), ("shifts", self.dist.global_shifts)):
                if name in st:
                    prm.copy_(as_t(st[name]).to(self.device).reshape(prm.shape))
            if self.focal is not None and "fx" in st:
                self.focal.fx.copy_(as_t(st["fx"]).to(self.device).reshape(self.focal.fx.shape))
                self.focal.fy.copy_(as_t(st["fy"]).to(self.device).reshape(self.focal.fy.shape))

    def state(self):
        import torch
        out = dict(net={k: v.detach().clone() for k, v in self.net.state_dict().items()}, r=self.pose.r.detach().clone(),
                   t=self.pose.t.detach().clone(), scales=self.dist.global_scales.detach().clone(),
                   shifts=self.dist.global_shifts.detach().clone())
        if self.focal is not None:
            out["fx"] = self.focal.fx.detach().clone(); out["fy"] = self.focal.fy.detach().clone()
        return out

    def train_step(self, data, it=1, epoch=0, scheduling_start=10000):
        return self.trainer.train_step(data, it=it, epoch=epoch, scheduling_start=scheduling_start, render_path="/tmp")

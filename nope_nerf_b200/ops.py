"""Torch-facing wrappers over the C ABI: tensors in, tensors out, everything enqueued on the
current CUDA stream.  torch is plumbing here (device memory, streams, autograd glue);
all arithmetic of the hot path happens in libnope_nerf_b200.so."""
import ctypes as C
import torch
from . import _lib as L

_DEFAULT_ENGINE = [L.ENGINE_TC]


def set_default_engine(name):
    _DEFAULT_ENGINE[0] = {"simt": L.ENGINE_SIMT, "tc": L.ENGINE_TC}[name]


def default_engine():
    return _DEFAULT_ENGINE[0]


TC_MIN_S = 16   # samples per ray: the tensor-core engine's lower limit; both engines go up to 1024


def pick_engine(engine, S):
    """the tensor-core engine serves 16 <= S <= 1024 samples per ray; fewer samples run on the exact-fp32 SIMT engine (still CUDA;
    there is no CPU path), which serves 2 <= S <= 1024.  An explicit ENGINE_SIMT is kept at every S."""
    if engine is None:
        engine = _DEFAULT_ENGINE[0]
    if engine == L.ENGINE_TC and S < TC_MIN_S:
        return L.ENGINE_SIMT
    return engine


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(t, name, allow_pinned=False):
    """device tensors only; `allow_pinned` additionally admits page-locked HOST tensors, which the kernels read in
    place over PCIe through the unified address space (used for the frame / DPT map, of which a step touches N pixels)"""
    if t is None or t.is_cuda:
        return
    if allow_pinned and t.is_pinned():
        return
    raise RuntimeError("nope_nerf_b200: %s must live on a CUDA device (no CPU fallback exists)" % name)


def _f32c(t):
    if t is None:
        return None
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.contiguous().float()
    return t


def flags_from_cfg(cfg, occ_activation="softplus", eval_=False, shift_first=False):
    """cfg = the reference's cfg['rendering'] dict (configs/default.yaml:32-44)."""
    f = 0
    if cfg["dist_alpha"]: f |= L.DIST_ALPHA
    if cfg["sample_option"] == "ndc": f |= L.NDC
    elif cfg["sample_option"] != "uniform":
        raise ValueError("sample_option must be 'uniform' or 'ndc' (model/rendering.py:98-101)")
    if cfg["normalise_ray"]: f |= L.NORMALISE
    if cfg["use_ray_dir"]: f |= L.USE_DIR
    if cfg["white_background"]: f |= L.WHITE_BG
    if occ_activation == "softplus": f |= L.SOFTPLUS
    if eval_: f |= L.EVAL
    if shift_first: f |= L.SHIFT_FIRST
    if cfg.get("outside_steps", 0) != 0:
        raise NotImplementedError("rendering.outside_steps != 0 is not supported")
    return f


class _WorkspacePool:
    def __init__(self):
        self.free = {}

    def take(self, nbytes, device):
        key = (nbytes, device.index)
        lst = self.free.get(key)
        if lst:
            return lst.pop()
        return torch.empty(max(nbytes, 256), dtype=torch.uint8, device=device)

    def give(self, ws):
        self.free.setdefault((ws.numel(), ws.device.index), []).append(ws)


_pool = _WorkspacePool()


class RenderCall:
    """One forward launch + the state its backward needs (workspace with the stash)."""
    frame = False         # FrameRenderCall: the differentiable frame's training pair
    exact_frame = False   # ExactFrameRenderCall: that pair on the exact-fp32 engine
    t_min = None          # frame_render_call(t_min): that pair with early ray termination (the _tmin calls); None: without
    stash_tmin = False    # stash_render_call(t_min): the per-sample stash pair with early ray termination (nnb_render_fwd_tmin / _bwd_tmin)
    exact_stash = False   # exact_stash_render_call(t_min): that pair on the exact-fp32 engine (the _tmin_engine calls on ENGINE_SIMT)

    def __init__(self, weights, c2w, cam, *, N, S, flags, engine, near, far, ray_idx=None, pixels=None, depth=None,
                 depth_map=None, scale=None, shift=None, noise=None, H=0, W=0, want_z_alpha=False, stash=False, hidden_dim=256):
        frame, exact = self.frame, self.exact_frame
        if self.stash_tmin:
            if want_z_alpha:
                raise ValueError("stash_render_call: want_z_alpha is not supported (no per-sample outputs)")
            if self.exact_stash:
                if not 2 <= S <= 1024:
                    raise ValueError("exact_stash_render_call needs 2 <= S <= 1024 (got %d)" % S)
                engine = L.ENGINE_SIMT
            elif pick_engine(engine, S) != L.ENGINE_TC:
                raise ValueError("stash_render_call runs on the tensor-core engine only (16 <= S <= 1024)")
            stash = True
        elif frame:
            if want_z_alpha:
                raise ValueError("FrameRenderCall: want_z_alpha is not supported (no per-sample outputs)")
            if exact:
                if not 2 <= S <= 1024:
                    raise ValueError("ExactFrameRenderCall needs 2 <= S <= 1024 (got %d)" % S)
                engine = L.ENGINE_SIMT
            elif pick_engine(engine, S) != L.ENGINE_TC:
                raise ValueError("FrameRenderCall runs on the tensor-core engine only (16 <= S <= 1024)")
            stash = True
        for n_, t_ in (("weights", weights), ("c2w", c2w), ("camera_mat", cam), ("ray_idx", ray_idx), ("pixels", pixels),
                       ("depth", depth), ("noise", noise)):
            _need_cuda(t_, n_)
        _need_cuda(depth_map, "depth_map")
        dev = weights.device
        self.keep = [weights, c2w, cam, ray_idx, pixels, depth, depth_map, scale, shift, noise]
        a = L.RenderArgs()
        a.weights = L.ptr(weights); a.c2w = L.ptr(c2w); a.cam = L.ptr(cam)
        a.ray_idx = L.ptr(ray_idx); a.pixels = L.ptr(pixels); a.depth = L.ptr(depth); a.depth_map = L.ptr(depth_map)
        a.scale = L.ptr(scale); a.shift = L.ptr(shift); a.noise = L.ptr(noise)
        a.N, a.S, a.H, a.W = N, S, H, W
        if depth_map is not None:
            a.h_d, a.w_d = depth_map.shape[-2], depth_map.shape[-1]
        a.near_, a.far_ = float(near), float(far)
        engine = pick_engine(engine, S)
        if stash and not frame and not self.stash_tmin:
            flags |= L.STASH
        a.flags = flags; a.engine = engine; a.hidden_dim = int(hidden_dim)
        self.hidden_dim = int(hidden_dim)
        self.rgb = torch.empty(N, 3, device=dev); self.depth_pred = torch.empty(N, device=dev)
        self.depth_gt = torch.empty(N, device=dev); self.mask = torch.empty(N, dtype=torch.uint8, device=dev)
        self.z_vals = torch.empty(N, S, device=dev) if want_z_alpha else None
        self.alpha = torch.empty(N, S, device=dev) if want_z_alpha else None
        a.rgb = L.ptr(self.rgb); a.depth_pred = L.ptr(self.depth_pred); a.depth_gt = L.ptr(self.depth_gt)
        a.mask = L.ptr(self.mask); a.z_vals = L.ptr(self.z_vals); a.alpha = L.ptr(self.alpha)
        if exact:
            nbytes = L.lib.nnb_render_frame_bwd_workspace_bytes_engine(N, S, int(hidden_dim), engine)
        elif frame:
            nbytes = L.lib.nnb_render_frame_bwd_workspace_bytes(N, S, int(hidden_dim))
        elif self.exact_stash:
            nbytes = L.lib.nnb_render_tmin_workspace_bytes_engine(N, S, int(hidden_dim), engine)
        elif self.stash_tmin:
            nbytes = L.lib.nnb_render_tmin_workspace_bytes(N, S, int(hidden_dim))
        else:
            nbytes = L.lib.nnb_workspace_bytes_dim(N, S, flags, engine, int(hidden_dim))
        if nbytes == 0:
            raise ValueError("nope_nerf_b200: hidden_dim %s is not supported (supported: %s)" % (hidden_dim, L.HIDDEN_DIMS))
        self.ws = _pool.take(nbytes, dev)
        a.workspace = L.ptr(self.ws); a.workspace_bytes = self.ws.numel()
        self.args = a; self.N = N; self.S = S; self.stash = stash; self.pooled = True
        if exact:
            L.check(L.lib.nnb_render_frame_train_fwd_engine(C.byref(a), _stream()), "nnb_render_frame_train_fwd_engine")
        elif self.t_min is not None:
            f = L.FrameArgs()
            f.fwd = a
            self.n_eval = torch.empty(N, dtype=torch.int32, device=dev)
            f.t_min = self.t_min; f.n_eval = L.ptr(self.n_eval); f.t_final = None
            name = ("nnb_render_fwd_tmin_engine" if self.exact_stash else "nnb_render_fwd_tmin") if self.stash_tmin \
                else "nnb_render_frame_train_fwd_tmin"
            L.check(getattr(L.lib, name)(C.byref(f), _stream()), name)
        elif frame:
            L.check(L.lib.nnb_render_frame_train_fwd(C.byref(a), _stream()), "nnb_render_frame_train_fwd")
        else:
            L.check(L.lib.nnb_render_fwd(C.byref(a), _stream()), "nnb_render_fwd")
        if not stash:
            self.release()

    def release(self):
        if self.ws is not None:
            if self.pooled: _pool.give(self.ws)
            self.ws = None

    def backward(self, g_rgb, g_depth_pred, g_depth_gt, g_weights, g_c2w, g_cam=None, g_depth=None, g_scale_shift=None):
        """all outputs are accumulated into (caller-zeroed) buffers; g_weights may be None (pose only)"""
        if self.ws is None:
            raise RuntimeError("backward called without a stashed forward")
        b = L.RenderBwdArgs()
        b.fwd = self.args
        keep = [_f32c(g_rgb), _f32c(g_depth_pred), _f32c(g_depth_gt)]
        b.g_rgb, b.g_depth_pred, b.g_depth_gt = L.ptr(keep[0]), L.ptr(keep[1]), L.ptr(keep[2])
        b.g_weights = L.ptr(g_weights); b.g_c2w = L.ptr(g_c2w); b.g_cam = L.ptr(g_cam); b.g_depth = L.ptr(g_depth)
        b.g_scale_shift = L.ptr(g_scale_shift)
        if self.exact_frame:
            L.check(L.lib.nnb_render_frame_train_bwd_engine(C.byref(b), _stream()), "nnb_render_frame_train_bwd_engine")
        elif self.exact_stash:
            L.check(L.lib.nnb_render_bwd_tmin_engine(C.byref(b), _stream()), "nnb_render_bwd_tmin_engine")
        elif self.stash_tmin:
            L.check(L.lib.nnb_render_bwd_tmin(C.byref(b), _stream()), "nnb_render_bwd_tmin")
        elif self.frame and self.t_min is not None:
            L.check(L.lib.nnb_render_frame_train_bwd_tmin(C.byref(b), _stream()), "nnb_render_frame_train_bwd_tmin")
        elif self.frame:
            L.check(L.lib.nnb_render_frame_train_bwd(C.byref(b), _stream()), "nnb_render_frame_train_bwd")
        else:
            L.check(L.lib.nnb_render_bwd(C.byref(b), _stream()), "nnb_render_bwd")
        self.release()


class FrameRenderCall(RenderCall):
    """RenderCall on the differentiable frame's training pair (tensor-core engine), with RenderCall's arguments, outputs, pooling and
    backward() rules.  The forward is nnb_render_frame_train_fwd, which gives the bits of RenderCall's forward, jitter included, and
    backward() is nnb_render_frame_train_bwd, in one workspace of nnb_render_frame_bwd_workspace_bytes: its only part that grows with S is
    one float per ray and 32-sample chunk, where RenderCall(stash=True) keeps every sample.  The workspace is always kept for backward(),
    so `stash` is implied and ignored.  want_z_alpha, and an engine that pick_engine does not resolve to the tensor-core engine
    (ENGINE_SIMT, or S < 16), are a ValueError, raised before any other check."""
    frame = True


_frame_tmin_calls = {}


def frame_render_call(t_min):
    """the FrameRenderCall class that trains with early ray termination at t_min (one class per value, cached): its forward is
    nnb_render_frame_train_fwd_tmin, which stops each ray as render_frame(t_min=...) does and exposes the samples each ray evaluated as
    the int32 [N] tensor `n_eval`, and backward() is nnb_render_frame_train_bwd_tmin, whose reverse rounds visit only the rays that
    evaluated each chunk.  The gradients are those of the truncated render.  t_min = 0 gives FrameRenderCall's bits.  A negative or NaN
    t_min is a ValueError."""
    t = float(t_min)
    if not t >= 0.0:
        raise ValueError("frame_render_call: t_min must be >= 0 (got %r)" % (t_min,))
    t = float(C.c_float(t).value)   # the value the library receives
    cls = _frame_tmin_calls.get(t)
    if cls is None:
        cls = type("FrameRenderCall_tmin", (FrameRenderCall,), {"t_min": t, "__doc__": frame_render_call.__doc__})
        _frame_tmin_calls[t] = cls
    return cls


_stash_tmin_calls = {}


def stash_render_call(t_min):
    """the RenderCall class that trains with early ray termination on the per-sample stash at t_min (one class per value, cached), with
    RenderCall's arguments, outputs, pooling and backward() rules.  Its forward is nnb_render_fwd_tmin, which stops each ray as
    render_frame(t_min=...) does, evaluates each sample once with the training stash, and exposes the samples each ray evaluated as the
    int32 [N] tensor `n_eval`; backward() is nnb_render_bwd_tmin, which runs the data-gradient chain and one weight-gradient stage on the
    rows the forward evaluated.  Outputs and n_eval are frame_render_call(t_min)'s bits, the gradients those of the truncated render;
    t_min = 0 gives RenderCall(stash=True)'s outputs.  Its workspace is the stash path's worst case (every ray runs every chunk), so
    `stash` is implied and ignored.  A negative or NaN t_min is a ValueError; so are want_z_alpha and an engine that pick_engine does not
    resolve to the tensor-core engine, raised before any other check."""
    t = float(t_min)
    if not t >= 0.0:
        raise ValueError("stash_render_call: t_min must be >= 0 (got %r)" % (t_min,))
    t = float(C.c_float(t).value)   # the value the library receives
    cls = _stash_tmin_calls.get(t)
    if cls is None:
        cls = type("StashRenderCall_tmin", (RenderCall,), {"t_min": t, "stash_tmin": True, "__doc__": stash_render_call.__doc__})
        _stash_tmin_calls[t] = cls
    return cls


_exact_stash_tmin_calls = {}


def exact_stash_render_call(t_min):
    """stash_render_call(t_min) on the exact-fp32 engine (nnb_render_fwd_tmin_engine / _bwd_tmin_engine on ENGINE_SIMT) at any S from 2 to
    1024, whatever `engine` says (one class per value, cached), with RenderCall's arguments, outputs, pooling and backward() rules and
    `n_eval`.  At S <= 32 (one round) its outputs and gradients are RenderCall(engine=ENGINE_SIMT, stash=True)'s bits and n_eval is S; at
    t_min = 0 its outputs are RenderCall(engine=ENGINE_SIMT)'s and its pose, camera and scale-shift gradients ExactFrameRenderCall's at
    every S; without jitter its outputs and n_eval are render_frame_engine(engine=ENGINE_SIMT, t_min=t_min)'s.  A negative or NaN t_min,
    want_z_alpha, and S outside 2..1024 are a ValueError."""
    t = float(t_min)
    if not t >= 0.0:
        raise ValueError("exact_stash_render_call: t_min must be >= 0 (got %r)" % (t_min,))
    t = float(C.c_float(t).value)   # the value the library receives
    cls = _exact_stash_tmin_calls.get(t)
    if cls is None:
        cls = type("ExactStashRenderCall_tmin", (RenderCall,), {"t_min": t, "stash_tmin": True, "exact_stash": True,
                                                               "__doc__": exact_stash_render_call.__doc__})
        _exact_stash_tmin_calls[t] = cls
    return cls


class ExactFrameRenderCall(FrameRenderCall):
    """FrameRenderCall on the exact-fp32 engine (nnb_render_frame_train_fwd_engine / _bwd_engine on ENGINE_SIMT) at any S from 2 to
    1024, whatever `engine` says.  Its forward gives the bits of RenderCall(engine=ENGINE_SIMT), jitter included; its workspace packs
    min(S, 32) stash rows per ray, so it stays near 650 KB per ray at D = 256 for every S where the exact stash path keeps about 20 KB per
    sample.  At S <= 32 the gradients are the exact stash path's bits.  want_z_alpha, or S outside 2..1024, is a ValueError."""
    exact_frame = True


def render_frame(weights, c2w, cam, *, N, S, flags, engine, near, far, ray_idx=None, pixels=None, depth=None, depth_map=None, scale=None,
                 shift=None, noise=None, H=0, W=0, want_z_alpha=False, stash=False, hidden_dim=256, t_min=0.0, want_stats=False):
    """nnb_render_frame: the forward of RenderCall (stash=False) on the tensor-core engine with compositing fused into the field's
    forward, in a workspace that does not grow with S.  t_min = 0 gives RenderCall's bits; t_min > 0 stops a ray after the first
    32-sample chunk that leaves its transmittance below t_min (the error bound is in include/nope_nerf_b200.h).
    Returns (rgb, depth_pred, depth_gt, mask), and (n_eval, t_final) after them with want_stats.  noise, want_z_alpha and stash are
    RenderCall's arguments and are rejected here, as is an engine other than the tensor-core engine (no fall-back)."""
    return _render_frame(L.lib.nnb_render_frame, "nnb_render_frame", L.lib.nnb_render_frame_workspace_bytes(N, S, int(hidden_dim)),
                         L.ENGINE_TC if engine is None else engine, weights, c2w, cam, N=N, S=S, flags=flags, near=near, far=far,
                         ray_idx=ray_idx, pixels=pixels, depth=depth, depth_map=depth_map, scale=scale, shift=shift, noise=noise, H=H, W=W,
                         want_z_alpha=want_z_alpha, stash=stash, hidden_dim=hidden_dim, t_min=t_min, want_stats=want_stats)


def render_frame_engine(weights, c2w, cam, *, N, S, flags, engine, near, far, ray_idx=None, pixels=None, depth=None, depth_map=None,
                        scale=None, shift=None, noise=None, H=0, W=0, want_z_alpha=False, stash=False, hidden_dim=256, t_min=0.0,
                        want_stats=False):
    """nnb_render_frame_engine: render_frame on either engine.  engine=None resolves through pick_engine (so S < 16 runs on the exact
    engine); ENGINE_TC gives render_frame's bits; ENGINE_SIMT renders on the exact-fp32 engine at any S from 2 to 1024, and at t_min = 0
    gives the bits of RenderCall(engine=ENGINE_SIMT, stash=False)."""
    engine = pick_engine(engine, S)
    return _render_frame(L.lib.nnb_render_frame_engine, "nnb_render_frame_engine",
                         L.lib.nnb_render_frame_workspace_bytes_engine(N, S, int(hidden_dim), engine), engine, weights, c2w, cam, N=N, S=S,
                         flags=flags, near=near, far=far, ray_idx=ray_idx, pixels=pixels, depth=depth, depth_map=depth_map, scale=scale,
                         shift=shift, noise=noise, H=H, W=W, want_z_alpha=want_z_alpha, stash=stash, hidden_dim=hidden_dim, t_min=t_min,
                         want_stats=want_stats)


def _render_frame(fn, name, nbytes, engine, weights, c2w, cam, *, N, S, flags, near, far, ray_idx, pixels, depth, depth_map, scale, shift,
                  noise, H, W, want_z_alpha, stash, hidden_dim, t_min, want_stats):
    """the body of render_frame / render_frame_engine: fn is the C entry point, nbytes its workspace size (0: the call rejects it)"""
    if noise is not None or want_z_alpha or stash:
        raise ValueError("render_frame: noise, want_z_alpha and stash are not supported (inference without jitter)")
    for n_, t_ in (("weights", weights), ("c2w", c2w), ("camera_mat", cam), ("ray_idx", ray_idx), ("pixels", pixels),
                   ("depth", depth), ("depth_map", depth_map)):
        _need_cuda(t_, n_)
    dev = weights.device
    f = L.FrameArgs()
    a = f.fwd
    a.weights = L.ptr(weights); a.c2w = L.ptr(c2w); a.cam = L.ptr(cam)
    a.ray_idx = L.ptr(ray_idx); a.pixels = L.ptr(pixels); a.depth = L.ptr(depth); a.depth_map = L.ptr(depth_map)
    a.scale = L.ptr(scale); a.shift = L.ptr(shift)
    a.N, a.S, a.H, a.W = N, S, H, W
    if depth_map is not None:
        a.h_d, a.w_d = depth_map.shape[-2], depth_map.shape[-1]
    a.near_, a.far_ = float(near), float(far)
    a.flags = flags; a.engine = engine; a.hidden_dim = int(hidden_dim)
    rgb = torch.empty(N, 3, device=dev); depth_pred = torch.empty(N, device=dev)
    depth_gt = torch.empty(N, device=dev); mask = torch.empty(N, dtype=torch.uint8, device=dev)
    a.rgb = L.ptr(rgb); a.depth_pred = L.ptr(depth_pred); a.depth_gt = L.ptr(depth_gt); a.mask = L.ptr(mask)
    n_eval = torch.empty(N, dtype=torch.int32, device=dev) if want_stats else None
    t_final = torch.empty(N, device=dev) if want_stats else None
    f.t_min = float(t_min); f.n_eval = L.ptr(n_eval); f.t_final = L.ptr(t_final)
    ws = _pool.take(nbytes, dev) if nbytes else None
    a.workspace = L.ptr(ws); a.workspace_bytes = 0 if ws is None else ws.numel()
    try:
        L.check(fn(C.byref(f), _stream()), name)
    finally:
        if ws is not None:
            _pool.give(ws)
    outs = (rgb, depth_pred, depth_gt, mask)
    return outs + (n_eval, t_final) if want_stats else outs


def render_frame_bwd(weights, c2w, cam, g_rgb, g_depth_pred, g_depth_gt, g_weights, g_c2w, g_cam=None, g_depth=None, g_scale_shift=None, *, N,
                     S, flags, near, far, ray_idx=None, pixels=None, depth=None, depth_map=None, scale=None, shift=None, H=0, W=0,
                     hidden_dim=256, engine=L.ENGINE_TC):
    """nnb_render_frame_bwd_engine: the gradients of render_frame_engine's outputs (t_min = 0) in a workspace whose only part that grows
    with S is one float per ray and 32-sample chunk.  engine: ENGINE_TC (nnb_render_frame_bwd's bits, 16 <= S <= 1024) or ENGINE_SIMT (the
    exact engine, 2 <= S <= 1024).  The g_* outputs follow RenderCall.backward (accumulated; g_depth overwritten; g_weights may be None).
    Returns (rgb, depth_pred, depth_gt, mask) of the call's own forward, the bits of render_frame_engine on that engine."""
    for n_, t_ in (("weights", weights), ("c2w", c2w), ("camera_mat", cam), ("ray_idx", ray_idx), ("pixels", pixels), ("depth", depth),
                   ("depth_map", depth_map)):
        _need_cuda(t_, n_)
    dev = weights.device
    b = L.RenderBwdArgs()
    a = b.fwd
    a.weights = L.ptr(weights); a.c2w = L.ptr(c2w); a.cam = L.ptr(cam)
    a.ray_idx = L.ptr(ray_idx); a.pixels = L.ptr(pixels); a.depth = L.ptr(depth); a.depth_map = L.ptr(depth_map)
    a.scale = L.ptr(scale); a.shift = L.ptr(shift)
    a.N, a.S, a.H, a.W = N, S, H, W
    if depth_map is not None:
        a.h_d, a.w_d = depth_map.shape[-2], depth_map.shape[-1]
    a.near_, a.far_ = float(near), float(far)
    a.flags = flags; a.engine = int(engine); a.hidden_dim = int(hidden_dim)
    rgb = torch.empty(N, 3, device=dev); depth_pred = torch.empty(N, device=dev)
    depth_gt = torch.empty(N, device=dev); mask = torch.empty(N, dtype=torch.uint8, device=dev)
    a.rgb = L.ptr(rgb); a.depth_pred = L.ptr(depth_pred); a.depth_gt = L.ptr(depth_gt); a.mask = L.ptr(mask)
    keep = [_f32c(g_rgb), _f32c(g_depth_pred), _f32c(g_depth_gt)]
    b.g_rgb, b.g_depth_pred, b.g_depth_gt = L.ptr(keep[0]), L.ptr(keep[1]), L.ptr(keep[2])
    b.g_weights = L.ptr(g_weights); b.g_c2w = L.ptr(g_c2w); b.g_cam = L.ptr(g_cam); b.g_depth = L.ptr(g_depth)
    b.g_scale_shift = L.ptr(g_scale_shift)
    nbytes = L.lib.nnb_render_frame_bwd_workspace_bytes_engine(N, S, int(hidden_dim), int(engine))
    ws = _pool.take(nbytes, dev) if nbytes else None
    a.workspace = L.ptr(ws); a.workspace_bytes = 0 if ws is None else ws.numel()
    try:
        L.check(L.lib.nnb_render_frame_bwd_engine(C.byref(b), _stream()), "nnb_render_frame_bwd_engine")
    finally:
        if ws is not None:
            _pool.give(ws)
    return rgb, depth_pred, depth_gt, mask


class _FrameGradFn(torch.autograd.Function):
    """render_frame_grad's autograd glue: the forward is render_frame_engine on meta's engine at t_min = 0 (RenderCall's bits without a
    stash), the backward render_frame_bwd on that engine, which evaluates the field again chunk by chunk.  Differentiable inputs as in
    _RenderFn."""

    @staticmethod
    def forward(ctx, meta, flat, c2w, cam, depth, scale, shift, *params):
        meta = dict(meta)
        ctx.param_slices = meta.pop("param_slices", None)
        det = lambda t: None if t is None else _f32c(t.detach())
        kw = dict(meta, depth=det(depth), scale=det(scale), shift=det(shift))
        ctx.kw = kw; ctx.inputs = (flat, det(c2w), det(cam))
        ctx.nparams = len(params)
        ctx.has = (depth is not None, scale is not None, shift is not None)
        ctx.params_need = any(p.requires_grad for p in params)
        rgb, dp, dg, mask = render_frame_engine(flat, ctx.inputs[1], ctx.inputs[2], t_min=0.0, **kw)
        ctx.mark_non_differentiable(mask)
        return rgb, dp, dg, mask

    @staticmethod
    def backward(ctx, g_rgb, g_dp, g_dg, _g_mask):
        kw = ctx.kw
        flat, c2w, cam = ctx.inputs
        dev = flat.device
        N = kw["N"]
        if g_rgb is None: g_rgb = torch.zeros(N, 3, device=dev)
        g_c2w = torch.zeros(4, 4, device=dev); g_cam = torch.zeros(4, 4, device=dev)
        g_w = torch.zeros(L.num_params(kw.get("hidden_dim", 256)), device=dev) if ctx.params_need else None
        has_depth, has_scale, has_shift = ctx.has
        g_depth = torch.empty(N, device=dev) if has_depth else None
        g_ss = torch.zeros(2, device=dev) if (has_scale or has_shift) else None
        render_frame_bwd(flat, c2w, cam, g_rgb, g_dp, g_dg, g_w, g_c2w, g_cam, g_depth, g_ss, **kw)
        gp = [None] * ctx.nparams
        if g_w is not None:
            slices = ctx.param_slices
            if slices is None:
                from .model.official_nerf import PARAM_SLICES as slices
            gp = [g_w[o:o + n].view(shape) for (o, n, shape) in slices]
        return (None, None, g_c2w, g_cam, g_depth, g_ss[0] if has_scale else None, g_ss[1] if has_shift else None) + tuple(gp)


def render_frame_grad(meta, flat, c2w, cam, depth, scale, shift, params, frame_engine=None):
    """render_autograd on the differentiable frame: (rgb, depth_pred, depth_gt, mask) of render_frame_engine (t_min = 0; the bits of
    RenderCall), with gradients to the MLP parameters, c2w, cam, depth and scale / shift from nnb_render_frame_bwd_engine, whose memory
    does not grow with S but by one float per ray and 32-sample chunk.  meta as render_autograd's without noise, want_z_alpha and stash
    (no jitter, no per-sample outputs).  frame_engine None (or ENGINE_TC): the tensor-core engine, to which meta's engine must resolve;
    ENGINE_SIMT: the exact-fp32 engine at any S from 2 to 1024, whatever meta's engine says."""
    meta = dict(meta)
    if meta.pop("noise", None) is not None or meta.pop("want_z_alpha", False) or meta.pop("stash", False):
        raise ValueError("render_frame_grad: noise, want_z_alpha and stash are not supported (no jitter, no per-sample outputs)")
    if frame_engine == L.ENGINE_SIMT:
        if not 2 <= meta["S"] <= 1024:
            raise ValueError("render_frame_grad on the exact engine needs 2 <= S <= 1024 (got %d)" % meta["S"])
        meta["engine"] = L.ENGINE_SIMT
    elif frame_engine is None or frame_engine == L.ENGINE_TC:
        if pick_engine(meta.get("engine"), meta["S"]) != L.ENGINE_TC:
            raise ValueError("render_frame_grad runs on the tensor-core engine only (16 <= S <= 1024)")
        meta["engine"] = L.ENGINE_TC   # render_frame_engine's forward and nnb_render_frame_bwd run this engine only
    else:
        raise ValueError("render_frame_grad: frame_engine must be None, ENGINE_TC or ENGINE_SIMT (got %r)" % (frame_engine,))
    return _FrameGradFn.apply(meta, flat, c2w, cam, depth, scale, shift, *params)


class _RenderFn(torch.autograd.Function):
    """autograd glue for the drop-in Renderer / nope_nerf modules.
    differentiable inputs: c2w (4,4), cam (4,4), depth (N,) | (scale, shift) and the 24 MLP parameters.
    meta['param_slices'] (optional): the model's (offset, numel, shape) list (OfficialStaticNerf.param_slices); meta['hidden_dim']
    its width (default 256)."""

    @staticmethod
    def forward(ctx, meta, flat, c2w, cam, depth, scale, shift, *params):
        # (grad mode is always off inside Function.forward: decide from the inputs' requires_grad)
        need_grad = any(ctx.needs_input_grad)
        meta = dict(meta)
        ctx.param_slices = meta.pop("param_slices", None)
        call = RenderCall(flat, _f32c(c2w.detach()), _f32c(cam.detach()), stash=need_grad,
                          depth=None if depth is None else _f32c(depth.detach()),
                          scale=None if scale is None else _f32c(scale.detach()),
                          shift=None if shift is None else _f32c(shift.detach()), **meta)
        ctx.call = call; ctx.nparams = len(params)
        ctx.has = (depth is not None, scale is not None, shift is not None)
        ctx.params_need = any(p.requires_grad for p in params)
        ctx.mark_non_differentiable(call.mask)
        outs = (call.rgb, call.depth_pred, call.depth_gt, call.mask)
        if call.z_vals is not None:
            ctx.mark_non_differentiable(call.z_vals, call.alpha)
            outs += (call.z_vals, call.alpha)
        return outs

    @staticmethod
    def backward(ctx, g_rgb, g_dp, g_dg, *unused):
        call = ctx.call
        dev = call.rgb.device
        if g_rgb is None: g_rgb = torch.zeros(call.N, 3, device=dev)
        g_c2w = torch.zeros(4, 4, device=dev); g_cam = torch.zeros(4, 4, device=dev)
        g_w = torch.zeros(L.num_params(call.hidden_dim), device=dev) if ctx.params_need else None
        has_depth, has_scale, has_shift = ctx.has
        g_depth = torch.empty(call.N, device=dev) if has_depth else None
        g_ss = torch.zeros(2, device=dev) if (has_scale or has_shift) else None
        call.backward(g_rgb, g_dp, g_dg, g_w, g_c2w, g_cam, g_depth, g_ss)
        gp = [None] * ctx.nparams
        if g_w is not None:
            slices = ctx.param_slices
            if slices is None:
                from .model.official_nerf import PARAM_SLICES as slices
            gp = [g_w[o:o + n].view(shape) for (o, n, shape) in slices]
        return (None, None, g_c2w, g_cam, g_depth, g_ss[0] if has_scale else None, g_ss[1] if has_shift else None) + tuple(gp)


def render_autograd(meta, flat, c2w, cam, depth, scale, shift, params):
    return _RenderFn.apply(meta, flat, c2w, cam, depth, scale, shift, *params)


class _PoseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, r, t, init, cam_id):
        c2w = torch.empty(4, 4, device=r.device)
        L.check(L.lib.nnb_pose_fwd(L.ptr(r), L.ptr(t), L.ptr(init), cam_id, L.ptr(c2w), _stream()), "nnb_pose_fwd")
        ctx.save_for_backward(r, t, init if init is not None else r.new_empty(0))
        ctx.cam_id = cam_id; ctx.has_init = init is not None
        return c2w

    @staticmethod
    def backward(ctx, g):
        r, t, init = ctx.saved_tensors
        g_r = torch.zeros_like(r) if ctx.needs_input_grad[0] else None
        g_t = torch.zeros_like(t) if ctx.needs_input_grad[1] else None
        L.check(L.lib.nnb_pose_bwd(L.ptr(r), L.ptr(t), L.ptr(init) if ctx.has_init else None, ctx.cam_id, L.ptr(_f32c(g)),
                                   L.ptr(g_r), L.ptr(g_t), _stream()), "nnb_pose_bwd")
        return g_r, g_t, None, None


def pose_c2w(r, t, init, cam_id):
    _need_cuda(r, "LearnPose.r")
    return _PoseFn.apply(r, t, init, int(cam_id))


def pose_fwd_raw(r, t, init, cam_id, out):
    L.check(L.lib.nnb_pose_fwd(L.ptr(r), L.ptr(t), L.ptr(init), int(cam_id), L.ptr(out), _stream()), "nnb_pose_fwd")


def pose_bwd_raw(r, t, init, cam_id, g_c2w, g_r, g_t):
    L.check(L.lib.nnb_pose_bwd(L.ptr(r), L.ptr(t), L.ptr(init), int(cam_id), L.ptr(g_c2w), L.ptr(g_r), L.ptr(g_t), _stream()),
            "nnb_pose_bwd")


def loss_rgb_depth(rgb, depth_pred, depth_gt, mask, w_rgb, w_depth, rgb_l2, *, rgb_gt=None, img=None, ray_idx=None,
                   grad_scale=1.0):
    """returns (losses[4] = loss, loss_rgb, loss_depth, l2_mean ; g_rgb, g_depth_pred, g_depth_gt)"""
    N = rgb.shape[0]; dev = rgb.device
    _need_cuda(img, "img", allow_pinned=True); _need_cuda(rgb_gt, "rgb_gt")
    out = torch.empty(4, device=dev)
    g_rgb = torch.empty(N, 3, device=dev); g_dp = torch.empty(N, device=dev); g_dg = torch.empty(N, device=dev)
    HW = 0 if img is None else (img.shape[-1] if img.dim() == 2 else img.shape[-1] * img.shape[-2])
    L.check(L.lib.nnb_loss_rgb_depth(L.ptr(rgb), L.ptr(rgb_gt), L.ptr(img), L.ptr(ray_idx), HW, L.ptr(depth_pred), L.ptr(depth_gt),
                                     L.ptr(mask), N, float(w_rgb), float(w_depth), int(bool(rgb_l2)), float(grad_scale), L.ptr(out),
                                     L.ptr(g_rgb), L.ptr(g_dp), L.ptr(g_dg), _stream()), "nnb_loss_rgb_depth")
    return out, g_rgb, g_dp, g_dg


class _ChamferFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, X, Y):
        X = _f32c(X); Y = _f32c(Y)
        P, Q = X.shape[0], Y.shape[0]
        need = X.requires_grad or Y.requires_grad
        if need:                                           # the adjoints' fixed-point group sums need more scratch than the search keys
            nbytes = L.lib.nnb_chamfer_workspace_bytes(P, Q)
            if nbytes == 0:
                raise RuntimeError("nnb_chamfer_workspace_bytes(%d, %d) failed" % (P, Q))
            keys = torch.empty((nbytes + 7) // 8, dtype=torch.int64, device=X.device)
        else:
            keys = torch.empty(P + Q, dtype=torch.int64, device=X.device)
        loss = torch.zeros(1, device=X.device)
        gX = torch.zeros_like(X) if need else None; gY = torch.zeros_like(Y) if need else None
        L.check(L.lib.nnb_chamfer(L.ptr(X), P, L.ptr(Y), Q, L.ptr(keys), None, None, L.ptr(loss), 1.0, L.ptr(gX), L.ptr(gY),
                                  _stream()), "nnb_chamfer")
        ctx.save_for_backward(gX if need else X.new_empty(0), gY if need else X.new_empty(0))
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        gX, gY = ctx.saved_tensors
        return (gX * g if ctx.needs_input_grad[0] else None), (gY * g if ctx.needs_input_grad[1] else None)


def chamfer(X, Y):
    """Loss.get_pc_loss (dense) for X (P,3), Y (Q,3) on the GPU."""
    _need_cuda(X, "X")
    return _ChamferFn.apply(X, Y)


_rs_ws = {}


def refstage_flags(scale_pcs=True, detach_rgbs_scale=False, shift_first=False, with_ssim=False, grad_ref=False):
    """nnb_refstage_args.flags"""
    return ((L.RS_SCALE_PCS if scale_pcs else 0) | (L.RS_DETACH_RGBS_SCALE if detach_rgbs_scale else 0) | (L.RS_SHIFT_FIRST if shift_first else 0) |
            (L.RS_WITH_SSIM if with_ssim else 0) | (L.RS_GRAD_REF if grad_ref else 0))


def refstage_raw(c2w_cur, dist_cur, c2w_ref, dist_ref, dpt_cur, dpt_ref, *, H, W, img_cur=None, img_ref=None, img_pp=None, is_last=False,
                 kx=0.0, ky=0.0, cam=None, cam_idx_dev=None, num_cams=0, weights_dev=None, nearest_limit=0.01, pc_ratio=4, scale_pcs=True,
                 detach_rgbs_scale=False, shift_first=False, w_pc=1.0, w_rgb_s=1.0, losses=None, g_c2w=None, g_dist=None, g_kxy=None,
                 loss_total=None, grad_scale=1.0, workspace=None, with_ssim=False, g_c2w_ref=None, g_dist_ref=None):
    """nnb_refstage: the reference-image stage of Trainer.compute_loss (model/training.py:280-365), forward + adjoint in one call.
    All tensor arguments are device tensors (frames may be page-locked host tensors); g_* / loss_total ACCUMULATE.
    with_ssim: warped-RGB loss 0.15 L1 + 0.85 SSIM (training.with_ssim).  g_c2w_ref (4,4) / g_dist_ref (2): also the gradients w.r.t. the
    reference view's pose matrix and effective distortion (training.detach_ref_img = False); both or neither."""
    _need_cuda(c2w_cur, "c2w_cur")
    for n_, t_ in (("img_cur", img_cur), ("img_ref", img_ref)):
        _need_cuda(t_, n_, allow_pinned=True)
    dev = c2w_cur.device
    hd, wd = int(dpt_cur.shape[-2]), int(dpt_cur.shape[-1])
    flags = refstage_flags(scale_pcs, detach_rgbs_scale, shift_first, with_ssim, g_c2w_ref is not None or g_dist_ref is not None)
    nbytes = L.lib.nnb_refstage_workspace_bytes_flags(hd, wd, int(pc_ratio), flags)
    if nbytes == 0:
        raise ValueError("reference-image stage: DPT map %dx%d too small for pc_ratio %d" % (hd, wd, pc_ratio))
    if workspace is None:
        key = (nbytes, dev.index)
        workspace = _rs_ws.get(key)
        if workspace is None:
            workspace = _rs_ws[key] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    if losses is None:
        losses = torch.zeros(2, device=dev)
    a = L.RefStageArgs()
    a.img_cur, a.img_ref, a.dpt_cur, a.dpt_ref = L.ptr(img_cur), L.ptr(img_ref), L.ptr(dpt_cur), L.ptr(dpt_ref)
    a.c2w_cur, a.c2w_ref, a.dist_cur, a.dist_ref = L.ptr(c2w_cur), L.ptr(c2w_ref), L.ptr(dist_cur), L.ptr(dist_ref)
    a.H, a.W, a.h_d, a.w_d, a.pc_ratio, a.is_last = int(H), int(W), hd, wd, int(pc_ratio), int(bool(is_last))
    a.flags = flags
    a.kx, a.ky, a.nearest_limit, a.w_pc, a.w_rgb_s = float(kx), float(ky), float(nearest_limit), float(w_pc), float(w_rgb_s)
    a.losses, a.g_c2w, a.g_dist = L.ptr(losses), L.ptr(g_c2w), L.ptr(g_dist)
    a.workspace, a.workspace_bytes = L.ptr(workspace), workspace.numel()
    a.img_pp, a.cam, a.cam_idx_dev, a.num_cams, a.weights_dev = L.ptr(img_pp), L.ptr(cam), L.ptr(cam_idx_dev), int(num_cams), L.ptr(weights_dev)
    a.g_kxy, a.loss_total, a.grad_scale = L.ptr(g_kxy), L.ptr(loss_total), float(grad_scale)
    a.g_c2w_ref, a.g_dist_ref = L.ptr(g_c2w_ref), L.ptr(g_dist_ref)
    L.check(L.lib.nnb_refstage(C.byref(a), _stream()), "nnb_refstage")
    return losses


class _RefStageFn(torch.autograd.Function):
    """w_pc * loss_pc + w_rgb_s * loss_rgb_s of the reference-image stage (model/training.py:280-365) as a function of the current
    view's pose matrix, effective distortion {scale, shift} and (kx, ky) and, when they require grad, the reference view's pose matrix
    and distortion (training.detach_ref_img = False); forward and adjoint come out of ONE library call."""

    @staticmethod
    def forward(ctx, c2w_cur, dist_cur, kxy, c2w_ref, dist_ref, img_cur, img_ref, dpt_cur, dpt_ref, is_last, nearest_limit, pc_ratio,
                scale_pcs, detach_rgbs_scale, shift_first, w_pc, w_rgb_s, with_ssim):
        dev = c2w_cur.device
        f = lambda t: _f32c(t.detach())
        H, W = img_cur.shape[-2:]
        g_c2w = torch.zeros(4, 4, device=dev); g_dist = torch.zeros(2, device=dev); g_kxy = torch.zeros(2, device=dev)
        grad_ref = ctx.needs_input_grad[3] or ctx.needs_input_grad[4]
        g_c2w_ref = torch.zeros(4, 4, device=dev) if grad_ref else None
        g_dist_ref = torch.zeros(2, device=dev) if grad_ref else None
        kx, ky = (float(v) for v in kxy.detach().cpu())
        flags = refstage_flags(scale_pcs, detach_rgbs_scale, shift_first, with_ssim, grad_ref)
        losses = refstage_raw(f(c2w_cur), f(dist_cur), f(c2w_ref), f(dist_ref), _f32c(dpt_cur), _f32c(dpt_ref), H=H, W=W, img_cur=_f32c(img_cur),
                              img_ref=_f32c(img_ref), is_last=is_last, kx=kx, ky=ky, nearest_limit=nearest_limit, pc_ratio=pc_ratio,
                              scale_pcs=scale_pcs, detach_rgbs_scale=detach_rgbs_scale, shift_first=shift_first, w_pc=w_pc, w_rgb_s=w_rgb_s,
                              g_c2w=g_c2w, g_dist=g_dist, g_kxy=g_kxy, with_ssim=with_ssim, g_c2w_ref=g_c2w_ref, g_dist_ref=g_dist_ref,
                              workspace=torch.empty(L.lib.nnb_refstage_workspace_bytes_flags(int(dpt_cur.shape[-2]), int(dpt_cur.shape[-1]),
                                                                                              int(pc_ratio), flags) or 1, dtype=torch.uint8, device=dev))
        if grad_ref:
            ctx.save_for_backward(g_c2w, g_dist, g_kxy, g_c2w_ref, g_dist_ref)
        else:
            ctx.save_for_backward(g_c2w, g_dist, g_kxy)
        ctx.mark_non_differentiable(losses)
        return float(w_pc) * losses[0] + float(w_rgb_s) * losses[1], losses

    @staticmethod
    def backward(ctx, g, _g_losses):
        saved = ctx.saved_tensors
        g_c2w, g_dist, g_kxy = saved[:3]
        g_c2w_ref, g_dist_ref = saved[3:] if len(saved) == 5 else (None, None)
        return (g_c2w * g if ctx.needs_input_grad[0] else None, g_dist * g if ctx.needs_input_grad[1] else None,
                g_kxy * g if ctx.needs_input_grad[2] else None, g_c2w_ref * g if ctx.needs_input_grad[3] else None,
                g_dist_ref * g if ctx.needs_input_grad[4] else None) + (None,) * 13


def refstage(c2w_cur, dist_cur, c2w_ref, dist_ref, img_cur, img_ref, dpt_cur, dpt_ref, is_last, kx, ky, nearest_limit=0.01, pc_ratio=4,
             scale_pcs=True, detach_rgbs_scale=False, shift_first=False, w_pc=1.0, w_rgb_s=1.0, with_ssim=False):
    """(total, losses[2] = {loss_pc, loss_rgb_s}); total is differentiable w.r.t. c2w_cur (4,4), dist_cur = [scale_eff, shift], when
    kx / ky are tensors the intrinsics, and when c2w_ref / dist_ref require grad the reference view's pose matrix and distortion
    (training.detach_ref_img = False).  with_ssim: warped-RGB loss 0.15 L1 + 0.85 SSIM (training.with_ssim).  Autograd wrapper over
    refstage_raw; the Trainer calls refstage_raw directly."""
    _need_cuda(c2w_cur, "c2w_cur")
    if isinstance(kx, torch.Tensor) or isinstance(ky, torch.Tensor):
        kxy = torch.stack([torch.as_tensor(kx, device=c2w_cur.device).reshape(()), torch.as_tensor(ky, device=c2w_cur.device).reshape(())])
    else:
        kxy = torch.tensor([float(kx), float(ky)], device=c2w_cur.device)
    return _RefStageFn.apply(c2w_cur, dist_cur, kxy, c2w_ref, dist_ref, img_cur, img_ref, dpt_cur, dpt_ref, is_last, nearest_limit, pc_ratio,
                             scale_pcs, detach_rgbs_scale, shift_first, w_pc, w_rgb_s, bool(with_ssim))


def adam_step(p, g, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    L.check(L.lib.nnb_adam_step(L.ptr(p), L.ptr(g), L.ptr(m), L.ptr(v), p.numel(), int(step), float(lr), beta1, beta2, eps,
                                _stream()), "nnb_adam_step")


# ---- CUDA-graph friendly variants (device-resident per-step scalars) -----------------------------------------
def pose_fwd_dev(r, t, init, cam_idx_dev, out):
    L.check(L.lib.nnb_pose_fwd_dev(L.ptr(r), L.ptr(t), L.ptr(init), L.ptr(cam_idx_dev), L.ptr(out), _stream()), "nnb_pose_fwd_dev")


def pose_bwd_dev(r, t, init, cam_idx_dev, g_c2w, g_r, g_t):
    L.check(L.lib.nnb_pose_bwd_dev(L.ptr(r), L.ptr(t), L.ptr(init), L.ptr(cam_idx_dev), L.ptr(g_c2w), L.ptr(g_r), L.ptr(g_t), _stream()),
            "nnb_pose_bwd_dev")


def distortion_fwd_dev(scales, shifts, cam_idx_dev, fix_last, out2):
    L.check(L.lib.nnb_distortion_fwd_dev(L.ptr(scales), L.ptr(shifts), scales.shape[0], L.ptr(cam_idx_dev), int(bool(fix_last)), L.ptr(out2),
                                         _stream()), "nnb_distortion_fwd_dev")


def distortion_bwd_dev(scales, cam_idx_dev, fix_last, g_ss, g_scales, g_shifts):
    L.check(L.lib.nnb_distortion_bwd_dev(L.ptr(scales), scales.shape[0], L.ptr(cam_idx_dev), int(bool(fix_last)), L.ptr(g_ss), L.ptr(g_scales),
                                         L.ptr(g_shifts), _stream()), "nnb_distortion_bwd_dev")


def adam_step_dev(p, g, m, v, step_dev, lr_dev, beta1=0.9, beta2=0.999, eps=1e-8):
    L.check(L.lib.nnb_adam_step_dev(L.ptr(p), L.ptr(g), L.ptr(m), L.ptr(v), p.numel(), L.ptr(step_dev), L.ptr(lr_dev), beta1, beta2, eps,
                                    _stream()), "nnb_adam_step_dev")


def counter_incr(counters):
    L.check(L.lib.nnb_counter_incr(L.ptr(counters), counters.numel(), _stream()), "nnb_counter_incr")


def loss_rgb_depth_indirect(rgb, depth_pred, depth_gt, mask, w_rgb, w_depth, rgb_l2, img_pp, ray_idx, HW, out, g_rgb, g_dp, g_dg, grad_scale=1.0,
                            w_dev=None):
    L.check(L.lib.nnb_loss_rgb_depth_indirect(L.ptr(rgb), L.ptr(img_pp), L.ptr(ray_idx), int(HW), L.ptr(depth_pred), L.ptr(depth_gt), L.ptr(mask),
                                              rgb.shape[0], float(w_rgb), float(w_depth), int(bool(rgb_l2)), float(grad_scale), L.ptr(out),
                                              L.ptr(g_rgb), L.ptr(g_dp), L.ptr(g_dg), L.ptr(w_dev), _stream()), "nnb_loss_rgb_depth_indirect")


def depth_invariant(depth_pred, depth_gt, mask, w_dev, out, g_dp, g_dg=None, grad_scale=1.0):
    """scale / shift invariant depth term (Loss.depth_loss_dpt over the masked rays) with weight w_dev[0]: out[2] = the term,
    out[0] += w * term, g_dp / g_dg (None: detached ground truth) += grad_scale * w * its seeds"""
    for n_, t_ in (("depth_pred", depth_pred), ("depth_gt", depth_gt), ("mask", mask), ("w_dev", w_dev), ("out", out), ("g_dp", g_dp)):
        _need_cuda(t_, n_)
    L.check(L.lib.nnb_depth_invariant(L.ptr(depth_pred), L.ptr(depth_gt), L.ptr(mask), int(depth_pred.shape[0]), L.ptr(w_dev), float(grad_scale),
                                      L.ptr(out), L.ptr(g_dp), L.ptr(g_dg), _stream()), "nnb_depth_invariant")


def focal_fwd(fx, fy, order, cam):
    """cam (4,4) = diag(fx', -fy', -1, 1) of LearnFocal (fy None: fx_only)"""
    _need_cuda(fx, "fx")
    L.check(L.lib.nnb_focal_fwd(L.ptr(fx), L.ptr(fy), int(order), L.ptr(cam), _stream()), "nnb_focal_fwd")


def focal_bwd(fx, fy, order, g_cam, g_kxy, g_fx, g_fy):
    """g_fx / g_fy += the focal parameters' gradient from the camera-matrix gradient g_cam (4,4) and g_kxy (2,) (or None)"""
    _need_cuda(fx, "fx")
    L.check(L.lib.nnb_focal_bwd(L.ptr(fx), L.ptr(fy), int(order), L.ptr(g_cam), L.ptr(g_kxy), L.ptr(g_fx), L.ptr(g_fy), _stream()), "nnb_focal_bwd")


def pose_smooth(t, w_dev, out2, loss_total=None, g_t=None, grad_scale=1.0):
    """pose-smoothness terms of the translations t (V,3) with weights w_dev[0:2]: out2 = {loss_dist_1st, loss_dist_2nd},
    loss_total += grad_scale * (w1 1st + w2 2nd), g_t += grad_scale * its gradient"""
    _need_cuda(t, "t")
    L.check(L.lib.nnb_pose_smooth(L.ptr(t), int(t.shape[0]), L.ptr(w_dev), float(grad_scale), L.ptr(out2), L.ptr(loss_total), L.ptr(g_t), _stream()),
            "nnb_pose_smooth")


def sample_pixels(hw, n, device):
    """n distinct pixel ids uniform in [0, hw) (distribution of torch.randperm(hw)[:n])"""
    u = torch.rand(2 * n, device=device)
    out = torch.empty(n, dtype=torch.int64, device=device)
    L.check(L.lib.nnb_sample_pixels(L.ptr(u), int(hw), int(n), L.ptr(out), _stream()), "nnb_sample_pixels")
    return out

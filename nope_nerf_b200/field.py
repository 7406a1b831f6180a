"""OfficialStaticNerf.forward on explicit points (reference: model/official_nerf.py:69-96) through nnb_field_fwd/bwd: used by direct
callers of the field module and the geometry view; the nope_nerf render path never materialises points.  The exact-fp32 engine
serves every call; a call that needs no gradient can ask for the tensor-core engine (field_query(engine='tc')), and a call that needs one
can stay there too (field_query_grad(engine='tc', grad_engine='tc'), whose backward is nnb_field_grad)."""
import ctypes as C
import torch
from . import _lib as L
from . import ops


class _FieldFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flags, net, flat, p, d, *params):
        M = p.shape[0]
        need = any(ctx.needs_input_grad)
        if need: flags |= L.STASH
        a = L.RenderArgs()
        p_c = ops._f32c(p.detach()); d_c = None if d is None else ops._f32c(d.detach())
        a.weights = L.ptr(flat); a.pts = L.ptr(p_c); a.dirs = L.ptr(d_c)
        a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_SIMT; a.hidden_dim = net.hidden_dim
        nbytes = L.lib.nnb_workspace_bytes_dim(M, 1, flags, L.ENGINE_SIMT, net.hidden_dim)
        ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=p.device)
        a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
        out = torch.empty(M, 4, device=p.device)
        L.check(L.lib.nnb_field_fwd(C.byref(a), L.ptr(out), ops._stream()), "nnb_field_fwd")
        ctx.args = a; ctx.keep = (ws, p_c, d_c, flat); ctx.M = M; ctx.nparams = len(params); ctx.has_d = d is not None
        ctx.slices = net.param_slices
        return out[:, :3], out[:, 3]

    @staticmethod
    def backward(ctx, g_rgb, g_a):
        M = ctx.M; dev = ctx.keep[0].device
        g = torch.zeros(M, 4, device=dev)
        if g_rgb is not None: g[:, :3] = g_rgb
        if g_a is not None: g[:, 3] = g_a
        g_p = torch.empty(M, 4, device=dev); g_d = torch.empty(M, 4, device=dev)
        need_w = any(ctx.needs_input_grad[5:])
        g_w = torch.zeros(ctx.keep[3].numel(), device=dev) if need_w else None
        L.check(L.lib.nnb_field_bwd(C.byref(ctx.args), L.ptr(g), L.ptr(g_p), L.ptr(g_d), L.ptr(g_w), ops._stream()), "nnb_field_bwd")
        gp = [None] * ctx.nparams
        if g_w is not None:
            gp = [g_w[o:o + n].view(s) for (o, n, s) in ctx.slices]
        return (None, None, None, g_p[:, :3], g_d[:, :3] if ctx.has_d else None) + tuple(gp)


def _field_flags(net):
    return (L.DIST_ALPHA if net.dist_alpha else 0) | (L.SOFTPLUS if net.occ_activation == 'softplus' else 0)


class _GradFn(torch.autograd.Function):
    """n = d s / d p of the density logit s (OfficialStaticNerf.gradient, official_nerf.py:46-58), differentiable once more.
    forward: nnb_field_fwd + nnb_field_bwd with cotangent 1 on the logit.  backward: nnb_field_hvp, which recomputes everything from the
    points and weights, so only p is kept."""

    @staticmethod
    def forward(ctx, net, flat, p, *params):
        M = p.shape[0]
        dev = p.device
        flags = _field_flags(net) | L.RAW_DENSITY | L.STASH
        a = L.RenderArgs()
        p_c = ops._f32c(p.detach())
        a.weights = L.ptr(flat); a.pts = L.ptr(p_c); a.dirs = None
        a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_SIMT; a.hidden_dim = net.hidden_dim
        nbytes = L.lib.nnb_workspace_bytes_dim(M, 1, flags, L.ENGINE_SIMT, net.hidden_dim)
        ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
        a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
        out = torch.empty(M, 4, device=dev)
        L.check(L.lib.nnb_field_fwd(C.byref(a), L.ptr(out), ops._stream()), "nnb_field_fwd")
        g = torch.zeros(M, 4, device=dev); g[:, 3] = 1.0
        g_p = torch.empty(M, 4, device=dev); g_d = torch.empty(M, 4, device=dev)
        L.check(L.lib.nnb_field_bwd(C.byref(a), L.ptr(g), L.ptr(g_p), L.ptr(g_d), None, ops._stream()), "nnb_field_bwd")
        ctx.net = net; ctx.flat = flat; ctx.nparams = len(params); ctx.slices = net.param_slices
        ctx.save_for_backward(p_c)
        return g_p[:, :3]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, u):
        p_c, = ctx.saved_tensors
        net, flat = ctx.net, ctx.flat
        need_p = ctx.needs_input_grad[2]
        need_w = any(ctx.needs_input_grad[3:])
        M = p_c.shape[0]; dev = p_c.device
        flags = _field_flags(net) | L.RAW_DENSITY | L.STASH | L.HVP
        u4 = torch.zeros(M, 4, device=dev); u4[:, :3] = u
        g_p = torch.empty(M, 4, device=dev) if need_p else None
        g_w = torch.zeros(flat.numel(), device=dev) if need_w else None
        if need_p or need_w:
            a = L.RenderArgs()
            a.weights = L.ptr(flat); a.pts = L.ptr(p_c); a.dirs = None
            a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_SIMT; a.hidden_dim = net.hidden_dim
            nbytes = L.lib.nnb_workspace_bytes_dim(M, 1, flags, L.ENGINE_SIMT, net.hidden_dim)
            ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
            a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
            L.check(L.lib.nnb_field_hvp(C.byref(a), L.ptr(u4), L.ptr(g_p), L.ptr(g_w), ops._stream()), "nnb_field_hvp")
        gp = [None] * ctx.nparams
        if g_w is not None:
            gp = [g_w[o:o + n].view(s) for (o, n, s) in ctx.slices]
        return (None, None, g_p[:, :3] if need_p else None) + tuple(gp)


def field_normal(net, p, engine=None, grad_engine=None):
    """n = d(density logit)/d p, shape (M, 3), for p (M, 3).  Differentiable with respect to p and the MLP parameters (the second-order
    backward is nnb_field_hvp); a third derivative raises.  M == 0 returns an empty tensor without a library call.
    engine: None or 'simt' = the exact-fp32 engine.  'tc' (or ENGINE_TC) = the tensor-core data gradient (nnb_field_vjp) when the call
    needs no autograd graph (the rule of field_query); a call that needs one runs on the exact engine, which has the second-order
    backward.  The tensor-core normals agree with float64 to 1.4e-5 of their maximum (the exact engine's to 5e-7), where both use the same
    ReLU gates; at a point whose pre-activation lies within rounding of 0 the engines may gate a unit differently, and the normal, which is
    discontinuous there, then differs by that unit's contribution.
    grad_engine: the engine of a call that needs the autograd graph (the rule of field_query_grad).  None or 'simt' = the exact engine (the
    rule above).  'tc' (or ENGINE_TC) needs engine='tc' (ValueError otherwise): the normals are then the bits of the detached
    tensor-core normals (nnb_field_vjp) and their backward is the tensor-core second-order backward nnb_field_hvp_tc, once differentiable,
    with gradients to p and the MLP parameters."""
    ops._need_cuda(p, "p")
    g_engine = None if grad_engine is None else _grad_engine_id(engine, grad_engine)
    if p.shape[0] == 0:
        return p * 0.0          # shape (0, 3), connected to p when p requires grad, so a backward over it gives zeros
    if _engine_id(engine) == L.ENGINE_TC:
        if not needs_grad(net, p):
            return _normal_tc(net, p)
        if g_engine == L.ENGINE_TC:
            return _GradTcFn.apply(net, net.flat_weights(), p, *list(net.parameters()))
    return _GradFn.apply(net, net.flat_weights(), p, *list(net.parameters()))


class _GradTcFn(torch.autograd.Function):
    """n = d s / d p of the density logit on the tensor-core engine under autograd (field_normal(engine='tc', grad_engine='tc')).
    forward: nnb_field_vjp with cotangent 1 on the logit (_normal_tc), so n is the detached gradient(engine='tc') normals' bits.  backward:
    nnb_field_hvp_tc, which recomputes everything from the points and weights, so only p is kept.  Differentiable once, like _GradFn."""

    @staticmethod
    def forward(ctx, net, flat, p, *params):
        p_c = ops._f32c(p.detach())
        n = _normal_tc(net, p_c)
        ctx.net = net; ctx.flat = flat; ctx.nparams = len(params); ctx.slices = net.param_slices
        ctx.save_for_backward(p_c)
        return n

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, u):
        p_c, = ctx.saved_tensors
        net, flat = ctx.net, ctx.flat
        need_p = ctx.needs_input_grad[2]
        need_w = any(ctx.needs_input_grad[3:])
        M, dev = p_c.shape[0], p_c.device
        u4 = torch.zeros(M, 4, device=dev); u4[:, :3] = u
        g_p = torch.empty(M, 4, device=dev) if need_p else None
        g_w = torch.zeros(flat.numel(), device=dev) if need_w else None
        if need_p or need_w:
            flags = L.RAW_DENSITY | L.OCC_ONLY
            a = L.RenderArgs()
            a.weights = L.ptr(flat); a.pts = L.ptr(p_c); a.dirs = None
            a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_TC; a.hidden_dim = net.hidden_dim
            ws = torch.empty(L.lib.nnb_field_hvp_tc_workspace_bytes(M, flags, net.hidden_dim), dtype=torch.uint8, device=dev)
            a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
            L.check(L.lib.nnb_field_hvp_tc(C.byref(a), L.ptr(u4), L.ptr(g_p), L.ptr(g_w), ops._stream()), "nnb_field_hvp_tc")
        gp = [None] * ctx.nparams
        if g_w is not None:
            gp = [g_w[o:o + n].view(s) for (o, n, s) in ctx.slices]
        return (None, None, g_p[:, :3] if need_p else None) + tuple(gp)


def _normal_tc(net, p):
    """nnb_field_vjp with the cotangent (0, 0, 0, 1) on the raw density logit, occupancy-only: d logit / d p (M, 3).  No autograd."""
    M, dev = p.shape[0], p.device
    flags = L.RAW_DENSITY | L.OCC_ONLY
    a = L.RenderArgs()
    flat = net.flat_weights()
    p_c = ops._f32c(p.detach())
    a.weights = L.ptr(flat); a.pts = L.ptr(p_c); a.dirs = None
    a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_TC; a.hidden_dim = net.hidden_dim
    g = torch.zeros(M, 4, device=dev); g[:, 3] = 1.0
    g_p = torch.empty(M, 4, device=dev)
    ws = torch.empty(L.lib.nnb_field_vjp_workspace_bytes(M, flags, net.hidden_dim), dtype=torch.uint8, device=dev)
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    L.check(L.lib.nnb_field_vjp(C.byref(a), L.ptr(g), None, L.ptr(g_p), None, ops._stream()), "nnb_field_vjp")
    return g_p[:, :3]


def _field_tc(net, flags, p, d):
    """nnb_field_fwd on the tensor-core engine: p (M, 3), d (M, 3) or None -> out (M, 4).  No autograd."""
    M = p.shape[0]
    a = L.RenderArgs()
    flat = net.flat_weights()
    p_c = ops._f32c(p.detach()); d_c = None if d is None else ops._f32c(d.detach())
    a.weights = L.ptr(flat); a.pts = L.ptr(p_c); a.dirs = L.ptr(d_c)
    a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_TC; a.hidden_dim = net.hidden_dim
    ws = torch.empty(L.lib.nnb_workspace_bytes_dim(M, 1, flags, L.ENGINE_TC, net.hidden_dim), dtype=torch.uint8, device=p.device)
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    out = torch.empty(M, 4, device=p.device)
    L.check(L.lib.nnb_field_fwd(C.byref(a), L.ptr(out), ops._stream()), "nnb_field_fwd")
    return out


class _FieldTcFn(torch.autograd.Function):
    """A field query on the tensor-core engine under autograd (field_query_grad(engine='tc', grad_engine='tc')).
    forward: nnb_field_fwd on tensor cores, so the outputs are the inference query's bits.  backward: nnb_field_grad, which recomputes the
    forward from the points, directions and weights (only they are kept) and returns the gradients to p, ray_d and every parameter, with
    NNB_OCC_ONLY when the caller uses the occupancy alone.  Differentiable once, like nnb_field_bwd's _FieldFn."""

    @staticmethod
    def forward(ctx, flags, net, flat, p, d, *params):
        p_c = ops._f32c(p.detach()); d_c = None if d is None else ops._f32c(d.detach())
        out = _field_tc(net, flags, p_c, d_c)
        ctx.flags = flags; ctx.net = net; ctx.flat = flat; ctx.nparams = len(params); ctx.slices = net.param_slices
        ctx.save_for_backward(p_c, d_c)
        return out[:, :3], out[:, 3]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_rgb, g_a):
        p_c, d_c = ctx.saved_tensors
        net, flat, flags = ctx.net, ctx.flat, ctx.flags
        M, dev = p_c.shape[0], p_c.device
        occ = bool(flags & L.OCC_ONLY)
        need_d = ctx.needs_input_grad[4] and not occ   # the occupancy does not depend on the view direction
        need_w = any(ctx.needs_input_grad[5:])
        g = torch.zeros(M, 4, device=dev)
        if g_rgb is not None and not occ: g[:, :3] = g_rgb
        if g_a is not None: g[:, 3] = g_a
        g_p = torch.empty(M, 4, device=dev)
        g_d = torch.empty(M, 4, device=dev) if need_d else None
        g_w = torch.zeros(flat.numel(), device=dev) if need_w else None
        a = L.RenderArgs()
        a.weights = L.ptr(flat); a.pts = L.ptr(p_c); a.dirs = L.ptr(d_c)
        a.N = M; a.S = 1; a.flags = flags; a.engine = L.ENGINE_TC; a.hidden_dim = net.hidden_dim
        ws = torch.empty(L.lib.nnb_field_grad_workspace_bytes(M, flags, net.hidden_dim), dtype=torch.uint8, device=dev)
        a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
        L.check(L.lib.nnb_field_grad(C.byref(a), L.ptr(g), None, L.ptr(g_p), L.ptr(g_d), L.ptr(g_w), ops._stream()), "nnb_field_grad")
        gp = [None] * ctx.nparams
        if g_w is not None:
            gp = [g_w[o:o + n].view(s) for (o, n, s) in ctx.slices]
        return (None, None, None, g_p[:, :3] if ctx.needs_input_grad[3] else None, g_d[:, :3] if need_d else None) + tuple(gp)


MARCH_BLOCK = 128   # steps one round of nnb_ray_march advances every ray that is still searching


def _march_engine_id(engine):
    """the engine of ray_march / geometry_frame: 'tc' (or ENGINE_TC) or 'simt' (or ENGINE_SIMT); anything else raises ValueError"""
    e = _engine_id(engine)
    if e is None:
        raise ValueError("engine must be 'simt', 'tc', ENGINE_SIMT or ENGINE_TC (got None)")
    return e


def ray_march(net, ray0, dirs, far, frac, near, n_secant, tau, want_bracket=False, engine='tc'):
    """nnb_ray_march_engine: Renderer.ray_marching + Renderer.secant for N rays in one call, without points or occupancies in global memory.
    ray0, dirs (N, 3); far (N,) per-ray far depth; frac (n_steps,) = torch.linspace(0, 1, n_steps); near, tau floats.  Returns depth (N,):
    the refined depth on a hit, 0 where the first sample is occupied, inf otherwise.  No autograd.
    engine: 'tc' (or ENGINE_TC, the default) = the tensor-core engine, bit-identical to the torch march over field_query(engine='tc',
    occ_only=True); 'simt' (or ENGINE_SIMT) = the exact-fp32 engine, bit-identical to the torch march over the default field_query.
    want_bracket: returns (depth, first (N,) int32, bracket (N, 4), counts) with first / bracket as nnb_ray_march documents them and
    counts (rounds + 1,) int32 = [rays that hit, rays that took part in round 1, 2, ...] (round 0 takes every ray)."""
    eng = _march_engine_id(engine)
    ops._need_cuda(ray0, "ray0")
    N, n_steps, dev = ray0.shape[0], frac.shape[0], ray0.device
    depth = torch.empty(N, device=dev)
    first = torch.empty(N, dtype=torch.int32, device=dev) if want_bracket else None
    bracket = torch.empty(N, 4, device=dev) if want_bracket else None
    rounds = (n_steps + MARCH_BLOCK - 1) // MARCH_BLOCK
    if N == 0:
        return (depth, first, bracket, torch.zeros(rounds + 1, dtype=torch.int32, device=dev)) if want_bracket else depth
    a = L.RayMarchArgs()
    keep = [net.flat_weights()] + [ops._f32c(t.detach()) for t in (ray0, dirs, far, frac)]
    a.weights, a.ray0, a.ray_dir, a.far_, a.frac = [L.ptr(t) for t in keep]
    a.N = N; a.n_steps = n_steps; a.n_secant = n_secant; a.hidden_dim = net.hidden_dim
    a.near_ = near; a.tau = tau; a.flags = _field_flags(net); a.engine = eng
    a.depth = L.ptr(depth); a.first = L.ptr(first); a.bracket = L.ptr(bracket)
    ws = ops._pool.take(L.lib.nnb_ray_march_workspace_bytes_engine(N, n_steps, net.hidden_dim, eng), dev)
    a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
    try:
        L.check(L.lib.nnb_ray_march_engine(C.byref(a), ops._stream()), "nnb_ray_march_engine")
        counts = ws[:4 * (rounds + 1)].view(torch.int32).clone() if want_bracket else None
    finally:
        ops._pool.give(ws)   # stream-ordered: the next call on this stream that takes it runs after this one
    return (depth, first, bracket, counts) if want_bracket else depth


def geometry_frame(net, T, pixels, frac, radius, n_secant=8, tau=0.5, near=0.0, want_intermediates=False, engine='tc'):
    """nnb_geometry_frame_engine: the geometry view (Renderer.phong_renderer) of N pixels in one call, with each pixel's camera ray computed on
    its own: ray setup, fused march (ray_march), normals (gradient()), shading and surface colour (field_query()), with no host round
    trip.  engine: 'tc' (or ENGINE_TC, the default) = every field query on the tensor-core engine (gradient(engine='tc'),
    field_query(engine='tc')); 'simt' (or ENGINE_SIMT) = every field query on the exact-fp32 engine, the default engine of gradient() and
    field_query().  T (4, 4) or (1, 4, 4) = S^-1 W^-1 K^-1; pixels (..., 2) image-plane
    coordinates (N = their count); frac (n_steps,) = torch.linspace(0, 1, n_steps); radius, tau, near floats.  Returns rgb, rgb_surf
    (N, 3): the shaded view (1 where no surface is hit) and the surface colour (0 there).  A pixel's outputs do not depend on the other
    pixels of the call.  No autograd.
    want_intermediates: also returns {'ray0', 'ray_dir' (N, 3), 'far', 'depth' (N,), 'grad' (N, 3)}: the call's rays, far sphere
    depths, march depths and -d logit / d p on the object rays (0 elsewhere)."""
    eng = _march_engine_id(engine)
    ops._need_cuda(pixels, "pixels")
    ops._need_cuda(T, "T")
    px = ops._f32c(pixels.detach().reshape(-1, 2))
    N, dev = px.shape[0], px.device
    rgb = torch.empty(N, 3, device=dev); surf = torch.empty(N, 3, device=dev)
    inter = None
    if want_intermediates:
        inter = dict(ray0=torch.empty(N, 3, device=dev), ray_dir=torch.empty(N, 3, device=dev), far=torch.empty(N, device=dev),
                     depth=torch.empty(N, device=dev), grad=torch.empty(N, 4, device=dev))
    if N > 0:
        a = L.GeometryArgs()
        keep = [net.flat_weights(), ops._f32c(T.detach().reshape(16)), px, ops._f32c(frac.detach())]
        a.weights, a.T, a.pixels, a.frac = [L.ptr(t) for t in keep]
        a.N = N; a.n_steps = frac.shape[0]; a.n_secant = n_secant; a.hidden_dim = net.hidden_dim
        a.near_ = near; a.tau = tau; a.radius = radius; a.flags = _field_flags(net); a.engine = eng
        a.rgb = L.ptr(rgb); a.rgb_surf = L.ptr(surf)
        if inter is not None:
            a.ray0, a.ray_dir, a.far_, a.depth, a.grad = [L.ptr(inter[k]) for k in ("ray0", "ray_dir", "far", "depth", "grad")]
        ws = ops._pool.take(L.lib.nnb_geometry_frame_workspace_bytes_engine(N, a.n_steps, net.hidden_dim, eng), dev)
        a.workspace = L.ptr(ws); a.workspace_bytes = ws.numel()
        try:
            L.check(L.lib.nnb_geometry_frame_engine(C.byref(a), ops._stream()), "nnb_geometry_frame_engine")
        finally:
            ops._pool.give(ws)   # stream-ordered, as in ray_march
    if inter is None:
        return rgb, surf
    inter["grad"] = inter["grad"][:, :3]
    return rgb, surf, inter


def needs_grad(net, *tensors):
    """whether a field call on these inputs has to be differentiable: grad mode is on and an input or a parameter of net requires grad"""
    return torch.is_grad_enabled() and (any(t is not None and t.requires_grad for t in tensors)
                                        or any(q.requires_grad for q in net.parameters()))


def _engine_id(engine):
    if engine is None or engine in (L.ENGINE_SIMT, L.ENGINE_TC):
        return engine
    try:
        return {"simt": L.ENGINE_SIMT, "tc": L.ENGINE_TC}[engine]
    except (KeyError, TypeError):
        raise ValueError("engine must be None, 'simt', 'tc', ENGINE_SIMT or ENGINE_TC (got %r)" % (engine,))


def _grad_engine_id(engine, grad_engine):
    """the engine of a call that needs a gradient: None (the exact engine, the default) or ENGINE_TC, which needs engine='tc'"""
    g = _engine_id(grad_engine)
    if g is None or g == L.ENGINE_SIMT:
        return None
    if _engine_id(engine) != L.ENGINE_TC:
        raise ValueError("grad_engine='tc' needs engine='tc' (got engine=%r): a query and its gradient on different engines would use "
                         "different ReLU gates" % (engine,))
    return g


def field_query(net, p, ray_d, raw_density=False, occ_only=False, engine=None):
    """field_query_grad with grad_engine=None: a call that needs a gradient runs on the exact engine (see there)"""
    return field_query_grad(net, p, ray_d, raw_density, occ_only, engine)


def field_query_grad(net, p, ray_d, raw_density=False, occ_only=False, engine=None, grad_engine=None):
    """returns (rgb (..,3), a (..,1)) with a = alpha (or sigma when rendering.dist_alpha), like return_addocc=True;
    raw_density: a = the density logit (OfficialStaticNerf.infer_occ, official_nerf.py:60-67).
    engine: None or 'simt' = the exact-fp32 engine.  'tc' (or ENGINE_TC) = the tensor-core engine when the call needs no gradient
    (grad mode off, or neither p, ray_d nor a parameter of net requires grad); a call that needs one runs on the exact engine, which
    has the backward.  The engines agree to about 1e-6 of the output's maximum, not bit for bit.
    grad_engine: the engine of a call that needs a gradient.  None or 'simt' = the exact engine (the rule above).  'tc' (or ENGINE_TC)
    needs engine='tc' (ValueError otherwise): the call then runs on tensor cores under autograd, its outputs the bits of the inference
    query and its backward nnb_field_grad, once differentiable, with gradients to p, ray_d and every parameter of net.
    occ_only: the caller uses a only.  On the tensor-core engine the colour branch is then skipped and rgb is zeros (a is bit-identical
    to the full query's), in the backward too; the exact engine evaluates everything regardless.
    No point (M == 0) returns empty tensors without a library call."""
    ops._need_cuda(p, "p")
    g_engine = None if grad_engine is None else _grad_engine_id(engine, grad_engine)
    shp = p.shape[:-1]
    flags = (L.DIST_ALPHA if net.dist_alpha else 0) | (L.SOFTPLUS if net.occ_activation == 'softplus' else 0) | (L.RAW_DENSITY if raw_density else 0)
    d = None if ray_d is None else ray_d.reshape(-1, 3)
    if p.numel() == 0:
        z = p.reshape(-1, 3)[:, :1] * 0.0      # stays connected to p, like an empty result of the library would
        return z.expand(-1, 3).reshape(*shp, 3), z.reshape(*shp, 1)
    if _engine_id(engine) == L.ENGINE_TC:
        if not needs_grad(net, p, d):
            out = _field_tc(net, flags | (L.OCC_ONLY if occ_only else 0), p.reshape(-1, 3), d)
            return out[:, :3].reshape(*shp, 3), out[:, 3].reshape(*shp, 1)
        if g_engine == L.ENGINE_TC:
            rgb, a = _FieldTcFn.apply(flags | (L.OCC_ONLY if occ_only else 0), net, net.flat_weights(), p.reshape(-1, 3), d,
                                      *list(net.parameters()))
            return rgb.reshape(*shp, 3), a.reshape(*shp, 1)
    rgb, a = _FieldFn.apply(flags, net, net.flat_weights(), p.reshape(-1, 3), d, *list(net.parameters()))
    return rgb.reshape(*shp, 3), a.reshape(*shp, 1)

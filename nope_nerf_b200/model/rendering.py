"""Renderer (reference: model/rendering.py:10-167).  forward() keeps the reference's
signature and output dict; the whole nope_nerf render (ray generation, sampling, encoding,
MLP, compositing) is one call into the CUDA library with autograd glue."""
import torch
import torch.nn as nn
from .. import ops
from .. import _lib as L
from ..field import ray_march, needs_grad, _engine_id, geometry_frame as field_geometry_frame

# Pixels per phong_renderer call of a whole-frame geometry view (Extract_Images.render_geometry, Trainer.render_visdata), on every
# engine: the reference's 1024.  The field queries do not depend on the chunk (every point's result is its own on the tensor-core
# engine), but the camera rays do: the batched matmul T @ ph of _rays_world rounds differently with the number of pixels in the call
# (measured on an H100: about 1 % of a 60 x 80 frame's pixels change between one call and 1024-pixel chunks), so a larger chunk would
# change the frame's bits.  Renderer(geometry_frame=True) computes the rays per pixel instead (phong_frame), and its callers pass the
# whole frame in one call.
GEOMETRY_CHUNK = 1024


def _frame_grad_engine(value, frame_grad, owner):
    """the frame_grad_engine keyword of Renderer / Trainer: None, 'tc' or 'simt', and only together with frame_grad=True"""
    if value not in (None, 'tc', 'simt'):
        raise ValueError("%s: frame_grad_engine must be None, 'tc' or 'simt' (got %r)" % (owner, value))
    if value is not None and not frame_grad:
        raise ValueError("%s: frame_grad_engine needs frame_grad=True" % owner)
    return value


class Renderer(nn.Module):
    def __init__(self, model, cfg, device=None, **kwargs):
        super().__init__()
        self._device = device
        self.depth_range = cfg['depth_range']
        self.n_max_network_queries = cfg['n_max_network_queries']   # accepted, unused: nothing is chunked
        self.white_background = cfg['white_background']
        self.cfg = cfg
        self.model = model.to(device)
        self.engine = kwargs.get("engine", None)
        # engine of the geometry view's explicit-point queries (ray marching, secant steps, surface colour): None = exact fp32,
        # 'tc' = tensor cores (OfficialStaticNerf.forward(engine=)); ray marching and the secant steps are then one fused call
        # (field.ray_march).
        self.field_engine = kwargs.get("field_engine", None)
        # engine of the geometry view's normals (OfficialStaticNerf.gradient(engine=)): None = exact fp32, 'tc' = the tensor-core data
        # gradient.  Separate from field_engine, so that a renderer built with field_engine='tc' keeps the bits it had.
        self.normal_engine = kwargs.get("normal_engine", None)
        # engine of the differentiable normals of rendering.normal_loss (_normal_diff): None = the exact engine whatever normal_engine
        # says; 'tc' (needs normal_engine='tc', ValueError otherwise) = the tensor-core normals with the tensor-core second-order backward
        # (OfficialStaticNerf.gradient_grad(engine='tc', grad_engine='tc')).
        self.normal_grad_engine = kwargs.get("normal_grad_engine", None)
        if self.normal_grad_engine is not None:
            from ..field import _grad_engine_id
            _grad_engine_id(self.normal_engine, self.normal_grad_engine)
        # geometry_frame=True: forward(..., 'phong_renderer') runs phong_frame (one tensor-core call for any number of pixels, rays
        # computed per pixel), and Extract_Images.render_geometry / Trainer.render_visdata pass the whole frame in one call.  Its
        # frames differ from phong_renderer's in the last bits of the rays, so it is off by default.
        self.geometry_frame = kwargs.get("geometry_frame", False)
        # engine of that frame (field.geometry_frame(engine=)): None or 'tc' = the tensor-core frame; 'simt' = the exact-fp32 frame, whose
        # march, normals and surface colour are the default engine's bits on the frame's own rays.
        self.geometry_frame_engine = kwargs.get("geometry_frame_engine", None)
        if self.geometry_frame_engine is not None:
            from ..field import _march_engine_id
            _march_engine_id(self.geometry_frame_engine)
        # fused_march=True: ray_marching on the exact engine (field_engine None or 'simt', no gradient needed, CUDA tensors) is one fused
        # call (field.ray_march(engine='simt')) instead of the torch march, with the same bits.  Off by default.
        self.fused_march = bool(kwargs.get("fused_march", False))
        # frame_t_min: None keeps Extract_Images.render_frame (and so generate_images / Eval_Images.eval_images) on nnb_render_fwd.  A
        # float t >= 0 renders those frames with ops.render_frame (nnb_render_frame: compositing fused into the tensor-core forward, a
        # workspace that does not grow with the sample count); t = 0 gives the same bits, t > 0 stops a ray once its transmittance is
        # below t (bounded error, see the header).  Tensor-core engine only: with the SIMT engine (an explicit engine, or fewer than 16
        # samples per ray) the frame takes the nnb_render_fwd path as before, unless frame_engine='simt' (below) is given too.
        # Trainer.render_visdata does not use it.
        t_min = kwargs.get("frame_t_min", None)
        if t_min is not None and not float(t_min) >= 0.0:
            raise ValueError("frame_t_min must be None or a float >= 0 (got %r)" % (t_min,))
        self.frame_t_min = None if t_min is None else float(t_min)
        # frame_engine: None keeps the routing above.  'simt' renders those frames with ops.render_frame_engine on the exact-fp32 engine
        # (nnb_render_frame_engine: the same fused frame, at any sample count from 2 to 1024; t = 0 gives nnb_render_fwd's exact-engine
        # bits) whatever `engine` says; it needs frame_t_min, without which it would do nothing.  'tc' is the default routing.
        frame_engine = kwargs.get("frame_engine", None)
        if frame_engine not in (None, 'tc', 'simt'):
            raise ValueError("frame_engine must be None, 'tc' or 'simt' (got %r)" % (frame_engine,))
        if frame_engine == 'simt' and self.frame_t_min is None:
            raise ValueError("frame_engine='simt' needs frame_t_min (a float >= 0)")
        self.frame_engine = frame_engine
        # frame_grad=True: training renders of nope_nerf (eval_=False) run on ops.render_frame_grad (nnb_render_frame_bwd: the same bits,
        # gradients from a backward whose memory does not grow with the sample count) instead of render_autograd.  Tensor-core engine
        # only, without jitter: such a render with add_noise on uniform sampling, or on the SIMT engine, is a ValueError.  Its output
        # dict has z_vals and alpha None (the frame keeps no per-sample values).  Off by default.
        self.frame_grad = bool(kwargs.get("frame_grad", False))
        # frame_grad_engine: None or 'tc' keeps those renders on the tensor-core engine; 'simt' runs them on the exact-fp32 engine
        # (nnb_render_frame_bwd_engine, any sample count from 2 to 1024, whatever `engine` says), still without jitter.  Needs frame_grad.
        self.frame_grad_engine = _frame_grad_engine(kwargs.get("frame_grad_engine", None), self.frame_grad, "Renderer")

    def to(self, device):
        model = super().to(device)
        model._device = device
        return model

    def forward(self, pixels, depth, camera_mat, world_mat, scale_mat, rendering_technique, add_noise=True, eval_=False,
                it=1000000):
        if rendering_technique == 'nope_nerf':
            return self.nope_nerf(pixels, depth, camera_mat, world_mat, scale_mat, it=it, add_noise=add_noise, eval_=eval_)
        if rendering_technique == 'phong_renderer':
            if self.geometry_frame:
                return self.phong_frame(pixels, camera_mat, world_mat, scale_mat, it)
            return self.phong_renderer(pixels, camera_mat, world_mat, scale_mat, it)
        raise ValueError(rendering_technique)

    def render_meta(self, N, eval_, extra=None):
        cfg = self.cfg
        ndc = cfg['sample_option'] == 'ndc'
        meta = dict(N=N, S=int(cfg['num_points']), near=0.0 if ndc else float(self.depth_range[0]),
                    far=1.0 if ndc else float(self.depth_range[1]),
                    flags=ops.flags_from_cfg(cfg, self.model.occ_activation, eval_=eval_),
                    engine=self.engine if self.engine is not None else ops.default_engine(),
                    hidden_dim=getattr(self.model, 'hidden_dim', 256))
        if extra: meta.update(extra)
        return meta

    def nope_nerf(self, pixels, depth, camera_mat, world_mat, scale_mat, add_noise=False, it=100000, eval_=False,
                  c2w=None, normal_noise=None):
        """rendering.py:36-167.  camera_mat must be diag(kx,ky,-1,1) and scale_mat identity (the only
        forms the reference constructs: dataset.py:101-104,199; training.py:247-252).
        With rendering.normal_loss and not eval_, out['normal'] is the reference's diff_norm (rendering.py:133-141): |n(x) - n(x')| of
        the unit normals at each valid ray's surface point x and a jittered neighbour x' = x + 0.01 (U - 0.5), differentiable with
        respect to the MLP, the pose, the camera matrix and the prior depth.  normal_noise (valid rays, 3) replaces the draw U."""
        batch_size, n_points, _ = pixels.shape
        if batch_size != 1:
            raise NotImplementedError("batch_size must be 1 (configs/default.yaml:14)")
        if scale_mat is not None and not scale_mat.is_cuda:
            if not torch.equal(scale_mat.reshape(-1, 4, 4)[0], torch.eye(4)):
                raise NotImplementedError("scale_mat must be the identity")
        if c2w is None:
            c2w = torch.linalg.inv(world_mat.reshape(4, 4))       # common.py:139-141 (invert=True)
        cam = camera_mat.reshape(4, 4)
        S = int(self.cfg['num_points'])
        noise = None
        if add_noise and self.cfg['sample_option'] == 'uniform':
            noise = torch.rand(batch_size, n_points, S, device=pixels.device)[0]     # rendering.py:189
        meta = self.render_meta(n_points, eval_, dict(pixels=pixels.reshape(n_points, 2).contiguous().float(), noise=noise,
                                                      want_z_alpha=True, param_slices=getattr(self.model, 'param_slices', None)))
        flat = self.model.flat_weights()
        d = depth.reshape(n_points)
        if self.frame_grad and not eval_:
            if noise is not None:
                raise ValueError("Renderer(frame_grad=True) renders without jitter: call with add_noise=False or use ndc sampling")
            meta.update(want_z_alpha=False, noise=None)
            rgb, dp, dg, mask = ops.render_frame_grad(meta, flat, c2w, cam, d, None, None, list(self.model.parameters()),
                                                      frame_engine=L.ENGINE_SIMT if self.frame_grad_engine == 'simt' else None)
            z = alpha = None
        else:
            rgb, dp, dg, mask, z, alpha = ops.render_autograd(meta, flat, c2w, cam, d, None, None, list(self.model.parameters()))
        m = mask.bool()
        diff_norm = None
        if self.cfg.get('normal_loss', False) and not eval_:
            diff_norm = self._normal_diff(pixels.reshape(n_points, 2), d, c2w, cam, m, it, normal_noise)
        return {'rgb': rgb.reshape(1, n_points, 3), 'z_vals': z, 'normal': diff_norm,
                'depth_pred': dp[m], 'depth_gt': dg[m], 'alpha': alpha}

    def _normal_diff(self, pix, depth, c2w, cam, m, it, noise=None):
        """rendering.py:53-94,133-141 on the valid-prior rays m: surface point camera_world + ray_vector * dists, in torch from the same
        c2w / camera matrix / depth as the render call so that gradients reach the pose, the focal and the distortion"""
        kx, ky = cam[0, 0], cam[1, 1]
        R, t = c2w[:3, :3], c2w[:3, 3]
        x, y = pix[m, 0], pix[m, 1]
        dc = torch.stack([x / kx, y / ky, -torch.ones_like(x)], dim=-1)        # K^-1 (x, y, 1): camera-space direction at depth 1
        dt = dc @ R.t()                                                         # pixels_world - camera_world
        d_i = (depth[m].unsqueeze(-1) * dt).norm(2, dim=-1)                     # |points_world - camera_world|
        nrm = dt.norm(2, dim=-1)
        if self.cfg['normalise_ray']:
            points = t + (dt / nrm.unsqueeze(-1)) * d_i.unsqueeze(-1)
        else:
            points = t + dt * (d_i / nrm).unsqueeze(-1)
        N = points.shape[0]
        if N == 0:
            return points.sum(-1) * 0.0          # shape (0,), still connected to whatever the points depend on; no library call
        if noise is None:
            noise = torch.rand_like(points)
        neig = points + (noise - 0.5) * 0.01
        pp = torch.cat([points, neig], dim=0)
        if torch.is_grad_enabled() and not pp.requires_grad:
            # fixed pose, camera and depth: like the reference (official_nerf.py:48, p.requires_grad_(True) inside gradient()), the
            # points this renderer owns become a leaf that requires grad, so the normal term still reaches the MLP
            pp.requires_grad_(True)
        if self.normal_grad_engine is None:
            g = self.model.gradient(pp, it)[:, 0, :]
        else:
            g = self.model.gradient_grad(pp, it, engine=self.normal_engine, grad_engine=self.normal_grad_engine)[:, 0, :]
        normals = g / (g.norm(2, dim=1).unsqueeze(-1) + 10 ** (-5))
        return torch.norm(normals[:N] - normals[N:], dim=-1)

    # ---- geometry visualiser (SURVEY.md 8(f) rank 4; reference rendering.py:198-418): evaluation-time only (render_visdata every
    #      `visualize_every` iterations).  Host logic mirrors the reference; every field evaluation (occupancy along the rays, secant
    #      refinement, normals = gradient(), surface colour) is a call into the CUDA library (nnb_field_fwd / nnb_field_bwd). ----
    @staticmethod
    def _ray_transform(camera_mat, world_mat, scale_mat, dev):
        """T = S^-1 W^-1 K^-1: image plane (x, y, 1, 1) -> world (common.py:186-237, invert=True)"""
        Ki = torch.inverse(camera_mat.to(dev)); Wi = torch.inverse(world_mat.to(dev)); Si = torch.inverse(scale_mat.to(dev))
        return Si @ Wi @ Ki

    @staticmethod
    def _rays_world(pixels, camera_mat, world_mat, scale_mat):
        """image_points_to_world / origin_to_world (common.py:186-237, invert=True): ray origins and unit directions"""
        b, n, _ = pixels.shape
        dev = pixels.device
        T = Renderer._ray_transform(camera_mat, world_mat, scale_mat, dev)
        ph = torch.cat([pixels.permute(0, 2, 1), torch.ones(b, 2, n, device=dev)], dim=1)          # depth 1: (x, y, 1, 1)
        pw = (T @ ph)[:, :3].permute(0, 2, 1)
        o = torch.zeros(b, 4, n, device=dev); o[:, -1] = 1.
        cw = (T @ o)[:, :3].permute(0, 2, 1)
        d = pw - cw
        return cw, d / d.norm(2, 2).unsqueeze(-1)

    @staticmethod
    def _sphere_far(cam_loc, dirs, r):
        """far intersection depth of the rays with the sphere |x| = r (rendering.py:439-460), 0 where the ray misses"""
        dot = torch.bmm(dirs, cam_loc.unsqueeze(-1)).reshape(-1)
        under = dot ** 2 - (cam_loc.norm(2, 1) ** 2 - r ** 2).reshape(-1, 1).expand(-1, dirs.shape[1]).reshape(-1)
        far = torch.zeros_like(dot)
        m = under > 0
        far[m] = torch.sqrt(under[m]) - dot[m]
        return far.clamp_min(0.0).reshape(dirs.shape[0], dirs.shape[1])

    def phong_renderer(self, pixels, camera_mat, world_mat, scale_mat, it):
        batch_size, num_pixels, _ = pixels.shape
        dev = pixels.device
        rad = self.cfg['radius']
        camera_world, ray_vector = self._rays_world(pixels, camera_mat, world_mat, scale_mat)
        light_source = camera_world[0, 0]
        light = (light_source / light_source.norm(2)).unsqueeze(1)
        diffuse_per = torch.tensor([0.7, 0.7, 0.7], device=dev); ambiant = torch.tensor([0.3, 0.3, 0.3], device=dev)
        self.model.eval()
        with torch.no_grad():
            d_i = self.ray_marching(camera_world, ray_vector, self.model, n_secant_steps=8, n_steps=[512, 513], rad=rad)
            mask_zero_occupied = d_i == 0
            mask_pred = torch.isfinite(d_i)                                # common.get_mask
            dists = torch.ones_like(d_i)
            dists[mask_pred] = d_i[mask_pred]
            dists[mask_zero_occupied] = 0.
            network_object_mask = (mask_pred & ~mask_zero_occupied)[0]
            dists = dists[0]
            cw = camera_world.reshape(-1, 3); rv = ray_vector.reshape(-1, 3)
            points = cw + rv * dists.unsqueeze(-1)
            view_vol = -rv
            rgb_values = torch.ones_like(points)
            surface_points = points[network_object_mask]
            surface_view_vol = view_vol[network_object_mask]
        rgb_val = torch.zeros(batch_size * num_pixels, 3, device=dev)
        if surface_points.shape[0] > 0:
            grad = self.model.gradient(surface_points, it, engine=self.normal_engine)[:, 0, :].detach()
            surface_normals = grad / grad.norm(2, 1, keepdim=True)
            diffuse = torch.mm(surface_normals, light).clamp_min(0).repeat(1, 3) * diffuse_per.unsqueeze(0)
            rgb_values[network_object_mask] = (ambiant.unsqueeze(0) + diffuse).clamp_max(1.0)
            with torch.no_grad():
                rgb_val[network_object_mask] = self.model(surface_points, surface_view_vol, engine=self.field_engine)
        return {'rgb': rgb_values.reshape(batch_size, -1, 3), 'normal': None, 'rgb_surf': rgb_val.reshape(batch_size, -1, 3)}

    def phong_frame(self, pixels, camera_mat, world_mat, scale_mat, it):
        """phong_renderer's view and output dict in one call for any number of pixels (field.geometry_frame), on the tensor-core engine,
        or on the exact engine with geometry_frame_engine='simt'.  Each pixel's camera ray is computed on its own, so a pixel's result does not depend on how the frame is split
        into calls; it differs from phong_renderer's, whose rays come from a batched matmul over the call's pixels, in the last bits of
        the rays.  Draws the single torch.randint that ray_marching draws (n_steps = 512), so a call consumes the same random numbers."""
        batch_size, num_pixels, _ = pixels.shape
        if batch_size != 1:
            raise NotImplementedError("batch_size must be 1 (configs/default.yaml:14)")
        ops._need_cuda(pixels, "pixels")
        dev = pixels.device
        T = self._ray_transform(camera_mat, world_mat, scale_mat, dev)
        n_steps = int(torch.randint(512, 513, (1,)).item())
        frac = torch.linspace(0, 1, steps=n_steps, device=dev)
        self.model.eval()
        engine = 'tc' if self.geometry_frame_engine is None else self.geometry_frame_engine
        with torch.no_grad():
            rgb, rgb_surf = field_geometry_frame(self.model, T, pixels, frac, float(self.cfg['radius']), n_secant=8, tau=0.5, near=0.0,
                                                 engine=engine)
        return {'rgb': rgb.reshape(batch_size, -1, 3), 'normal': None, 'rgb_surf': rgb_surf.reshape(batch_size, -1, 3)}

    def ray_marching(self, ray0, ray_direction, model, c=None, tau=0.5, n_steps=[128, 129], n_secant_steps=8, depth_range=[0., 2.4],
                     max_points=3500000, rad=1.0):
        """rendering.py:274-384: first sign change of (occupancy - tau) along each ray, refined by the secant method.  With
        field_engine='tc' and no gradient needed (the rule of field.field_query) the march and the secant steps are one fused call into
        the library; it returns the bits the torch march below returns on that engine.  So does fused_march=True on the exact engine."""
        batch_size, n_pts, _ = ray0.shape
        dev = ray0.device
        tau = 0.5
        n_steps = int(torch.randint(n_steps[0], n_steps[1], (1,)).item())
        if _engine_id(self.field_engine) == L.ENGINE_TC and not needs_grad(model, ray0, ray_direction) and ray0.is_cuda:
            d_intersect = self._sphere_far(ray0[:, 0], ray_direction, rad)
            frac = torch.linspace(0, 1, steps=n_steps, device=dev)
            return ray_march(model, ray0.reshape(-1, 3), ray_direction.reshape(-1, 3), d_intersect.reshape(-1), frac,
                             float(depth_range[0]), n_secant_steps, tau).view(batch_size, n_pts)
        if (self.fused_march and _engine_id(self.field_engine) in (None, L.ENGINE_SIMT) and not needs_grad(model, ray0, ray_direction)
                and ray0.is_cuda):
            d_intersect = self._sphere_far(ray0[:, 0], ray_direction, rad)
            frac = torch.linspace(0, 1, steps=n_steps, device=dev)
            return ray_march(model, ray0.reshape(-1, 3), ray_direction.reshape(-1, 3), d_intersect.reshape(-1), frac,
                             float(depth_range[0]), n_secant_steps, tau, engine='simt').view(batch_size, n_pts)
        return self._ray_marching_torch(ray0, ray_direction, model, n_steps, n_secant_steps, depth_range, max_points, rad,
                                        self.field_engine)

    def _ray_marching_torch(self, ray0, ray_direction, model, n_steps, n_secant_steps, depth_range, max_points, rad, engine):
        """the march in torch over explicit-point field queries on `engine`: the exact engine's path, and the reference the fused
        march is checked against"""
        batch_size, n_pts, _ = ray0.shape
        dev = ray0.device
        tau = 0.5
        d_intersect = self._sphere_far(ray0[:, 0], ray_direction, rad)
        d_proposal = torch.linspace(0, 1, steps=n_steps, device=dev).view(1, 1, n_steps, 1)
        d_proposal = depth_range[0] * (1. - d_proposal) + d_intersect.view(1, -1, 1, 1) * d_proposal
        p_proposal = ray0.unsqueeze(2) + ray_direction.unsqueeze(2) * d_proposal
        with torch.no_grad():
            val = torch.cat([model(p_split, only_occupancy=True, engine=engine) - tau
                             for p_split in torch.split(p_proposal.reshape(batch_size, -1, 3), int(max_points / batch_size), dim=1)],
                            dim=1).view(batch_size, -1, n_steps)
        mask_0_not_occupied = val[:, :, 0] < 0
        sign_matrix = torch.cat([torch.sign(val[:, :, :-1] * val[:, :, 1:]), torch.ones(batch_size, n_pts, 1, device=dev)], dim=-1)
        cost_matrix = sign_matrix * torch.arange(n_steps, 0, -1, device=dev).float()
        values, indices = torch.min(cost_matrix, -1)
        mask_sign_change = values < 0
        bi = torch.arange(batch_size, device=dev).unsqueeze(-1); pi = torch.arange(n_pts, device=dev).unsqueeze(0)
        mask_neg_to_pos = val[bi, pi, indices] < 0
        mask = mask_sign_change & mask_neg_to_pos & mask_0_not_occupied
        n = batch_size * n_pts
        ar = torch.arange(n, device=dev)
        dp = d_proposal.expand(batch_size, n_pts, n_steps, 1).reshape(n, n_steps)
        vv = val.reshape(n, n_steps)
        d_low = dp[ar, indices.view(n)].view(batch_size, n_pts)[mask]
        f_low = vv[ar, indices.view(n)].view(batch_size, n_pts)[mask]
        indices = torch.clamp(indices + 1, max=n_steps - 1)
        d_high = dp[ar, indices.view(n)].view(batch_size, n_pts)[mask]
        f_high = vv[ar, indices.view(n)].view(batch_size, n_pts)[mask]
        ray0_masked = ray0[mask]; ray_direction_masked = ray_direction[mask]
        d_pred_out = torch.ones(batch_size, n_pts, device=dev)
        if ray0_masked.shape[0] != 0:
            d_pred_out[mask] = self._secant(f_low, f_high, d_low, d_high, n_secant_steps, ray0_masked, ray_direction_masked, tau, 0,
                                            engine)
        d_pred_out[mask == 0] = float('inf')
        d_pred_out[mask_0_not_occupied == 0] = 0
        return d_pred_out

    def secant(self, f_low, f_high, d_low, d_high, n_secant_steps, ray0_masked, ray_direction_masked, tau, it=0):
        """rendering.py:386-418"""
        return self._secant(f_low, f_high, d_low, d_high, n_secant_steps, ray0_masked, ray_direction_masked, tau, it, self.field_engine)

    def _secant(self, f_low, f_high, d_low, d_high, n_secant_steps, ray0_masked, ray_direction_masked, tau, it, engine):
        d_pred = -f_low * (d_high - d_low) / (f_high - f_low) + d_low
        for _ in range(n_secant_steps):
            p_mid = ray0_masked + d_pred.unsqueeze(-1) * ray_direction_masked
            with torch.no_grad():
                f_mid = self.model(p_mid, batchwise=False, only_occupancy=True, it=it, engine=engine)[..., 0] - tau
            ind_low = f_mid < 0
            d_low = torch.where(ind_low, d_pred, d_low); f_low = torch.where(ind_low, f_mid, f_low)
            d_high = torch.where(ind_low, d_high, d_pred); f_high = torch.where(ind_low, f_high, f_mid)
            d_pred = -f_low * (d_high - d_low) / (f_high - f_low) + d_low
        return d_pred

"""Extract_Images (reference: model/extracting_images.py:13-124): full-frame novel-view rendering, the caller of
BASELINE config 4.  The reference splits a frame into 100 000-ray chunks x 64 000-sample MLP chunks (~4 200 Python-loop
iterations per 1080p frame); here one frame (or one row block of it, for ray-sharded multi-GPU rendering) is ONE library
call — the persistent tensor-core kernel walks all 128-sample tiles itself.  File output is plain numpy / PIL."""
import os
import numpy as np
import torch
from .. import ops
from .. import _lib as L


class Extract_Images(object):
    def __init__(self, renderer, cfg, use_learnt_poses=True, use_learnt_focal=True, device=None, render_type=None):
        self.points_batch_size = 100000          # kept for API compatibility; nothing is chunked
        self.renderer = renderer
        self.resolution = cfg['extract_images']['resolution']
        self.device = device
        self.use_learnt_poses = use_learnt_poses
        self.use_learnt_focal = use_learnt_focal
        self.render_type = render_type

    def render_frame(self, c2w, camera_mat, h, w, rows=None):
        """rgb (rows,w,3) and z-depth (rows,w) of one view; eval mode, no jitter, prior depth = 1
        (extracting_images.py:52-77).  rows=(r0,r1) renders a row block (multi-GPU sharding of one frame).  With
        Renderer(frame_t_min=t) on the tensor-core engine the frame is one ops.render_frame call (nnb_render_frame) instead, and with
        Renderer(frame_t_min=t, frame_engine='simt') one ops.render_frame_engine call on the exact-fp32 engine at any engine and S."""
        rend = self.renderer
        net = rend.model
        r0, r1 = (0, h) if rows is None else rows
        dev = self.device
        ray_idx = torch.arange(r0 * w, r1 * w, device=dev, dtype=torch.int64)
        n = ray_idx.numel()
        ndc = rend.cfg['sample_option'] == 'ndc'
        S = int(rend.cfg['num_points'])
        engine = rend.engine if rend.engine is not None else ops.default_engine()
        args = (net.flat_weights(), c2w.detach().reshape(4, 4).contiguous().float(), camera_mat.detach().reshape(4, 4).contiguous().float())
        kw = dict(N=n, S=S, flags=ops.flags_from_cfg(rend.cfg, net.occ_activation, eval_=True), engine=engine,
                  near=0.0 if ndc else rend.depth_range[0], far=1.0 if ndc else rend.depth_range[1],
                  ray_idx=ray_idx, depth_map=torch.ones(1, 1, device=dev), H=h, W=w, stash=False, hidden_dim=net.hidden_dim)
        t_min = getattr(rend, 'frame_t_min', None)
        if t_min is not None and getattr(rend, 'frame_engine', None) == 'simt':   # Renderer(frame_engine='simt'): the exact frame
            rgb, depth_pred = ops.render_frame_engine(*args, t_min=t_min, **dict(kw, engine=L.ENGINE_SIMT))[:2]
            return rgb.view(r1 - r0, w, 3), depth_pred.view(r1 - r0, w)
        if t_min is not None and ops.pick_engine(engine, S) == L.ENGINE_TC:   # Renderer(frame_t_min=t): the fused frame renderer
            rgb, depth_pred = ops.render_frame(*args, t_min=t_min, **kw)[:2]
            return rgb.view(r1 - r0, w, 3), depth_pred.view(r1 - r0, w)
        call = ops.RenderCall(*args, **kw)
        return call.rgb.view(r1 - r0, w, 3), call.depth_pred.view(r1 - r0, w)

    def render_geometry(self, c2w, camera_mat, scale_mat, h, w, it=0):
        """phong-shaded surface view (extracting_images.py:80-97): Renderer.forward(..., 'phong_renderer') over chunks of
        rendering.GEOMETRY_CHUNK pixels of the frame, or in one call with Renderer(geometry_frame=True), (h,w,3) uint8 -- the same
        call sequence as the geometry view of Trainer.render_visdata"""
        from .rendering import GEOMETRY_CHUNK
        from .common import arange_pixels
        dev = self.device
        _, pixels = arange_pixels(resolution=(h, w), device=dev)
        world_mat = torch.linalg.inv(c2w.detach().reshape(4, 4).float()).unsqueeze(0)
        cam = camera_mat.detach().reshape(1, 4, 4).float()
        chunk = pixels.shape[1] if getattr(self.renderer, 'geometry_frame', False) else GEOMETRY_CHUNK
        with torch.no_grad():
            rgb = torch.cat([self.renderer(px, None, cam, world_mat, scale_mat, 'phong_renderer', eval_=True, it=it, add_noise=False)['rgb']
                             for px in torch.split(pixels, chunk, dim=1)], dim=1)
        return (rgb.reshape(h, w, 3).cpu().numpy() * 255).astype(np.uint8)

    def generate_images(self, data, render_dir, c2ws, fxfy, it, output_geo):
        self.renderer.eval()
        device = self.device
        camera_mat = data.get('img.camera_mat').to(device)
        img_idx = int(data.get('img.idx'))
        c2w = c2ws[img_idx] if self.use_learnt_poses else torch.eye(4, device=device)
        if self.use_learnt_focal:
            camera_mat = torch.diag(torch.stack([fxfy[0], -fxfy[1], -torch.ones((), device=device), torch.ones((), device=device)]))
        h, w = self.resolution
        with torch.no_grad():
            rgb, depth = self.render_frame(c2w, camera_mat, h, w)
            rgb_pred = rgb.cpu().numpy(); depth_out = depth.cpu().numpy()
        img_out = (rgb_pred * 255).astype(np.uint8)
        if render_dir is not None:
            from PIL import Image
            img_dir = os.path.join(render_dir, 'img_out'); dep_dir = os.path.join(render_dir, 'depth_out')
            os.makedirs(img_dir, exist_ok=True); os.makedirs(dep_dir, exist_ok=True)
            np.save(os.path.join(dep_dir, '{}.npy'.format(img_idx)), depth_out)
            d8 = (np.clip(255.0 / depth_out.max() * (depth_out - depth_out.min()), 0, 255)).astype(np.uint8)
            Image.fromarray(img_out).save(os.path.join(img_dir, str(img_idx).zfill(4) + '.png'))
            Image.fromarray(d8).save(os.path.join(dep_dir, str(img_idx).zfill(4) + '.png'))
            depth_out = d8
        geo_out = None
        if output_geo:
            scale_mat = data.get('img.scale_mat')
            geo_out = self.render_geometry(c2w, camera_mat, scale_mat.to(device) if scale_mat is not None else None, h, w, it=it)
            if render_dir is not None:
                from PIL import Image
                geo_dir = os.path.join(render_dir, 'geo_out'); os.makedirs(geo_dir, exist_ok=True)
                Image.fromarray(geo_out).save(os.path.join(geo_dir, str(img_idx).zfill(4) + '.png'))
        return {'img': img_out, 'depth': depth_out, 'geo': geo_out}

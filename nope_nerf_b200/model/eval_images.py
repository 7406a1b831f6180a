"""Eval_Images (reference: model/eval_images.py:16-137): novel-view evaluation of one test frame — render, PSNR / SSIM / LPIPS,
depth statistics inputs, image dumps.  The reference walks the frame in `points_batch_size` chunks through Renderer.forward
(eval_images.py:73-84); here the frame is ONE library call (Extract_Images.render_frame -> the persistent tensor-core forward) and MSE,
PSNR and SSIM are computed on the device from the rendered frame (the reference's third_party/pytorch_ssim formula: 11x11
Gaussian window, sigma 1.5, zero padding, mean over the map).  LPIPS stays the caller's network (`lpips_vgg_fn`, eval_nvs.py)."""
import os
import math
import numpy as np
import torch
import torch.nn.functional as F
from .extracting_images import Extract_Images


def mse2psnr(mse):
    """model/common.py:16-24"""
    if mse == 0:
        return 100.0
    return -10.0 * math.log10(mse)


def _gauss_window(channel, device, size=11, sigma=1.5):
    g = torch.tensor([math.exp(-(x - size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(size)], device=device)
    g = (g / g.sum()).unsqueeze(1)
    return (g @ g.t()).float()[None, None].expand(channel, 1, size, size).contiguous()


def ssim(img1, img2, window_size=11):
    """third_party/pytorch_ssim/__init__.py:20-49 (use_padding=True, size_average=True); img* (B,C,H,W) in [0,1]"""
    c = img1.shape[1]
    w = _gauss_window(c, img1.device, window_size)
    p = window_size // 2
    mu1 = F.conv2d(img1, w, padding=p, groups=c); mu2 = F.conv2d(img2, w, padding=p, groups=c)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1 = F.conv2d(img1 * img1, w, padding=p, groups=c) - mu1_sq
    s2 = F.conv2d(img2 * img2, w, padding=p, groups=c) - mu2_sq
    s12 = F.conv2d(img1 * img2, w, padding=p, groups=c) - mu12
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu12 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))).mean()


class Eval_Images(object):
    def __init__(self, renderer, cfg, points_batch_size=100000, use_learnt_poses=True, use_learnt_focal=True, device=None,
                 render_type=None, c2ws=None, img_list=None):
        self.points_batch_size = points_batch_size          # API compatibility; the frame is not chunked
        self.renderer = renderer
        self.resolution = cfg['extract_images']['resolution']
        self.device = device
        self.use_learnt_poses = use_learnt_poses
        self.use_learnt_focal = use_learnt_focal
        self.render_type = render_type
        self.c2ws = c2ws
        self.img_list = img_list
        self._ex = Extract_Images(renderer, cfg, use_learnt_poses=use_learnt_poses, use_learnt_focal=use_learnt_focal, device=device,
                                  render_type=render_type)

    def process_data_dict(self, data):
        """eval_images.py:30-44"""
        device = self.device
        img = data.get('img').to(device)
        batch_size, _, h, w = img.shape
        depth_img = data.get('img.depth', torch.ones(batch_size, h, w))
        img_idx = data.get('img.idx')
        camera_mat = data.get('img.camera_mat').to(device)
        scale_mat = data.get('img.scale_mat').to(device)
        return (img, depth_img, camera_mat, scale_mat, img_idx)

    def eval_images(self, data, render_dir, fxfy, lpips_vgg_fn, logger, min_depth=0.1, max_depth=20, it=0):
        """eval_images.py:46-137; returns the same img_dict (lpips is None when no network is passed)"""
        if self.render_type not in (None, 'nope_nerf'):
            raise NotImplementedError("Eval_Images: only the volumetric 'nope_nerf' render type is on the hot path")
        self.renderer.eval()
        (img_gt, depth_gt, camera_mat, scale_mat, img_idx) = self.process_data_dict(data)
        img_idx = int(img_idx)
        img_gt = img_gt.squeeze(0).permute(1, 2, 0)
        depth_gt = depth_gt.squeeze(0).cpu().numpy()
        mask = (depth_gt > min_depth) * (depth_gt < max_depth)
        dev = self.device
        c2w = self.c2ws[img_idx] if self.use_learnt_poses else torch.eye(4, device=dev)
        if self.use_learnt_focal:
            camera_mat = torch.diag(torch.stack([torch.as_tensor(fxfy[0], device=dev).float().reshape(()),
                                                 -torch.as_tensor(fxfy[1], device=dev).float().reshape(()),
                                                 -torch.ones((), device=dev), torch.ones((), device=dev)]))
        h, w = self.resolution
        with torch.no_grad():
            rgb, depth = self._ex.render_frame(c2w.to(dev), camera_mat.reshape(4, 4).to(dev), h, w)     # ONE call per frame
            img_out = rgb.view(h, w, 3)
            mse = F.mse_loss(img_out, img_gt).item()
            psnr = mse2psnr(mse)
            ssim_v = ssim(img_out.permute(2, 0, 1).unsqueeze(0), img_gt.permute(2, 0, 1).unsqueeze(0)).item()
            lpips_loss = None
            if lpips_vgg_fn is not None:
                lpips_loss = lpips_vgg_fn(img_out.permute(2, 0, 1).unsqueeze(0).contiguous(),
                                          img_gt.permute(2, 0, 1).unsqueeze(0).contiguous(), normalize=True).item()
            gt_h, gt_w = depth_gt.shape[:2]
            # cv2.resize(..., INTER_NEAREST) of the reference: source index = floor(dst * src / dst_size)
            ri = (torch.arange(gt_h, device=dev) * h // gt_h).clamp_(max=h - 1); ci = (torch.arange(gt_w, device=dev) * w // gt_w).clamp_(max=w - 1)
            depth_out = depth.view(h, w)[ri][:, ci].cpu().numpy()
        if logger is not None:
            logger.info('%4d img: PSNR: %.2f, SSIM: %.2f%s' % (img_idx, psnr, ssim_v, '' if lpips_loss is None else ',  LPIPS %.2f' % lpips_loss))
        depth_out = (np.clip(255.0 / depth_out.max() * (depth_out - depth_out.min()), 0, 255)).astype(np.uint8)
        img_np = (img_out.cpu().numpy() * 255).astype(np.uint8)
        gt_np = (img_gt.cpu().numpy() * 255).astype(np.uint8)
        if render_dir is not None:
            from PIL import Image
            for sub, arr in (('img_out', img_np), ('depth_out', depth_out), ('img_gt_out', gt_np)):
                d = os.path.join(render_dir, sub)
                os.makedirs(d, exist_ok=True)
                Image.fromarray(arr).save(os.path.join(d, str(img_idx).zfill(4) + '.png'))
        depth_out = depth_out[mask]
        depth_gt = depth_gt[mask]
        return {'img': img_np, 'depth': depth_out, 'mse': mse, 'psnr': psnr, 'ssim': ssim_v, 'lpips': lpips_loss,
                'depth_pred': depth_out, 'depth_gt': depth_gt}

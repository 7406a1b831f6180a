"""Trainer_pose (reference: model/eval_pose_one_epoch.py:9-98): test-time pose optimisation with
a frozen field — forward + data-gradient to the pose only (no weight gradients are computed)."""
import torch
from .. import ops
from .. import _lib as L
from .losses import Loss_Eval


class Trainer_pose(object):
    def __init__(self, model, cfg, device=None, optimizer_pose=None, pose_param_net=None, focal_net=None, **kwargs):
        self.model = model
        self.device = device
        self.optimizer_pose = optimizer_pose
        self.pose_param_net = pose_param_net
        self.focal_net = focal_net
        self.n_points = cfg['n_points']
        self.rendering_technique = cfg['type']
        self.loss = Loss_Eval()

    def train_step(self, data, it=100000):
        self.model.eval()
        self.pose_param_net.train()
        self.optimizer_pose.zero_grad()
        if self.focal_net is not None:
            self.focal_net.eval()
        loss_dict = self.compute_loss(data, it=it, backward=True)
        self.optimizer_pose.step()
        return loss_dict

    def compute_loss(self, data, eval_mode=False, it=100000, backward=False):
        """eval_pose_one_epoch.py:62-98: prior depth = ones, eval mode, no jitter, loss = mse(rgb)."""
        device = self.device
        img = data.get('img').to(device, non_blocking=True)
        img_idx = int(data.get('img.idx'))
        _, _, h, w = img.shape
        camera_mat = data.get('img.camera_mat').to(device).reshape(4, 4).contiguous().float()
        if self.focal_net is not None:
            fxfy = self.focal_net(0).detach()
            camera_mat = torch.diag(torch.stack([fxfy[0], -fxfy[1], -torch.ones((), device=device), torch.ones((), device=device)]))
        pose = self.pose_param_net
        rend = self.model.renderer; net = rend.model
        n = self.n_points
        ray_idx = torch.randperm(h * w, device=device)[:n]
        c2w = torch.empty(4, 4, device=device)
        init = None if pose.init_c2w is None else pose.init_c2w.detach()
        ops.pose_fwd_raw(pose.r.detach(), pose.t.detach(), init, img_idx, c2w)
        ndc = rend.cfg['sample_option'] == 'ndc'
        ones = torch.ones(n, device=device)
        call = ops.RenderCall(net.flat_weights(), c2w, camera_mat, N=n, S=int(rend.cfg['num_points']),
                              flags=ops.flags_from_cfg(rend.cfg, net.occ_activation, eval_=True),
                              engine=rend.engine if rend.engine is not None else ops.default_engine(),
                              near=0.0 if ndc else rend.depth_range[0], far=1.0 if ndc else rend.depth_range[1],
                              ray_idx=ray_idx, depth=ones, H=h, W=w, stash=backward, hidden_dim=net.hidden_dim)
        # F.mse_loss(rgb, rgb_gt) == l2_mean; seeds: d/d rgb = 2 diff / (3 N)  -> w_rgb = 1/3 with the l2 form
        out4, g_rgb, g_dp, g_dg = ops.loss_rgb_depth(call.rgb, call.depth_pred, call.depth_gt, call.mask, 1.0 / 3.0, 0.0, True,
                                                     img=img.reshape(3, h * w), ray_idx=ray_idx)
        if backward:
            g_c2w = torch.zeros(4, 4, device=device)
            call.backward(g_rgb, None, None, None, g_c2w)
            g_r = torch.zeros_like(pose.r) if pose.r.requires_grad else None
            g_t = torch.zeros_like(pose.t) if pose.t.requires_grad else None
            ops.pose_bwd_raw(pose.r.detach(), pose.t.detach(), init, img_idx, g_c2w, g_r, g_t)
            if g_r is not None: pose.r.grad = g_r
            if g_t is not None: pose.t.grad = g_t
        return {'loss': out4[3]}

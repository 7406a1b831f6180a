"""Trainer (reference: model/training.py:14-379) — one optimisation step of NoPe-NeRF.

Same constructor / train_step / render_visdata surface and the same loss_dict keys, but the
render + photometric/depth loss + backward of a step are a fixed sequence of calls into the
CUDA library (no autograd graph over the field):

    nnb_pose_fwd -> nnb_render_fwd(STASH) -> nnb_loss_rgb_depth -> nnb_render_bwd -> nnb_pose_bwd

Gradients land in ONE flat fp32 buffer [MLP | r | t | scales | shifts | (focal, when learned) | 4 loss scalars] whose
slices are installed as every parameter's .grad, so (a) train.py's own torch.optim.Adam
instances step unchanged and (b) data-parallel training is a single NCCL all-reduce of that
buffer per step (SURVEY.md 8(e)).  The point-cloud / warped-RGB terms of the reference-image
stage (training.py:280-365) are ONE more library call (nnb_refstage: forward + adjoint) whose pose /
distortion gradients accumulate into the same buffer.
"""
import logging
import os
import numpy as np
import torch
from .. import ops
from .. import _lib as L
from .losses import Loss
from .common import arange_pixels
from .rendering import GEOMETRY_CHUNK, _frame_grad_engine

logger_py = logging.getLogger(__name__)


class _FlatAdam:
    """torch.optim.Adam.step() for an optimizer whose parameters alias one flat buffer (or are few, small
    tensors), executed by nnb_adam_step.  The optimizer object stays the caller's (train.py:58,99,117):
    hyper-parameters are read from `param_groups` every step (LR schedulers keep working) and the moments live
    in `optimizer.state[p]` with torch's own keys ('step', 'exp_avg', 'exp_avg_sq'), so `state_dict()` /
    `load_state_dict()` round-trip with the reference's CheckpointIO unchanged."""

    def __init__(self, optimizer, flat_param=None, flat_slices=None):
        self.opt = optimizer
        self.flat_param = flat_param          # callable -> flat tensor aliasing all params (MLP) or None
        self.flat_slices = flat_slices
        self.m = self.v = None
        self.ok = self._supported()
        self.nsteps = 0              # steps taken so far (source of truth shared with the CUDA-graph path)
        self._synced = True
        self._ready = False          # moment buffers adopted into optimizer.state (re-checked after load_state_dict)
        self._loaded = False         # optimizer.load_state_dict() happened since the last step: adopt ITS step count
        try:
            optimizer.register_state_dict_pre_hook(lambda opt: self.sync_step_tensors())
        except Exception:
            pass
        try:
            optimizer.register_load_state_dict_post_hook(lambda opt: self._mark_loaded())
        except Exception:
            pass

    def _mark_loaded(self):
        self._loaded = True
        self._ready = False

    def adopt_loaded_step(self):
        """torch.optim.Adam continues bias correction from the loaded 'step' (checkpoint resume, train.py:60-67); so do we"""
        st0 = next((st for st in self.opt.state.values() if 'step' in st), None)
        if st0 is None:
            return
        if self._loaded:
            self.nsteps = int(st0['step']); self._synced = True
        elif self._synced and int(st0['step']) > self.nsteps:
            self.nsteps = int(st0['step'])
        self._loaded = False

    def sync_step_tensors(self):
        """optimizer.state[p]['step'] tensors follow `nsteps` lazily (the graph path does not touch them per step)"""
        for st in self.opt.state.values():
            if 'step' in st: st['step'].fill_(float(self.nsteps))
        self._synced = True

    def ensure_state(self):
        """allocate / adopt the moment buffers without stepping"""
        if self._ready and not self._loaded:
            return                   # per-step fast path: nothing changed since the last adoption
        self._ready = True
        g = self.opt.param_groups[0]
        if self.flat_param is not None:
            flat = self.flat_param(); plist = list(g['params']); n = flat.numel()
            if self.m is None or self.m.device != flat.device:
                self.m = torch.zeros(n, device=flat.device); self.v = torch.zeros(n, device=flat.device)
            for p, (o, k, sh) in zip(plist, self.flat_slices):
                self._state(p, self.m[o:o + k].view(sh), self.v[o:o + k].view(sh))
        else:
            if self.m is None:
                self.m = {}; self.v = {}
            for p in g['params']:
                key = id(p)
                if key not in self.m or self.m[key].shape != p.shape or self.m[key].device != p.device:
                    self.m[key] = torch.zeros_like(p); self.v[key] = torch.zeros_like(p)
                self._state(p, self.m[key], self.v[key])
        self.adopt_loaded_step()                     # e.g. optimizer state loaded from a checkpoint

    def _supported(self):
        o = self.opt
        if type(o) is not torch.optim.Adam or len(o.param_groups) != 1:
            return False
        g = o.param_groups[0]
        return not (g.get('amsgrad', False) or g.get('maximize', False) or g.get('weight_decay', 0) != 0 or
                    g.get('capturable', False) or g.get('differentiable', False))

    def _state(self, p, m_view, v_view):
        st = self.opt.state[p]
        if 'step' not in st:
            st['step'] = torch.tensor(0.0, dtype=torch.float32)
        for key, view in (('exp_avg', m_view), ('exp_avg_sq', v_view)):
            cur = st.get(key)
            if cur is None:
                view.zero_()
            elif cur.data_ptr() != view.data_ptr():          # e.g. after load_state_dict: adopt the loaded moments
                view.copy_(cur.to(view.device, view.dtype))
            st[key] = view
        return st

    def step(self):
        g = self.opt.param_groups[0]
        params = [p for p in g['params'] if p.requires_grad and p.grad is not None]
        if not self.ok or not params:
            return self.opt.step()
        if self._loaded or (self._synced and self.nsteps == 0):
            self.adopt_loaded_step()
        lr, (b1, b2), eps = g['lr'], g['betas'], g['eps']
        if self.flat_param is not None:
            flat = self.flat_param()
            plist = list(g['params'])
            if len(plist) != len(self.flat_slices) or any(p.data_ptr() != flat.data_ptr() + 4 * o
                                                          for p, (o, n, s) in zip(plist, self.flat_slices)):
                return self.opt.step()
            g0 = plist[0].grad
            n = flat.numel()
            if self.m is None or self.m.device != flat.device:
                self.m = torch.zeros(n, device=flat.device); self.v = torch.zeros(n, device=flat.device)
            sts = [self._state(p, self.m[o:o + k].view(sh), self.v[o:o + k].view(sh)) for p, (o, k, sh) in zip(plist, self.flat_slices)]
            step = self.nsteps + 1
            gflat_ptr_ok = all(p.grad is not None and p.grad.data_ptr() == g0.data_ptr() + 4 * o for p, (o, k, sh) in zip(plist, self.flat_slices))
            if not gflat_ptr_ok:
                return self.opt.step()
            gflat = torch.as_strided(g0, (n,), (1,))      # the installed .grad views alias one flat gradient buffer
            ops.adam_step(flat, gflat, self.m, self.v, step, lr, b1, b2, eps)
            self.nsteps = step; self._synced = False
        else:
            if self.m is None:
                self.m = {}; self.v = {}
            for p in params:
                key = id(p)
                if key not in self.m or self.m[key].shape != p.shape or self.m[key].device != p.device:
                    self.m[key] = torch.zeros_like(p); self.v[key] = torch.zeros_like(p)
                st = self._state(p, self.m[key], self.v[key])
                step = self.nsteps + 1
                gr = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                ops.adam_step(p.data, gr, self.m[key], self.v[key], step, lr, b1, b2, eps)
            self.nsteps += 1; self._synced = False


def _host_diag_check(camera_mat):
    """camera_mat must be diag(kx, ky, -1, 1) (dataset.py:101-104); checked on host tensors only."""
    if camera_mat.is_cuda:
        return
    m = camera_mat.reshape(4, 4)
    off = m - torch.diag(torch.diagonal(m))
    if off.abs().max() != 0 or m[2, 2] != -1 or m[3, 3] != 1:
        raise NotImplementedError("camera_mat must be diag(kx, ky, -1, 1)")


class _GraphStep:
    """The whole training step (pose exp-map, distortion, pixel sampling, render forward, losses, [reference-image stage],
    backward, [all-reduce], Adam x3) captured ONCE as a CUDA graph and replayed per frame.  Everything that changes from step
    to step is read from device memory: camera indices, frame pointers, DPT maps, camera matrix, loss weights (annealed per
    epoch), Adam step counters, learning rates.  The first call runs the same body eagerly (that IS that call's training step and
    warms every lazy initialisation), the second call captures, later calls replay.  With `use_ref` the reference-image stage
    (point-cloud + warped-RGB terms, training.py:280-365) runs on a forked stream beside the render forward / backward.
    Options of the trainer that add kernels to the step (each only when on, so the default step's graph is unchanged):
      * learned focal (pose.learn_focal): the camera matrix is written from the focal parameters on the device (nnb_focal_fwd), their
        gradient (render backward's g_cam + the reference-image stage's g_kxy) lands in the focal slot of the flat gradient buffer
        (nnb_focal_bwd) and the focal optimizer is one more Adam segment of the exchange;
      * invariant depth (training.depth_loss_type = invariant): nnb_depth_invariant replaces the L1 depth term and adds its seeds;
      * pose smoothness (training.weight_dist_1st_loss / weight_dist_2nd_loss): nnb_pose_smooth adds its translation gradient."""

    def __init__(self, tr, h, w, hd, wd, rgb_l2, use_ref):
        self.tr = tr; self.key = (h, w, hd, wd, bool(rgb_l2), bool(use_ref))
        dev = tr.device
        self.h, self.w, self.hd, self.wd = h, w, hd, wd
        self.rgb_l2, self.use_ref = bool(rgb_l2), bool(use_ref)
        self.focal = tr.optimizer_focal is not None
        self.inv = tr.depth_loss_type == 'invariant'
        self.smooth = tr._smoothness_on()
        # per-step host scalars travel as ONE 32-byte asynchronous copy from a ring of page-locked slots:
        # meta = int64 [camera index, reference camera index, frame pointer, reference frame pointer]
        self.meta = torch.zeros(4, dtype=torch.int64, device=dev)
        m32 = self.meta.view(torch.int32)
        self.idx = m32[0:1]; self.idx_ref = m32[2:3]
        self.imgpp = self.meta[2:4]                                       # frame pointers {current, reference}
        self.meta_host = torch.zeros(16, 4, dtype=torch.int64).pin_memory(); self.meta_np = self.meta_host.numpy()
        self.meta_ev = [None] * 16
        self.ev_pool = []                                   # recycled events of the host-frame keep-alive list
        self.dpt = torch.zeros(hd, wd, device=dev)
        self.cam = torch.zeros(4, 4, device=dev); self.cam_host = None
        self.ss = torch.zeros(2, device=dev)               # effective (scale, shift) of the current view
        self.c2w = torch.zeros(4, 4, device=dev)
        self.small = torch.zeros(16 + 2, device=dev)       # [g_c2w | g_scale_shift]
        n_opt = 4 if self.focal else 3
        self.steps = torch.zeros(n_opt, dtype=torch.int32, device=dev)   # Adam step counters: mlp, pose, distortion[, focal]
        self.lrs = torch.zeros(n_opt, device=dev); self.lr_host = [None] * n_opt
        # {w_rgb, w_depth (L1), w_pc, w_rgb_s, w_dist_1st, w_dist_2nd, w_depth (invariant), 0}
        self.wts = torch.zeros(8, device=dev); self.wts_host = None
        if self.focal:
            self.cam_gt = torch.zeros(4, 4, device=dev)          # the dataset's camera matrix (loss_dict['focalx'/'focaly'])
            self.g_focal = torch.zeros(16 + 2, device=dev)       # [g_cam | g_kxy]
        if self.smooth:
            self.dist_losses = torch.zeros(2, device=dev)        # {loss_dist_1st, loss_dist_2nd}
        self.out4 = torch.zeros(4, device=dev)
        N = tr.n_training_points // tr.world if tr.dp_mode == 'rays' else tr.n_training_points
        self.g_rgb = torch.zeros(N, 3, device=dev); self.g_dp = torch.zeros(N, device=dev); self.g_dg = torch.zeros(N, device=dev)
        self.graph = None; self.calls = 0; self.keep = []; self.host_refs = []; self.dev_refs = None
        self.rs_losses = torch.zeros(2, device=dev)        # {loss_pc, loss_rgb_s} of the reference-image stage (full-loss steps)
        self.rs_total = torch.zeros(1, device=dev)
        if self.use_ref:
            self.dpt_ref = torch.zeros(hd, wd, device=dev)
            self.c2w_ref = torch.zeros(4, 4, device=dev); self.ss_ref = torch.zeros(2, device=dev)
            self.with_ssim = bool(tr.loss.cfg.get('with_ssim', False))
            self.grad_ref = not tr.detach_ref_img
            flags = ops.refstage_flags(tr.scale_pcs, tr.detach_rgbs_scale, tr.shift_first, self.with_ssim, self.grad_ref)
            nbytes = L.lib.nnb_refstage_workspace_bytes_flags(hd, wd, int(tr.pc_ratio), flags)
            if nbytes == 0:
                raise ValueError("reference-image stage: DPT map %dx%d too small for pc_ratio %d" % (hd, wd, tr.pc_ratio))
            self.rs_ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            self.side = torch.cuda.Stream(device=dev)
            # training.detach_ref_img = False: [g_c2w_ref | g_scale_shift_ref] of the reference view, chained after the current view's
            self.small_ref = torch.zeros(16 + 2, device=dev) if self.grad_ref else None
            self.stage = None                              # device staging of host frames (2,3,h,w), allocated on first use
        self.fadams = None

    def _adams(self):
        tr = self.tr
        if self.fadams is None:
            self.fadams = [tr._fadam_for(tr.optimizer, True), tr._fadam_for(tr.optimizer_pose, False),
                           tr._fadam_for(tr.optimizer_distortion, False)]
            if self.focal:
                self.fadams.append(tr._fadam_for(tr.optimizer_focal, False))
        return self.fadams

    def _optimizers(self):
        tr = self.tr
        return (tr.optimizer, tr.optimizer_pose, tr.optimizer_distortion) + ((tr.optimizer_focal,) if self.focal else ())

    def _focal_params(self):
        """(fx, fy or None (fx_only), order) of the LearnFocal module"""
        fn = self.tr.focal_net
        return fn.fx, (None if fn.fx_only else fn.fy), int(fn.order)

    def eligible_optimizers(self):
        return all(fa.ok for fa in self._adams())

    def body(self):
        self.body_a()
        if self.tr._peer is not None:
            self.body_peer()
        else:
            self.reduce(); self.body_b()

    def body_peer(self):
        """data parallel: all-reduce of the flat gradient buffer over NVLink peer memory fused with the three Adam updates"""
        tr = self.tr
        net = tr.model.renderer.model; pose, dnet = tr.pose_param_net, tr.distortion_net
        V = pose.num_cams; o = net.num_params
        ops.counter_incr(self.steps)
        fa_m, fa_p, fa_d = self._adams()[:3]
        gm = tr.optimizer.param_groups[0]; b1, b2 = gm['betas']
        segs = [(net.flat_weights(), fa_m.m, fa_m.v, 0, o, self.lrs[0:1], self.steps[0:1], b1, b2, gm['eps'])]
        gp = tr.optimizer_pose.param_groups[0]; gd = tr.optimizer_distortion.param_groups[0]
        groups = [(pose.r, o, 3 * V, fa_p, gp, 1), (pose.t, o + 3 * V, 3 * V, fa_p, gp, 1),
                  (dnet.global_scales, o + 6 * V, V, fa_d, gd, 2), (dnet.global_shifts, o + 7 * V, V, fa_d, gd, 2)]
        if self.focal:                                      # focal slot [fx, fy] after the shifts
            fx, fy, _ = self._focal_params(); fa_f = self._adams()[3]; gf = tr.optimizer_focal.param_groups[0]
            groups += [(fx, o + 8 * V, 1, fa_f, gf, 3)] + ([(fy, o + 8 * V + 1, 1, fa_f, gf, 3)] if fy is not None else [])
        for prm, off, cnt, fa, g_, k in groups:
            if prm.requires_grad and id(prm) in fa.m:
                segs.append((prm.data, fa.m[id(prm)], fa.v[id(prm)], off, cnt, self.lrs[k:k + 1], self.steps[k:k + 1], g_['betas'][0], g_['betas'][1], g_['eps']))
        tr._peer.allreduce_adam(segs)

    def body_a(self):
        """everything up to the local gradients"""
        tr = self.tr; dev = tr.device
        pose, dnet = tr.pose_param_net, tr.distortion_net
        net = tr.model.renderer.model; rend = tr.model.renderer
        h, w = self.h, self.w
        gbuf, gv = tr._grad_buffer(peer_step=True)
        self.small.zero_()
        g_c2w = self.small[:16].view(4, 4); g_ss = self.small[16:18]
        grad_ref = self.use_ref and self.grad_ref
        if grad_ref:
            self.small_ref.zero_()
        g_cam = g_kxy = None
        if self.focal:                                      # camera matrix from the focal parameters (training.py:247-252)
            fx, fy, order = self._focal_params()
            ops.focal_fwd(fx.detach(), None if fy is None else fy.detach(), order, self.cam)
            self.g_focal.zero_()
            g_cam = self.g_focal[:16].view(4, 4)
            g_kxy = self.g_focal[16:18] if self.use_ref else None
        ops.distortion_fwd_dev(dnet.global_scales.detach(), dnet.global_shifts.detach(), self.idx, dnet.fix_scaleN, self.ss)
        init = None if pose.init_c2w is None else pose.init_c2w.detach()
        ops.pose_fwd_dev(pose.r.detach(), pose.t.detach(), init, self.idx, self.c2w)
        gs = 1.0 / tr.world
        n_points = tr.n_training_points
        if tr.pixel_sampler == 'randperm' or (tr.pixel_sampler == 'auto' and not tr.use_cuda_graph) or n_points > min(h * w // 2, 8192):
            ray_idx = torch.randperm(h * w, device=dev)[:n_points]                # training.py:257 (reference RNG stream)
        else:
            ray_idx = ops.sample_pixels(h * w, n_points, dev)                     # same distribution, no 2M-key sort
        S = int(rend.cfg['num_points'])
        noise = None
        if rend.cfg['sample_option'] == 'uniform':
            noise = torch.rand(1, n_points, S, device=dev)[0]                      # rendering.py:189
        if tr.world > 1 and tr.dp_mode == 'rays':
            ray_idx = ray_idx[tr.rank::tr.world].contiguous()
            if noise is not None: noise = noise[tr.rank::tr.world].contiguous()
        n_local = ray_idx.shape[0]
        flags = ops.flags_from_cfg(rend.cfg, net.occ_activation, eval_=False, shift_first=tr.shift_first)
        ndc = rend.cfg['sample_option'] == 'ndc'
        render_call = tr._train_render_call(True)
        call = render_call(net.flat_weights(), self.c2w, self.cam, N=n_local, S=S, flags=flags,
                           engine=rend.engine if rend.engine is not None else ops.default_engine(),
                           near=0.0 if ndc else rend.depth_range[0], far=1.0 if ndc else rend.depth_range[1],
                           ray_idx=ray_idx, depth_map=self.dpt, scale=self.ss[0:1], shift=self.ss[1:2], noise=noise, H=h, W=w, stash=True,
                           hidden_dim=net.hidden_dim)
        if rend.cfg.get('normal_loss', False) and not tr.use_cuda_graph:
            tr._normal_draw(call.mask)
        ops.loss_rgb_depth_indirect(call.rgb, call.depth_pred, call.depth_gt, call.mask, 0.0, 0.0, self.rgb_l2, self.imgpp,
                                    ray_idx, h * w, self.out4, self.g_rgb, self.g_dp, self.g_dg, grad_scale=gs, w_dev=self.wts)
        if self.inv:                                        # losses.py:34-57 (the L1 depth weight on the device is 0)
            ops.depth_invariant(call.depth_pred, call.depth_gt, call.mask, self.wts[6:7], self.out4, self.g_dp,
                                None if tr.detach_gt_depth else self.g_dg, grad_scale=gs)
        ws = call.ws
        call.pooled = False                                 # memory referenced by a captured graph never returns to the pool
        bw = (self.g_rgb, self.g_dp, None if tr.detach_gt_depth else self.g_dg, gbuf[:net.num_params], g_c2w, g_cam, None, g_ss)
        call.backward(*bw)
        if self.use_ref:
            # The reference-image stage only needs the two poses / distortions / frames.  It runs on a side stream that starts after
            # the whole render backward, so it sits on the step's critical path.  The stage sums in a fixed order (the chamfer's
            # adjoint groups exactly, in integers) and adds its pose / distortion gradients once per element into the buffers the
            # render backward also accumulates into; because the backward has finished by then, those adds always land in the same
            # order and the step is reproducible bit for bit.
            cur = torch.cuda.current_stream()
            self.side.wait_stream(cur)
            with torch.cuda.stream(self.side):
                ops.pose_fwd_dev(pose.r.detach(), pose.t.detach(), init, self.idx_ref, self.c2w_ref)
                ops.distortion_fwd_dev(dnet.global_scales.detach(), dnet.global_shifts.detach(), self.idx_ref, dnet.fix_scaleN, self.ss_ref)
                self.rs_total.zero_()
                ops.refstage_raw(self.c2w, self.ss, self.c2w_ref, self.ss_ref, self.dpt, self.dpt_ref, H=h, W=w, img_pp=self.imgpp, cam=self.cam,
                                 cam_idx_dev=self.idx, num_cams=pose.num_cams, weights_dev=self.wts[2:4], nearest_limit=tr.nearest_limit,
                                 pc_ratio=tr.pc_ratio, scale_pcs=tr.scale_pcs, detach_rgbs_scale=tr.detach_rgbs_scale, shift_first=tr.shift_first,
                                 losses=self.rs_losses, g_c2w=g_c2w, g_dist=g_ss, loss_total=self.rs_total, grad_scale=gs, workspace=self.rs_ws,
                                 with_ssim=self.with_ssim, g_c2w_ref=self.small_ref[:16].view(4, 4) if grad_ref else None,
                                 g_dist_ref=self.small_ref[16:18] if grad_ref else None, g_kxy=g_kxy)
            cur.wait_stream(self.side)
        self.keep.append((call, ws, ray_idx, noise))        # graph-owned memory stays referenced (and out of the workspace pool)
        ops.pose_bwd_dev(pose.r.detach(), pose.t.detach(), init, self.idx, g_c2w,
                         gv['r'] if pose.r.requires_grad else None, gv['t'] if pose.t.requires_grad else None)
        ops.distortion_bwd_dev(dnet.global_scales.detach(), self.idx, dnet.fix_scaleN, g_ss,
                               gv['scales'] if dnet.global_scales.requires_grad else None,
                               gv['shifts'] if dnet.global_shifts.requires_grad else None)
        if grad_ref:                                        # the reference view's rows, after the current view's (fixed order)
            ops.pose_bwd_dev(pose.r.detach(), pose.t.detach(), init, self.idx_ref, self.small_ref[:16].view(4, 4),
                             gv['r'] if pose.r.requires_grad else None, gv['t'] if pose.t.requires_grad else None)
            ops.distortion_bwd_dev(dnet.global_scales.detach(), self.idx_ref, dnet.fix_scaleN, self.small_ref[16:18],
                                   gv['scales'] if dnet.global_scales.requires_grad else None,
                                   gv['shifts'] if dnet.global_shifts.requires_grad else None)
        if self.focal:                                      # after the reference-image stage's g_kxy (fixed order)
            ops.focal_bwd(fx.detach(), None if fy is None else fy.detach(), order, g_cam, g_kxy, gv['fx'], gv.get('fy'))
        gv['losses'].copy_(self.out4 * gs if tr.world > 1 else self.out4)
        if self.use_ref:
            gv['losses'][0:1].add_(self.rs_total, alpha=gs)
        if self.smooth:                                     # losses.py:103-112; every rank holds the same t: 1/world of it each
            ops.pose_smooth(pose.t.detach(), self.wts[4:6], self.dist_losses, loss_total=gv['losses'][0:1],
                            g_t=gv['t'] if pose.t.requires_grad else None, grad_scale=gs)

    def reduce(self):
        tr = self.tr
        if tr.world > 1:
            torch.distributed.all_reduce(tr._gbuf, group=tr.dp_group)

    def body_b(self):
        """optimizers: device-side step counters / learning rates"""
        tr = self.tr
        gbuf = tr._gbuf
        net = tr.model.renderer.model
        ops.counter_incr(self.steps)
        fas = self._adams(); fa_m = fas[0]
        gm = tr.optimizer.param_groups[0]; b1, b2 = gm['betas']
        flat = net.flat_weights()
        ops.adam_step_dev(flat, gbuf[:net.num_params], fa_m.m, fa_m.v, self.steps[0:1], self.lrs[0:1], b1, b2, gm['eps'])
        for k, (fa, opt) in enumerate(zip(fas, self._optimizers())):
            if k == 0:
                continue
            g = opt.param_groups[0]; b1, b2 = g['betas']
            for p in g['params']:
                if p.requires_grad and p.grad is not None:
                    ops.adam_step_dev(p.data, p.grad, fa.m[id(p)], fa.v[id(p)], self.steps[k:k + 1], self.lrs[k:k + 1], b1, b2, g['eps'])

    def _frame_ptr(self, t, slot):
        """device pointer of a (1,3,h,w) frame: device tensors and page-locked host tensors are used in place (render-only steps read
        N pixels of them); full-loss steps bilinearly resample both whole frames, so host frames are staged in HBM first"""
        dev = self.tr.device
        if t.device.type == 'cpu' and (self.use_ref or not t.is_pinned()):
            if self.use_ref:
                if self.stage is None:
                    self.stage = torch.empty(2, 3, self.h, self.w, device=dev)
                self.stage[slot].copy_(t.reshape(3, self.h, self.w), non_blocking=True)
                return self.stage[slot], t
            t = t.to(dev, non_blocking=True)
        return t, t

    def run(self, data, wts):
        tr = self.tr; dev = tr.device
        cur_stream = torch.cuda.current_stream()
        img, img_keep = self._frame_ptr(data.get('img'), 0)
        meta = [int(data.get('img.idx')), 0, img.data_ptr(), 0]
        keep = [img_keep]
        self.dpt.copy_(data.get('img.dpt').reshape(self.hd, self.wd), non_blocking=True)
        if self.use_ref:
            ref, ref_keep = self._frame_ptr(data.get('img.ref_imgs'), 1)
            meta[3] = ref.data_ptr(); keep.append(ref_keep)
            meta[1] = int(data.get('img.ref_idxs'))
            self.dpt_ref.copy_(data.get('img.ref_dpts').reshape(self.hd, self.wd), non_blocking=True)
        if getattr(self, 'meta_last', None) != meta:
            k = self.calls % 16
            if self.meta_ev[k] is not None: self.meta_ev[k].synchronize()   # the slot's previous copy has run (16 steps ago)
            self.meta_np[k] = meta
            self.meta.copy_(self.meta_host[k], non_blocking=True)
            if self.meta_ev[k] is None: self.meta_ev[k] = torch.cuda.Event()
            self.meta_ev[k].record(cur_stream)
            self.meta_last = meta
        self.dev_refs = keep
        cm = data.get('img.camera_mat')
        cm_key = (cm.data_ptr(), cm._version)
        cam = self.cam_gt if self.focal else self.cam          # learned focal: the step's camera matrix comes from nnb_focal_fwd
        if cm.device.type == 'cpu' and self.cam_host is not None and getattr(self, 'cam_key', None) == cm_key:
            pass                                              # same host tensor as last step, unmodified
        elif self.cam_host is None or (cm.device.type == 'cpu' and not torch.equal(cm.reshape(4, 4), self.cam_host)):
            _host_diag_check(cm)
            self.cam_host = cm.reshape(4, 4).clone() if cm.device.type == 'cpu' else None
            cam.copy_(cm.reshape(4, 4))
        elif cm.device.type != 'cpu':
            cam.copy_(cm.reshape(4, 4))
        self.cam_key = cm_key
        if self.wts_host != wts:
            self.wts.copy_(torch.tensor(wts, dtype=torch.float32)); self.wts_host = list(wts)
        fas = self._adams()
        for k, (fa, opt) in enumerate(zip(fas, self._optimizers())):
            fa.ensure_state()
            lr = float(opt.param_groups[0]['lr'])
            if self.lr_host[k] != lr:
                self.lrs[k:k + 1].fill_(lr); self.lr_host[k] = lr
        want = [fa.nsteps for fa in fas]
        if getattr(self, 'steps_host', None) != want:
            self.steps.copy_(torch.tensor(want, dtype=torch.int32)); self.steps_host = list(want)
        self.calls += 1
        if self.calls == 1 or not tr.use_cuda_graph:
            self.body()                                   # eager (also the warm-up of every lazy initialisation)
            self.keep.clear()
        else:
            if self.graph is None:
                torch.cuda.synchronize()
                # world == 1: one graph for the whole step.  world > 1: the NCCL all-reduce stays an eager call between two
                # graphs (gradients | optimizers); thread_local because the NCCL watchdog thread touches the CUDA API
                self.graph = torch.cuda.CUDAGraph(keep_graph=True) if tr.keep_graph else torch.cuda.CUDAGraph()
                if tr.world == 1 or tr._peer is not None:      # peer exchange: the collective is one of the graph's kernels
                    with torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
                        self.body()
                else:
                    with torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
                        self.body_a()
                    self.graph_b = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(self.graph_b, capture_error_mode="thread_local"):
                        self.body_b()
            self.graph.replay()
            if tr.world > 1 and tr._peer is None:
                self.reduce()
                self.graph_b.replay()
        for fa in fas:
            fa.nsteps += 1; fa._synced = False
        self.steps_host = [fa.nsteps for fa in fas]
        if any(t.device.type == 'cpu' for t in keep):
            # a page-locked host frame is read IN PLACE (or copied asynchronously) by this step: keep it referenced until the step has
            # run (torch's pinned-memory allocator only tracks torch-issued copies, so a recycled DataLoader buffer could be refilled)
            ev = self.ev_pool.pop() if self.ev_pool else torch.cuda.Event()
            ev.record(cur_stream)
            self.host_refs.append((keep, ev))
            while len(self.host_refs) > 1 and self.host_refs[0][1].query():
                self.ev_pool.append(self.host_refs.pop(0)[1])
        # per-call snapshot (ONE small kernel): later steps overwrite the persistent buffers the graph writes to, and train.py
        # keeps loss_dict['scale'/'shift'] per view (train.py:215-216)
        parts = [(tr._peer.reduced if tr._peer is not None else tr._gbuf)[-4:], self.ss, self.rs_losses]
        if self.smooth:
            parts.append(self.dist_losses)
        if self.focal:                                        # {fx', -fy'} of this step's camera matrix over the dataset's {kx, ky}
            parts.append(self.cam.view(16)[0:6:5] / self.cam_gt.view(16)[0:6:5])
        snap = torch.cat(parts)
        s_ = snap.unbind(0)
        if getattr(self, 'zero', None) is None:
            self.zero = snap.new_zeros(())
        zero = self.zero
        ld = {'loss': s_[0], 'loss_rgb': s_[1], 'loss_depth': s_[2], 'l2_mean': s_[3],
              'loss_dist_1st': zero, 'loss_dist_2nd': zero, 'loss_pc': s_[6] if wts[2] != 0.0 else zero,
              'loss_rgb_s': s_[7] if wts[3] != 0.0 else zero, 'loss_depth_consistency': zero, 'scale': snap[4:5], 'shift': snap[5:6]}
        if self.smooth and (wts[4] != 0.0 or wts[5] != 0.0):
            ld['loss_dist_1st'], ld['loss_dist_2nd'] = s_[8], s_[9]
        if self.focal:
            j = 10 if self.smooth else 8
            ld['focalx'], ld['focaly'] = s_[j], -s_[j + 1]
        return ld


class Trainer(object):
    """Keyword options (besides the reference's arguments) include frame_grad (default False): with True, every training render that has
    a backward, in the captured graph step and in the general path, runs the differentiable frame's training pair ops.FrameRenderCall.
    Its workspace grows with rendering.num_points by one float per ray and 32-sample chunk instead of the per-sample stash, and it takes
    the jitter of sample_option 'uniform'.  The renderer's engine and rendering.num_points must resolve to the tensor-core engine
    (ValueError otherwise).  Renders without a backward are unchanged.  This is a Trainer keyword, not a reading of
    Renderer(frame_grad=...): that flag governs Renderer.nope_nerf, which the Trainer does not call.
    frame_grad_engine (default None, needs frame_grad=True): 'simt' runs those renders on the exact-fp32 engine's pair,
    ops.ExactFrameRenderCall, at any rendering.num_points from 2 to 1024 whatever the renderer's engine; None or 'tc' is the tensor-core
    pair above.
    frame_grad_t_min (default None, needs frame_grad=True on the tensor-core pair): train with early ray termination,
    ops.frame_render_call(t): a ray stops after the first 32-sample chunk that leaves its transmittance below t, and the backward
    differentiates that truncated render, visiting only the rays that evaluated each chunk.  0.0 gives the frame_grad=True step's bits.
    With frame_grad=False, frame_grad_engine='simt', or a negative or NaN value, it is a ValueError.
    train_t_min (default None): train with early ray termination on the per-sample stash, ops.stash_render_call(t), for every training
    render that has a backward: each sample is evaluated once and the backward runs one weight-gradient stage on the samples evaluated,
    in the stash path's worst-case memory (frame_grad_t_min is the choice when memory is the limit).  0.0 gives the default step's
    forward.  With frame_grad=True, a renderer that does not resolve to the tensor-core engine, or a negative or NaN value, it is a
    ValueError.
    train_t_min_engine (default None, needs train_t_min): 'simt' runs those renders on the exact-fp32 engine's pair,
    ops.exact_stash_render_call(t), at any rendering.num_points from 2 to 1024 whatever the renderer's engine, so that a truncated run can
    be told apart from the tensor cores' rounding; None or 'tc' is the tensor-core pair above.  Any other value, the keyword without
    train_t_min, or with frame_grad=True, is a ValueError."""

    def __init__(self, model, optimizer, cfg, device=None, optimizer_pose=None, pose_param_net=None,
                 optimizer_focal=None, focal_net=None, optimizer_distortion=None, distortion_net=None, **kwargs):
        self.model = model
        self.optimizer = optimizer
        self.device = device
        self.optimizer_pose = optimizer_pose
        self.pose_param_net = pose_param_net
        self.focal_net = focal_net
        self.optimizer_focal = optimizer_focal
        self.distortion_net = distortion_net
        self.optimizer_distortion = optimizer_distortion
        self.n_training_points = cfg['n_training_points']
        self.rendering_technique = cfg['type']
        self.vis_geo = cfg['vis_geo']
        self.detach_gt_depth = cfg['detach_gt_depth']
        self.pc_ratio = cfg['pc_ratio']
        self.match_method = cfg['match_method']
        self.shift_first = cfg['shift_first']
        self.detach_ref_img = cfg['detach_ref_img']
        self.scale_pcs = cfg['scale_pcs']
        self.detach_rgbs_scale = cfg['detach_rgbs_scale']
        self.vis_reprojection_every = cfg['vis_reprojection_every']
        self.nearest_limit = cfg['nearest_limit']
        self.annealing_epochs = cfg['annealing_epochs']
        self.pc_weight = cfg['pc_weight']
        self.rgb_s_weight = cfg['rgb_s_weight']
        self.rgb_weight = cfg['rgb_weight']
        self.depth_weight = cfg['depth_weight']
        self.weight_dist_2nd_loss = cfg['weight_dist_2nd_loss']
        self.weight_dist_1st_loss = cfg['weight_dist_1st_loss']
        self.depth_consistency_weight = cfg['depth_consistency_weight']
        if cfg['depth_loss_type'] not in ('l1', 'invariant'):
            raise ValueError("training.depth_loss_type must be 'l1' or 'invariant' (losses.py:59-64)")
        self.depth_loss_type = cfg['depth_loss_type']     # 'invariant': median / mean-abs-deviation normalised (losses.py:34-57)
        self.loss = Loss(cfg)
        # ---- data parallel (new component, SURVEY.md 8(e)) ----
        self.dp_group = kwargs.get('process_group', None)
        self.dp_mode = kwargs.get('dp_mode', 'rays')        # 'rays': shard one view's rays | 'views': one view per rank
        self.world = 1; self.rank = 0
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            self.world = torch.distributed.get_world_size(self.dp_group)
            self.rank = torch.distributed.get_rank(self.dp_group)
        if self.world > 1 and self.dp_mode == 'rays' and self.n_training_points % self.world != 0:
            raise ValueError("dp_mode='rays': training.n_training_points (%d) must be a multiple of the world size (%d): every rank "
                             "takes ray_idx[rank::world] and the loss normalisation assumes equal shards" % (self.n_training_points, self.world))
        self._gbuf = None
        self._peer = None
        # data-parallel exchange: ONE kernel over NVLink peer memory (all-reduce fused with the Adam updates, captured in the step
        # graph); peer_exchange=False / NNB_PEER_EXCHANGE=0 falls back to torch.distributed.all_reduce between two graphs
        self.peer_exchange = bool(kwargs.get('peer_exchange', os.environ.get('NNB_PEER_EXCHANGE', '1') == '1'))
        self._pix_cache = {}
        # fused flat-buffer Adam (SURVEY.md 8(f) rank 2); optimizers remain the caller's objects
        self.fused_adam = kwargs.get('fused_adam', True)
        self._fadam = {}
        # whole-step CUDA graph for render-only steps (statistically, not stream-, identical pixel/jitter draws)
        self.use_cuda_graph = kwargs.get('use_cuda_graph', os.environ.get('NNB_CUDA_GRAPH', '1') == '1')
        if self.world > 1 and os.environ.get('NNB_GRAPH_DP', '1') != '1':
            self.use_cuda_graph = False      # data parallel: two graphs around an eager NCCL all-reduce (NNB_GRAPH_DP=0 disables)
        self._gsteps = {}
        self.keep_graph = bool(kwargs.get('keep_graph', False))      # keep the cudaGraph_t for introspection (bench.py counts its nodes)
        # 'randperm' = the reference's torch.randperm(H*W)[:N] (identical RNG stream in eager mode); 'hash' = nnb_sample_pixels;
        # 'auto' = randperm when running eagerly, hash inside the CUDA graph (whose RNG stream differs from eager anyway)
        self.pixel_sampler = kwargs.get('pixel_sampler', 'auto')
        self.frame_grad = bool(kwargs.get('frame_grad', False))
        self.frame_grad_engine = _frame_grad_engine(kwargs.get('frame_grad_engine', None), self.frame_grad, "Trainer")
        if self.frame_grad_engine == 'simt':
            if not 2 <= int(model.renderer.cfg['num_points']) <= 1024:
                raise ValueError("Trainer(frame_grad_engine='simt') needs rendering.num_points in 2..1024")
        elif self.frame_grad:
            rend = model.renderer
            engine = rend.engine if rend.engine is not None else ops.default_engine()
            if ops.pick_engine(engine, int(rend.cfg['num_points'])) != L.ENGINE_TC:
                raise ValueError("Trainer(frame_grad=True) needs the tensor-core engine: the renderer's engine and rendering.num_points "
                                 "(16..1024) must resolve to it")
        self.frame_grad_t_min = kwargs.get('frame_grad_t_min', None)
        if self.frame_grad_t_min is not None:
            if not self.frame_grad:
                raise ValueError("Trainer: frame_grad_t_min needs frame_grad=True")
            if self.frame_grad_engine == 'simt':
                raise ValueError("Trainer: frame_grad_t_min runs on the tensor-core pair only (not with frame_grad_engine='simt')")
            ops.frame_render_call(self.frame_grad_t_min)   # ValueError for a negative or NaN value
        self.train_t_min = kwargs.get('train_t_min', None)
        self.train_t_min_engine = kwargs.get('train_t_min_engine', None)
        if self.train_t_min_engine not in (None, 'tc', 'simt'):
            raise ValueError("Trainer: train_t_min_engine must be None, 'tc' or 'simt' (got %r)" % (self.train_t_min_engine,))
        if self.train_t_min_engine is not None and self.train_t_min is None:
            raise ValueError("Trainer: train_t_min_engine needs train_t_min")
        if self.train_t_min_engine is not None and self.frame_grad:
            raise ValueError("Trainer: train_t_min_engine is not taken with frame_grad=True")
        if self.train_t_min is not None and self.train_t_min_engine == 'simt':
            if not 2 <= int(model.renderer.cfg['num_points']) <= 1024:
                raise ValueError("Trainer(train_t_min_engine='simt') needs rendering.num_points in 2..1024")
            ops.exact_stash_render_call(self.train_t_min)   # ValueError for a negative or NaN value
        elif self.train_t_min is not None:
            if self.frame_grad:
                raise ValueError("Trainer: train_t_min is not taken with frame_grad=True (use frame_grad_t_min)")
            rend = model.renderer
            engine = rend.engine if rend.engine is not None else ops.default_engine()
            if ops.pick_engine(engine, int(rend.cfg['num_points'])) != L.ENGINE_TC:
                raise ValueError("Trainer(train_t_min=...) needs the tensor-core engine: the renderer's engine and rendering.num_points "
                                 "(16..1024) must resolve to it")
            ops.stash_render_call(self.train_t_min)   # ValueError for a negative or NaN value

    # ------------------------------------------------------------------------------------
    def _train_render_call(self, backward):
        """the RenderCall class of a training render: the differentiable frame's pair (frame_grad), or the stash pair with early ray
        termination (train_t_min, on the engine train_t_min_engine names), when it has a backward"""
        if backward and self.train_t_min is not None:
            if self.train_t_min_engine == 'simt':
                return ops.exact_stash_render_call(self.train_t_min)
            return ops.stash_render_call(self.train_t_min)
        if not (self.frame_grad and backward):
            return ops.RenderCall
        if self.frame_grad_engine == 'simt':
            return ops.ExactFrameRenderCall
        return ops.FrameRenderCall if self.frame_grad_t_min is None else ops.frame_render_call(self.frame_grad_t_min)

    def _smoothness_on(self):
        """the pose-smoothness terms have a non-zero weight somewhere on their annealing schedule"""
        return any(float(v) != 0.0 for v in list(self.weight_dist_1st_loss) + list(self.weight_dist_2nd_loss))

    def _focal_graphable(self):
        """a LearnFocal module whose fx (and fy) are exactly the parameters of the focal optimizer"""
        fn = self.focal_net
        if fn is None or getattr(fn, 'order', None) not in (1, 2) or not isinstance(getattr(fn, 'fx', None), torch.nn.Parameter):
            return False
        prm = [fn.fx] if fn.fx_only else [fn.fx, getattr(fn, 'fy', None)]
        if any(p is None or p.numel() != 1 or p.dtype != torch.float32 or not p.is_cuda for p in prm):
            return False
        groups = self.optimizer_focal.param_groups
        return len(groups) == 1 and [id(p) for p in groups[0]['params']] == [id(p) for p in prm]

    def _grad_buffer(self, peer_step=False):
        """[MLP (595844 floats at hidden_dim 256) | r 3V | t 3V | scales V | shifts V | [fx, fy, 0, 0] | loss scalars 4], zeroed; the kernels
        accumulate into it.  The focal slot exists only with a learned focal (graph steps install it as the focal parameters' .grad; the
        general path keeps their autograd .grad).
        Installed as every parameter's .grad -- except in a peer-exchange step (data parallel, nnb_allreduce_adam), where .grad
        shows the buffer that receives the SUM over the ranks while the local contributions go to the IPC-shared buffer."""
        V = self.pose_param_net.num_cams if self.pose_param_net is not None else 0
        n_mlp = self.model.renderer.model.num_params
        n_focal = 4 if self.optimizer_focal else 0
        n = n_mlp + 8 * V + n_focal + 4
        dev = self.device
        if self._gbuf is None or self._gbuf.numel() != n:
            if self.peer_exchange and torch.device(dev).type == 'cuda' and (self.world > 1 or self.fused_adam):
                from ..peer import PeerGradExchange, LocalGradExchange
                # world == 1: the exchange kernel degenerates to ONE multi-tensor Adam launch over all parameter groups
                self._peer = PeerGradExchange(n, dev, self.dp_group) if self.world > 1 else LocalGradExchange(n, dev)
                self._gbuf = self._peer.grad
            else:
                self._peer = None
                self._gbuf = torch.zeros(n, device=dev)
        g = self._gbuf
        g.zero_()
        o = n_mlp
        net = self.model.renderer.model
        shown = self._peer.reduced if (peer_step and self._peer is not None) else g

        def split(buf):
            v = {}
            if self.pose_param_net is not None:
                v['r'] = buf[o:o + 3 * V].view(V, 3); v['t'] = buf[o + 3 * V:o + 6 * V].view(V, 3)
            if self.distortion_net is not None:
                v['scales'] = buf[o + 6 * V:o + 7 * V].view(V, 1); v['shifts'] = buf[o + 7 * V:o + 8 * V].view(V, 1)
            if n_focal:
                v['fx'] = buf[o + 8 * V]
                if not getattr(self.focal_net, 'fx_only', True): v['fy'] = buf[o + 8 * V + 1]
            v['losses'] = buf[n - 4:]
            return v
        views = split(g)
        sv = views if shown is g else split(shown)
        if n_focal and peer_step:
            for k in ('fx', 'fy'):
                prm = getattr(self.focal_net, k, None)
                if k in sv and prm.requires_grad: prm.grad = sv[k]
        net.flat_grad(zero=False, alias=shown[:o])
        if self.pose_param_net is not None:
            if self.pose_param_net.r.requires_grad: self.pose_param_net.r.grad = sv['r']
            if self.pose_param_net.t.requires_grad: self.pose_param_net.t.grad = sv['t']
        if self.distortion_net is not None:
            if self.distortion_net.global_scales.requires_grad: self.distortion_net.global_scales.grad = sv['scales']
            if self.distortion_net.global_shifts.requires_grad: self.distortion_net.global_shifts.grad = sv['shifts']
        return g, views

    def train_step(self, data, it=None, epoch=None, scheduling_start=None, render_path=None):
        """training.py:67-97"""
        # (nn.Module.train() walks every submodule: ~60 us of host time per step -- only when the mode actually changes)
        if not self.model.training: self.model.train()
        if self.pose_param_net and not self.pose_param_net.training: self.pose_param_net.train()
        if self.focal_net: self.focal_net.train()
        if self.distortion_net and not self.distortion_net.training: self.distortion_net.train()
        gs = self._graph_step_or_none(data, epoch, scheduling_start)
        if gs is not None:
            return gs[0].run(data, gs[1])          # fixed kernel sequence; replayed as one CUDA graph when use_cuda_graph
        if self.focal_net: self.optimizer_focal.zero_grad()     # (graph steps keep the focal slot of the gradient buffer as .grad)
        loss_dict = self.compute_loss(data, it=it, epoch=epoch, scheduling_start=scheduling_start,
                                      out_render_path=render_path, backward=True)
        self._opt_step(self.optimizer, mlp=True)
        if self.optimizer_pose: self._opt_step(self.optimizer_pose)
        if self.optimizer_focal: self.optimizer_focal.step()
        if self.optimizer_distortion: self._opt_step(self.optimizer_distortion)
        return loss_dict

    def _fadam_for(self, opt, mlp):
        fa = self._fadam.get(id(opt))
        if fa is None:
            if mlp:
                net = self.model.renderer.model
                fa = _FlatAdam(opt, flat_param=net.flat_weights, flat_slices=net.param_slices)
            else:
                fa = _FlatAdam(opt)
            self._fadam[id(opt)] = fa
        return fa

    def _opt_step(self, opt, mlp=False):
        if not self.fused_adam:
            return opt.step()
        self._fadam_for(opt, mlp).step()

    def _graph_step_or_none(self, data, epoch, scheduling_start):
        """fast path: the whole step as one fixed kernel sequence / CUDA graph.  Returns (graph step, device weights) or None for
        configurations that take the general path (no render terms, foreign optimizers or focal modules, invariant depth with the rays
        of one view sharded over ranks -- its median is over the whole batch)."""
        if not self.fused_adam or self.pose_param_net is None or self.distortion_net is None:
            return None
        if (self.optimizer_focal or self.depth_loss_type == 'invariant' or self._smoothness_on()) and not self.use_cuda_graph:
            return None          # eager trainers keep these options on the general path (torch autograd / median / Adam)
        if self.optimizer_focal and not self._focal_graphable():
            return None
        if self.depth_loss_type == 'invariant' and self.world > 1 and self.dp_mode == 'rays':
            return None
        if self.optimizer_pose is None or self.optimizer_distortion is None:
            return None
        names = ['rgb_weight', 'depth_weight', 'pc_weight', 'rgb_s_weight', 'depth_consistency_weight', 'weight_dist_2nd_loss',
                 'weight_dist_1st_loss']
        wts = {n: self.anneal(getattr(self, n)[0], getattr(self, n)[1], scheduling_start, self.annealing_epochs, epoch) for n in names}
        if wts['depth_consistency_weight'] != 0.0 or (wts['rgb_weight'] == 0.0 and wts['depth_weight'] == 0.0):
            return None
        use_ref = wts['pc_weight'] != 0.0 or wts['rgb_s_weight'] != 0.0
        if use_ref:
            self._check_ref_stage_cfg()
            if data.get('img.ref_imgs') is None:
                return None
        rgb_l2 = not (epoch < self.annealing_epochs + scheduling_start)
        img = data.get('img'); dpt = data.get('img.dpt')
        _, _, h, w = img.shape
        hd, wd = dpt.shape[-2:]
        key = (h, w, hd, wd, bool(rgb_l2), bool(use_ref))
        gs = self._gsteps.get(key)
        if gs is None:
            gs = _GraphStep(self, h, w, hd, wd, rgb_l2, use_ref)
            if not gs.eligible_optimizers():
                self._gsteps[key] = False
                return None
            self._gsteps[key] = gs
        if gs is False:
            return None
        inv = self.depth_loss_type == 'invariant'
        w_depth = float(wts['depth_weight'])
        return gs, [float(wts['rgb_weight']), 0.0 if inv else w_depth, float(wts['pc_weight']), float(wts['rgb_s_weight']),
                    float(wts['weight_dist_1st_loss']), float(wts['weight_dist_2nd_loss']), w_depth if inv else 0.0, 0.0]

    def graph_kernel_nodes(self):
        """{kernels, memcpy, memset, other} node counts of the captured step graph(s) (needs Trainer(keep_graph=True)); None if no
        graph has been captured or the CUDA runtime bindings are unavailable"""
        try:
            from cuda.bindings import runtime as rt
        except Exception:
            return None
        tot = {"kernels": 0, "memcpy": 0, "memset": 0, "other": 0}
        found = False
        for gs in self._gsteps.values():
            if not gs or gs.graph is None:
                continue
            for gr in (gs.graph, getattr(gs, 'graph_b', None)):
                if gr is None:
                    continue
                try:
                    raw = gr.raw_cuda_graph()
                    err, _, n = rt.cudaGraphGetNodes(raw, 0)
                    err, nodes, n = rt.cudaGraphGetNodes(raw, n)
                    for nd in nodes[:n]:
                        err, ty = rt.cudaGraphNodeGetType(nd)
                        k = {rt.cudaGraphNodeType.cudaGraphNodeTypeKernel: "kernels", rt.cudaGraphNodeType.cudaGraphNodeTypeMemcpy: "memcpy",
                             rt.cudaGraphNodeType.cudaGraphNodeTypeMemset: "memset"}.get(ty, "other")
                        tot[k] += 1
                    found = True
                except Exception:
                    return None
        return tot if found else None

    def _normal_draw(self, mask):
        """rendering.normal_loss: the reference's renderer draws the neighbour jitter of its surface normals, rand_like of the (valid rays,
        3) surface points, right after the sample jitter (rendering.py:133-141).  Its Loss never reads the normals, so losses and gradients
        are those of normal_loss False; an eager step only makes the same draw, to keep the reference's random stream.  One host read of
        the valid-ray count; the CUDA-graph step does not draw."""
        n_valid = int(mask.sum().item())
        if n_valid > 0:
            torch.rand(n_valid, 3, device=mask.device)

    def _check_ref_stage_cfg(self):
        """the fused reference-image stage (nnb_refstage) covers every option the reference's own Trainer accepts (detach_ref_img and
        with_ssim included); only 'dense' matching exists in the reference"""
        if self.match_method != 'dense':
            raise NotImplementedError("training.match_method=%r: only 'dense' (configs/default.yaml) is fused" % (self.match_method,))

    # ------------------------------------------------------------------------------------
    def process_data_dict(self, data, keep_pinned=False):
        """training.py:164-175.  With keep_pinned, page-locked host frames are NOT copied: a render-only step touches
        N pixels of the 3*H*W frame, which the loss kernel gathers in place over PCIe
        (the reference ships the whole 25 MB frame to the device every step)."""
        device = self.device
        img = data.get('img'); dpt = data.get('img.dpt')
        if not (keep_pinned and img.device.type == 'cpu' and img.is_pinned()):
            img = img.to(device, non_blocking=True)
        dpt = dpt.to(device, non_blocking=True)      # 1 MB; every kernel's ray setup reads it, so it lives in HBM
        img_idx = data.get('img.idx')
        dpt = dpt.unsqueeze(1)
        camera_mat = data.get('img.camera_mat')
        _host_diag_check(camera_mat)
        camera_mat = camera_mat.to(device, non_blocking=True)
        scale_mat = data.get('img.scale_mat')
        return (img, dpt, camera_mat, scale_mat, img_idx)

    def process_data_reference(self, data):
        device = self.device
        ref_imgs = data.get('img.ref_imgs').to(device, non_blocking=True)
        ref_dpts = data.get('img.ref_dpts').to(device, non_blocking=True).unsqueeze(1)
        ref_idxs = data.get('img.ref_idxs')
        return (ref_imgs, ref_dpts, ref_idxs)

    def anneal(self, start_weight, end_weight, anneal_start_epoch, anneal_epoches, current):
        if current <= anneal_start_epoch:
            return start_weight
        elif current >= anneal_start_epoch + anneal_epoches:
            return end_weight
        return start_weight + (end_weight - start_weight) * (current - anneal_start_epoch) / anneal_epoches

    def _pixels(self, res, device):
        key = (tuple(res), str(device))
        if key not in self._pix_cache:
            self._pix_cache[key] = arange_pixels(resolution=res, device=device)
        return self._pix_cache[key]

    # ------------------------------------------------------------------------------------
    def compute_loss(self, data, eval_mode=False, it=None, epoch=None, scheduling_start=None, out_render_path=None,
                     backward=False):
        """training.py:197-378.  With backward=True the gradients of every learnable tensor are
        also produced (into the flat gradient buffer, installed as .grad)."""
        names = ['rgb_weight', 'depth_weight', 'pc_weight', 'rgb_s_weight', 'depth_consistency_weight',
                 'weight_dist_2nd_loss', 'weight_dist_1st_loss']
        weights = {w: self.anneal(getattr(self, w)[0], getattr(self, w)[1], scheduling_start, self.annealing_epochs, epoch)
                   for w in names}
        rgb_loss_type = 'l1' if epoch < self.annealing_epochs + scheduling_start else 'l2'
        render_model = (weights['rgb_weight'] != 0.0) or (weights['depth_weight'] != 0.0)
        use_ref_imgs = (weights['pc_weight'] != 0.0) or (weights['rgb_s_weight'] != 0.0)
        if weights['depth_consistency_weight'] != 0.0:
            raise NotImplementedError("depth_consistency_weight != 0 has no producer in the reference either "
                                      "(training.py never passes d1_proj)")
        n_points = self.n_training_points
        (img, depth_input, camera_mat_gt, scale_mat, img_idx) = self.process_data_dict(data, keep_pinned=not use_ref_imgs)
        img_idx = int(img_idx)
        if use_ref_imgs:
            (ref_img, depth_ref, ref_idx) = self.process_data_reference(data)
            ref_idx = int(ref_idx)
        device = self.device
        _, _, h, w = img.shape
        _, _, h_depth, w_depth = depth_input.shape
        net = self.model.renderer.model
        rend = self.model.renderer
        pose = self.pose_param_net
        V = pose.num_cams
        gbuf, gv = self._grad_buffer() if backward else (None, None)
        losses4 = gv['losses'] if backward else torch.zeros(4, device=device)

        # ---- focal (off by default) -------------------------------------------------------
        fxfy = None
        if self.optimizer_focal:
            fxfy = self.focal_net(0)
            z4 = torch.zeros(4, device=device); one = torch.ones(1, device=device)
            camera_mat = torch.cat([fxfy[0:1], z4, -fxfy[1:2], z4, -one, z4, one]).view(1, 4, 4)   # training.py:247-252
        else:
            camera_mat = camera_mat_gt
        cam_dev = camera_mat.detach().reshape(4, 4).contiguous().float()

        # ---- distortion of the current view (distortions.py:19-27) ------------------------
        if self.distortion_net is not None:
            scale_input, shift_input = self.distortion_net(img_idx)
        else:
            scale_input = torch.ones(1, device=device); shift_input = torch.zeros(1, device=device)
        scale_dev = scale_input.detach().reshape(1).contiguous(); shift_dev = shift_input.detach().reshape(1).contiguous()

        # ---- pixel sampling (training.py:257-262), identical RNG call order to the reference ----
        ray_idx = torch.randperm(h * w, device=device)[:n_points]
        S = int(rend.cfg['num_points'])
        noise = None
        if render_model and rend.cfg['sample_option'] == 'uniform':
            noise = torch.rand(1, n_points, S, device=device)[0]                      # rendering.py:189
        if self.world > 1 and self.dp_mode == 'rays':                                  # shard this view's rays
            ray_idx = ray_idx[self.rank::self.world].contiguous()
            if noise is not None: noise = noise[self.rank::self.world].contiguous()
        n_local = ray_idx.shape[0]
        grad_scale = 1.0 / self.world

        loss_total = torch.zeros((), device=device)
        call = None
        if render_model:
            c2w = torch.empty(4, 4, device=device)
            init = None if pose.init_c2w is None else pose.init_c2w.detach()
            ops.pose_fwd_raw(pose.r.detach(), pose.t.detach(), init, img_idx, c2w)
            flags = ops.flags_from_cfg(rend.cfg, net.occ_activation, eval_=eval_mode, shift_first=self.shift_first)
            ndc = rend.cfg['sample_option'] == 'ndc'
            render_call = self._train_render_call(backward)
            call = render_call(net.flat_weights(), c2w, cam_dev, N=n_local, S=S, flags=flags,
                               engine=rend.engine if rend.engine is not None else ops.default_engine(),
                               near=0.0 if ndc else rend.depth_range[0], far=1.0 if ndc else rend.depth_range[1],
                               ray_idx=ray_idx, depth_map=depth_input.detach().reshape(h_depth, w_depth).contiguous(),
                               scale=scale_dev, shift=shift_dev, noise=noise, H=h, W=w, stash=backward, hidden_dim=net.hidden_dim)
            if rend.cfg.get('normal_loss', False) and not eval_mode:
                self._normal_draw(call.mask)
            inv = self.depth_loss_type == 'invariant' and weights['depth_weight'] != 0.0
            out4, g_rgb, g_dp, g_dg = ops.loss_rgb_depth(call.rgb, call.depth_pred, call.depth_gt, call.mask,
                                                         weights['rgb_weight'], 0.0 if inv else weights['depth_weight'], rgb_loss_type == 'l2',
                                                         img=img.reshape(3, h * w), ray_idx=ray_idx, grad_scale=grad_scale)
            if inv:
                # scale / shift invariant depth term (losses.py:34-57, off by default): a median and two mean-abs-deviations over the
                # N masked rays -- N-element glue, the seeds it yields go through the same fused backward as the L1 seeds
                m = call.mask.bool()
                dpv = call.depth_pred.detach()[m].requires_grad_(True); dgv = call.depth_gt.detach()[m].requires_grad_(True)
                l_inv = self.loss.depth_loss_dpt(dpv, dgv)
                gp_, gg_ = torch.autograd.grad(l_inv * (weights['depth_weight'] * grad_scale), [dpv, dgv])
                g_dp = g_dp.clone(); g_dg = g_dg.clone()
                g_dp[m] += gp_; g_dg[m] += gg_
                out4 = out4.clone(); out4[0] += weights['depth_weight'] * l_inv.detach(); out4[2] = l_inv.detach()
            losses4 += out4 * grad_scale if self.world > 1 else out4
            if backward:
                g_c2w = torch.zeros(4, 4, device=device)
                g_ss = torch.zeros(2, device=device)
                g_cam = torch.zeros(4, 4, device=device) if fxfy is not None else None
                call.backward(g_rgb, g_dp, None if self.detach_gt_depth else g_dg, gbuf[:net.num_params], g_c2w, g_cam, None, g_ss)
                ops.pose_bwd_raw(pose.r.detach(), pose.t.detach(), init, img_idx, g_c2w,
                                 gv['r'] if pose.r.requires_grad else None, gv['t'] if pose.t.requires_grad else None)
                # chain d/d(scale_eff, shift) into global_scales / global_shifts (clamp / fixed-last-view aware)
                outs, gouts = [], []
                if scale_input.requires_grad:
                    outs.append(scale_input); gouts.append(g_ss[0:1].reshape(scale_input.shape))
                if shift_input.requires_grad:
                    outs.append(shift_input); gouts.append(g_ss[1:2].reshape(shift_input.shape))
                if outs:
                    torch.autograd.backward(outs, gouts, retain_graph=use_ref_imgs)   # the distortion module is differentiated again by the reference-image stage
                if g_cam is not None and fxfy.requires_grad:
                    camera_mat.backward(g_cam.view(1, 4, 4), retain_graph=use_ref_imgs)

        ref_terms = {}
        if use_ref_imgs:
            # reference-image stage (training.py:280-365): point-cloud + warped-RGB terms, forward + adjoint in ONE library call
            self._check_ref_stage_cfg()
            _, _, h_depth, w_depth = depth_input.shape
            init = None if pose.init_c2w is None else pose.init_c2w.detach()
            c2w_cur = torch.empty(4, 4, device=device); c2w_ref = torch.empty(4, 4, device=device)
            ops.pose_fwd_raw(pose.r.detach(), pose.t.detach(), init, img_idx, c2w_cur)
            ops.pose_fwd_raw(pose.r.detach(), pose.t.detach(), init, ref_idx, c2w_ref)
            grad_ref = backward and not self.detach_ref_img       # training.py:288-292: gradients into the reference view too
            if self.distortion_net is not None:
                s_ref, h_ref = self.distortion_net(ref_idx)
            else:
                s_ref = torch.ones(1, device=device); h_ref = torch.zeros(1, device=device)
            dist_cur = torch.cat([scale_dev, shift_dev]); dist_ref = torch.stack([s_ref.detach().reshape(()), h_ref.detach().reshape(())]).float()
            rs_losses = torch.zeros(2, device=device); rs_total = torch.zeros(1, device=device)
            g_c2w_rs = torch.zeros(4, 4, device=device) if backward else None
            g_ss_rs = torch.zeros(2, device=device) if backward else None
            g_kxy_rs = torch.zeros(2, device=device) if (backward and fxfy is not None) else None
            g_c2w_ref_rs = torch.zeros(4, 4, device=device) if grad_ref else None
            g_ss_ref_rs = torch.zeros(2, device=device) if grad_ref else None
            ops.refstage_raw(c2w_cur, dist_cur, c2w_ref, dist_ref, depth_input.detach().reshape(h_depth, w_depth).contiguous(),
                             depth_ref.detach().reshape(h_depth, w_depth).contiguous(), H=h, W=w, img_cur=ops._f32c(img[0]), img_ref=ops._f32c(ref_img[0]),
                             is_last=(img_idx == V - 1), cam=cam_dev, nearest_limit=self.nearest_limit, pc_ratio=self.pc_ratio,
                             scale_pcs=self.scale_pcs, detach_rgbs_scale=self.detach_rgbs_scale, shift_first=self.shift_first,
                             w_pc=weights['pc_weight'], w_rgb_s=weights['rgb_s_weight'], losses=rs_losses, g_c2w=g_c2w_rs, g_dist=g_ss_rs,
                             g_kxy=g_kxy_rs, loss_total=rs_total, grad_scale=grad_scale, with_ssim=bool(self.loss.cfg.get('with_ssim', False)),
                             g_c2w_ref=g_c2w_ref_rs, g_dist_ref=g_ss_ref_rs)
            if weights['pc_weight'] != 0.0: ref_terms['loss_pc'] = rs_losses[0]
            if weights['rgb_s_weight'] != 0.0: ref_terms['loss_rgb_s'] = rs_losses[1]
            loss_total = loss_total + rs_total[0]
            if backward:
                ops.pose_bwd_raw(pose.r.detach(), pose.t.detach(), init, img_idx, g_c2w_rs,
                                 gv['r'] if pose.r.requires_grad else None, gv['t'] if pose.t.requires_grad else None)
                outs, gouts = [], []
                if scale_input.requires_grad:
                    outs.append(scale_input); gouts.append(g_ss_rs[0:1].reshape(scale_input.shape))
                if shift_input.requires_grad:
                    outs.append(shift_input); gouts.append(g_ss_rs[1:2].reshape(shift_input.shape))
                if outs:
                    torch.autograd.backward(outs, gouts)
                if g_kxy_rs is not None and fxfy.requires_grad:
                    fxfy.backward(torch.stack([g_kxy_rs[0], -g_kxy_rs[1]]))          # camera_mat = diag(fx, -fy, -1, 1)
                if grad_ref:
                    ops.pose_bwd_raw(pose.r.detach(), pose.t.detach(), init, ref_idx, g_c2w_ref_rs,
                                     gv['r'] if pose.r.requires_grad else None, gv['t'] if pose.t.requires_grad else None)
                    # through Learn_Distortion(ref_idx): its clamp and the fixed scale of the last view leave constants without a gradient
                    outs, gouts = [], []
                    if s_ref.requires_grad:
                        outs.append(s_ref); gouts.append(g_ss_ref_rs[0:1].reshape(s_ref.shape))
                    if h_ref.requires_grad:
                        outs.append(h_ref); gouts.append(g_ss_ref_rs[1:2].reshape(h_ref.shape))
                    if outs:
                        torch.autograd.backward(outs, gouts)

        # pose-smoothness terms (losses.py:103-112, weight 0 by default): every rank holds the same t, so each contributes
        # 1/world of the gradient BEFORE the all-reduce sums the ranks
        dist_terms = None
        if weights['weight_dist_2nd_loss'] != 0.0 or weights['weight_dist_1st_loss'] != 0.0:
            d1, d2 = self.loss.get_weight_dist_loss(pose.get_t())
            extra = weights['weight_dist_1st_loss'] * d1 + weights['weight_dist_2nd_loss'] * d2
            if backward: (extra * grad_scale).backward()
            dist_terms = (d1.detach(), d2.detach(), extra.detach())
        # ---- data-parallel: ONE all-reduce of [grads | loss scalars] -----------------------
        if backward and self.world > 1:
            torch.distributed.all_reduce(gbuf, group=self.dp_group)
            if self.optimizer_focal:         # focal gradients (2 floats, off by default) live outside the flat buffer
                for p_ in self.focal_net.parameters():
                    if p_.grad is not None: torch.distributed.all_reduce(p_.grad, group=self.dp_group)
        zero = torch.zeros((), device=device)
        loss_dict = {'loss': losses4[0] + loss_total, 'loss_rgb': losses4[1], 'loss_depth': losses4[2], 'l2_mean': losses4[3],
                     'loss_dist_1st': zero, 'loss_dist_2nd': zero, 'loss_pc': ref_terms.get('loss_pc', zero),
                     'loss_rgb_s': ref_terms.get('loss_rgb_s', zero), 'loss_depth_consistency': zero}
        if dist_terms is not None:
            loss_dict['loss_dist_1st'], loss_dict['loss_dist_2nd'] = dist_terms[0], dist_terms[1]
            loss_dict['loss'] = loss_dict['loss'] + dist_terms[2]
        if self.optimizer_focal:
            loss_dict['focalx'] = fxfy[0] / camera_mat_gt[0, 0, 0]
            loss_dict['focaly'] = fxfy[1] / camera_mat_gt[0, 1, 1]
        loss_dict['scale'] = scale_input.detach()     # logging values (training.py:376-377)
        loss_dict['shift'] = shift_input.detach()
        if call is not None and not backward:
            call.release()
        return loss_dict

    # ------------------------------------------------------------------------------------
    def render_visdata(self, data, resolution, it, out_render_path):
        """training.py:100-163: the volumetric view and, with training.vis_geo, the phong-shaded geometry view."""
        (img, dpt, camera_mat, scale_mat, img_idx) = self.process_data_dict(data)
        h, w = resolution
        c2w = self.pose_param_net(int(img_idx)).detach()
        world_mat = torch.linalg.inv(c2w).unsqueeze(0)
        if self.optimizer_focal:
            fxfy = self.focal_net(0).detach()
            camera_mat = torch.diag(torch.stack([fxfy[0], -fxfy[1], -torch.ones((), device=self.device),
                                                 torch.ones((), device=self.device)])).unsqueeze(0)
        p_idx = torch.arange(h * w, device=self.device)
        _, pixels = self._pixels((h, w), self.device)
        with torch.no_grad():
            out = self.model(pixels, p_idx, camera_mat, world_mat, scale_mat, self.rendering_technique, add_noise=False,
                             eval_mode=True, it=it, depth_img=dpt, img_size=(h, w))
            rgb_pred = out['rgb'].view(h, w, 3).cpu().numpy()
            depth = out['depth_pred'].view(h, w).cpu().numpy()
        img_out = (rgb_pred * 255).astype(np.uint8)
        if out_render_path is not None:
            from PIL import Image
            dn = np.clip(255.0 / depth.max() * (depth - depth.min()), 0, 255).astype(np.uint8)
            Image.fromarray(dn).save(os.path.join(out_render_path, '%04d_depth.png' % int(img_idx)))
            Image.fromarray(img_out).convert("RGB").save(os.path.join(out_render_path, '%04d_img.png' % int(img_idx)))
        if self.vis_geo:       # training.py:146-161: the shaded geometry view is what render_visdata returns when it is on
            # Renderer(geometry_frame=True): the whole frame in one call (its rays do not depend on the chunk)
            chunk = pixels.shape[1] if getattr(self.model.renderer, 'geometry_frame', False) else GEOMETRY_CHUNK
            with torch.no_grad():
                geo = torch.cat([self.model(px, None, camera_mat, world_mat, scale_mat, 'phong_renderer', add_noise=False, eval_mode=True,
                                            it=it, depth_img=dpt, img_size=(h, w))['rgb']
                                 for px in torch.split(pixels, chunk, dim=1)], dim=1)
            img_out = (geo.view(h, w, 3).cpu().numpy() * 255).astype(np.uint8)
            if out_render_path is not None:
                from PIL import Image
                Image.fromarray(img_out).convert("RGB").save(os.path.join(out_render_path, '%04d_geo.png' % int(img_idx)))
        return img_out

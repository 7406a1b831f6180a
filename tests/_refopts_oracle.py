"""numpy oracle of the reference-image stage with the two non-default options of the reference's configs/default.yaml that the fused
stage also covers: `training.detach_ref_img: False` (gradients into the reference view's pose and distortion, training.py:280-293)
and `training.with_ssim: True` (warped-RGB loss 0.15 * L1 + 0.85 * SSIM, losses.py:150-157, 222-253).  It extends
oracle.ref_stage / oracle.train_step and reduces to them with both options at their defaults (tests/test_refopts_golden.py checks
that, and pins this module to reference Trainer steps, tests/golden/train_full_{ssim,undetached}*.npz from tools/make_golden.py).

SSIM layout: training.py:338-343 hands Loss channel-last (1, rh, rw, 3) tensors, so the SSIM module treats the rh rows as channels
and slides its 3x3 windows over (column, colour channel) inside one low-resolution row, with reflection padding of both axes."""
import numpy as np
from oracle import nerf_oracle as O

SSIM_C1, SSIM_C2 = 0.01 ** 2, 0.03 ** 2


def _pad(a):
    """ReflectionPad2d(1) of the (column, channel) axes of a (rh, rw, 3) array"""
    return np.pad(a, ((0, 0), (1, 1), (1, 1)), mode="reflect")


def _pad_adj(gp):
    """adjoint of _pad: (rh, rw + 2, 5) -> (rh, rw, 3); a reflected entry adds into its source"""
    g = gp[:, 1:-1, 1:-1].copy()
    g[:, 1, :] += gp[:, 0, 1:-1]; g[:, -2, :] += gp[:, -1, 1:-1]
    g[:, :, 1] += gp[:, 1:-1, 0]; g[:, :, -2] += gp[:, 1:-1, -1]
    g[:, 1, 1] += gp[:, 0, 0]; g[:, 1, -2] += gp[:, 0, -1]; g[:, -2, 1] += gp[:, -1, 0]; g[:, -2, -2] += gp[:, -1, -1]
    return g


def _box(ap):
    """AvgPool2d(3, 1) of a padded array: (rh, rw + 2, 5) -> (rh, rw, 3)"""
    rw, nc = ap.shape[1] - 2, ap.shape[2] - 2
    s = sum(ap[:, i:i + rw, j:j + nc] for i in range(3) for j in range(3))
    return s / ap.dtype.type(9)


def _box_adj(g):
    rh, rw, nc = g.shape
    out = np.zeros((rh, rw + 2, nc + 2), g.dtype)
    for i in range(3):
        for j in range(3):
            out[:, i:i + rw, j:j + nc] += g / g.dtype.type(9)
    return out


def ssim_map(x, y, g_map=None):
    """class SSIM (losses.py:222-253) on channel-last (rh, rw, 3) arrays: clamp((1 - SSIM) / 2, 0, 1).  With g_map (the cotangent of
    the map) also returns d / d y (y = the warped image, the only input with a gradient)."""
    dt = x.dtype.type
    c1, c2 = dt(SSIM_C1), dt(SSIM_C2)
    xp, yp = _pad(x), _pad(y)
    mx, my = _box(xp), _box(yp)
    sx = _box(xp * xp) - mx * mx; sy = _box(yp * yp) - my * my; sxy = _box(xp * yp) - mx * my
    a1 = dt(2) * mx * my + c1; a2 = dt(2) * sxy + c2
    b1 = mx * mx + my * my + c1; b2 = sx + sy + c2
    s = a1 * a2 / (b1 * b2)
    raw = (dt(1) - s) / dt(2)
    m = np.clip(raw, dt(0), dt(1))
    if g_map is None:
        return m
    gs = np.where((raw >= 0) & (raw <= 1), g_map, dt(0)) * dt(-0.5)
    d_my = gs * (dt(2) * mx * a2 / (b1 * b2) - s * dt(2) * my / b1)
    d_sy = gs * (-s / b2)
    d_sxy = gs * (dt(2) * a1 / (b1 * b2))
    g_mean = d_my - dt(2) * my * d_sy - mx * d_sxy                   # coefficients of E[y], E[y^2], E[xy] of each window
    gyp = _box_adj(g_mean) + dt(2) * yp * _box_adj(d_sy) + xp * _box_adj(d_sxy)
    return m, _pad_adj(gyp)


def ref_stage(img, ref_img, d_in_raw, d_ref_raw, c2w, c2w_ref, scale_in, shift_in, scale_ref, shift_ref, is_last, kx, ky,
              w_pc=1.0, w_rgb_s=1.0, cfg=O.REF_CFG):
    """oracle.ref_stage plus cfg['detach_ref_img'] (default True) and cfg['with_ssim'] (default False).  Returns (losses, grads); with
    detach_ref_img False, grads also holds c2w_ref (4,4), scale_ref and shift_ref: the gradients w.r.t. the reference view's pose
    matrix and effective distortion."""
    dt = img.dtype.type
    nl = dt(cfg["nearest_limit"])
    detach_ref = bool(cfg.get("detach_ref_img", True)); with_ssim = bool(cfg.get("with_ssim", False))
    hd, wd = d_in_raw.shape
    res = (int(hd / cfg["pc_ratio"]), int(wd / cfg["pc_ratio"]))
    ys, xs = np.meshgrid(np.arange(res[0]), np.arange(res[1]), indexing="ij")
    px = (dt(2) * xs.reshape(-1).astype(img.dtype) / dt(res[1] - 1) - dt(1)); py = (dt(2) * ys.reshape(-1).astype(img.dtype) / dt(res[0] - 1) - dt(1))
    raw_in, _, _ = O.nearest_resize(d_in_raw, res); raw_ref, _, _ = O.nearest_resize(d_ref_raw, res)
    raw_in = raw_in.reshape(-1).astype(img.dtype); raw_ref = raw_ref.reshape(-1).astype(img.dtype)
    shift_first = bool(cfg.get("shift_first", False))
    if shift_first:
        din = (raw_in + dt(shift_in)) * dt(scale_in); dref = (raw_ref + dt(shift_ref)) * dt(scale_ref)
    else:
        din = raw_in * dt(scale_in) + dt(shift_in); dref = raw_ref * dt(scale_ref) + dt(shift_ref)
    live_in = din >= nl; live_ref = dref >= nl
    din_c = np.where(live_in, din, nl); dref_c = np.where(live_ref, dref, nl)
    bp = lambda d: np.stack([px * d / dt(kx), py * d / dt(ky), -d], -1)
    c2w = c2w.astype(img.dtype); c2w_ref = c2w_ref.astype(img.dtype)
    if not is_last:
        d1, d2 = din_c, dref_c; img1, img2 = img, ref_img
        M = np.linalg.inv(c2w_ref) @ c2w
        s2 = dt(scale_ref)
    else:
        d1, d2 = dref_c, din_c; img1, img2 = ref_img, img
        M = np.linalg.inv(c2w) @ c2w_ref
        s2 = dt(scale_in)
    M = M.astype(img.dtype)
    R, t = M[:3, :3], M[:3, 3]
    pc1, pc2 = bp(d1), bp(d2)
    g_pc1 = np.zeros_like(pc1); g_pc2 = np.zeros_like(pc2); gR = np.zeros((3, 3), img.dtype); gt = np.zeros(3, img.dtype)
    g_s2 = dt(0)
    g_kxy = np.zeros(2, img.dtype)
    losses = dict(loss_pc=dt(0), loss_rgb_s=dt(0))
    if w_rgb_s != 0.0:
        i1, i2 = O.bilinear_resize(img1, res), O.bilinear_resize(img2, res)
        rgb1 = O.grid_sample_bilinear(i1, np.stack([px, py], -1))
        Xr = pc1 @ R.T + t
        bad = (-Xr[:, 2] < nl)
        Xr_c = np.where(bad[:, None], nl, Xr)
        z = -Xr_c[:, 2]
        xy = np.stack([dt(kx) * Xr_c[:, 0] / z, dt(ky) * Xr_c[:, 1] / z], -1)
        valid = np.abs(xy).max(-1) <= 1
        nv = int(valid.sum()) * 3
        rgb2 = O.grid_sample_bilinear(i2, xy)
        diff = rgb1 - rgb2
        ad = np.clip(np.abs(diff), 0, 1)
        if with_ssim:
            shp = (res[0], res[1], 3)
            sm = ssim_map(rgb1.reshape(shp), rgb2.reshape(shp)).reshape(-1, 3)
            ad = dt(0.15) * ad + dt(0.85) * sm
        losses["loss_rgb_s"] = ad[valid].sum() / dt(max(nv, 1)) if nv > 0 else dt(0)
        if nv > 0:
            g_proj = np.where(valid[:, None] & (np.abs(diff) < 1), -np.sign(diff), dt(0)) * dt(w_rgb_s) / dt(nv)
            if with_ssim:
                g_map = np.where(np.repeat(valid[:, None], 3, 1), dt(0.85) * dt(w_rgb_s) / dt(nv), dt(0)).reshape(shp)
                _, g_y = ssim_map(rgb1.reshape(shp), rgb2.reshape(shp), g_map)
                g_proj = dt(0.15) * g_proj + g_y.reshape(-1, 3)      # the SSIM windows also read invalid points
            _, g_xy = O.grid_sample_bilinear(i2, xy, g_proj)
            gX = np.stack([g_xy[:, 0] * dt(kx) / z, g_xy[:, 1] * dt(ky) / z,
                           (g_xy[:, 0] * dt(kx) * Xr_c[:, 0] + g_xy[:, 1] * dt(ky) * Xr_c[:, 1]) / (z * z)], -1)
            gX = np.where(bad[:, None], dt(0), gX)
            g_kxy += np.array([(g_xy[:, 0] * Xr_c[:, 0] / z).sum(), (g_xy[:, 1] * Xr_c[:, 1] / z).sum()], img.dtype)
            gR += gX.T @ pc1; gt += gX.sum(0)
            if not cfg["detach_rgbs_scale"]:
                g_pc1 += gX @ R
    if w_pc != 0.0:
        X = pc1 @ R.T + t; Y = pc2
        if cfg["scale_pcs"]:
            Xs, Ys = X / s2, Y / s2
        else:
            Xs, Ys = X, Y
        l, gXs, gYs, _, _ = O.chamfer(Xs, Ys)
        losses["loss_pc"] = l
        gXs = gXs * dt(w_pc); gYs = gYs * dt(w_pc)
        if cfg["scale_pcs"]:
            g_s2 = -((gXs * Xs).sum() + (gYs * Ys).sum()) / s2
            gX, gY = gXs / s2, gYs / s2
        else:
            gX, gY = gXs, gYs
        gR += gX.T @ pc1; gt += gX.sum(0); g_pc1 += gX @ R; g_pc2 += gY
    gM = np.zeros((4, 4), img.dtype); gM[:3, :3] = gR; gM[:3, 3] = gt
    proj = lambda g: g[:, 0] * px / dt(kx) + g[:, 1] * py / dt(ky) - g[:, 2]       # d / d depth of a back-projected cloud
    inv_ref, inv_cur = np.linalg.inv(c2w_ref), np.linalg.inv(c2w)
    if not is_last:                                                               # M = inv(A) C, A = c2w_ref, C = c2w
        g_c2w = inv_ref.T @ gM
        g_c2w_ref = -(inv_ref.T @ (gM @ c2w.T) @ inv_ref.T)
        g_d, g_dr = proj(g_pc1), proj(g_pc2)
        g_scale_extra, g_scale_ref_extra = dt(0), g_s2                            # scale2 = the reference view's scale
    else:                                                                         # M = inv(C) A
        g_c2w = -(inv_cur.T @ (gM @ c2w_ref.T) @ inv_cur.T)
        g_c2w_ref = inv_cur.T @ gM
        g_d, g_dr = proj(g_pc2), proj(g_pc1)
        g_scale_extra, g_scale_ref_extra = g_s2, dt(0)
    g_d = np.where(live_in, g_d, dt(0)); g_dr = np.where(live_ref, g_dr, dt(0))
    g_kxy += np.array([-((g_pc1[:, 0] * pc1[:, 0]).sum() + (g_pc2[:, 0] * pc2[:, 0]).sum()) / dt(kx),
                       -((g_pc1[:, 1] * pc1[:, 1]).sum() + (g_pc2[:, 1] * pc2[:, 1]).sum()) / dt(ky)], img.dtype)
    if shift_first:
        g_scale, g_shift = (g_d * (raw_in + dt(shift_in))).sum(), (g_d * dt(scale_in)).sum()
        g_scale_r, g_shift_r = (g_dr * (raw_ref + dt(shift_ref))).sum(), (g_dr * dt(scale_ref)).sum()
    else:
        g_scale, g_shift = (g_d * raw_in).sum(), g_d.sum()
        g_scale_r, g_shift_r = (g_dr * raw_ref).sum(), g_dr.sum()
    grads = dict(c2w=g_c2w.astype(img.dtype), scale=g_scale + g_scale_extra, shift=g_shift, kxy=g_kxy)
    if not detach_ref:
        grads.update(c2w_ref=g_c2w_ref.astype(img.dtype), scale_ref=g_scale_r + g_scale_ref_extra, shift_ref=g_shift_r)
    return losses, grads


def train_step(state, img, dpt, ray_idx, noise, cam_id, kx, ky, cfg, ref, refcfg, w_rgb=1.0, w_depth=0.04, lrs=(1e-3, 5e-4, 5e-4)):
    """oracle.train_step (render + rgb L1 + depth L1 + reference-image stage, Adam x3) with the options of `refcfg` (REF_CFG keys plus
    shift_first, detach_ref_img, with_ssim); shift_first also applies to the render path's depth (training.py:241-245).  With
    detach_ref_img False the reference view's rows of r, t, scales, shifts receive gradients too."""
    P = state["P"]; dt = img.dtype.type
    H, W = img.shape[1:]
    V = state["r"].shape[0]
    shift_first = bool(refcfg.get("shift_first", False))
    ri = int(ref["idx"])
    c2w = O.make_c2w(state["r"][cam_id], state["t"][cam_id])
    c2w_ref = O.make_c2w(state["r"][ri], state["t"][ri])
    scale_eff, shift, live = O._distortion(state, cam_id, dt, cfg)
    s_ref, h_ref, live_ref = O._distortion(state, ri, dt, cfg)
    raw, _ = O.gather_prior_depth(dpt, ray_idx, H, W)
    depth = (raw + shift) * scale_eff if shift_first else raw * scale_eff + shift
    pixels = O.pixels_from_idx(ray_idx, H, W, dt)
    rgb_gt = img.reshape(3, -1)[:, ray_idx].T
    out, cache = O.render_forward(P, pixels, depth.astype(img.dtype), c2w, kx, ky, cfg, noise=noise)
    ld, g_rgb, g_dp, g_dg = O.loss_rgb_depth(out["rgb"], rgb_gt, out["depth_pred_full"], out["depth_gt_full"], out["mask"], w_rgb, w_depth, "l1")
    gr = O.render_backward(P, cache, g_rgb, g_dp, g_dg)
    g_c2w = gr["c2w"]
    if shift_first:
        g_scale, g_shift = (gr["depth"] * (raw + shift)).sum(), (gr["depth"] * scale_eff).sum()
    else:
        g_scale, g_shift = (gr["depth"] * raw).sum(), gr["depth"].sum()
    g_scale = g_scale if live else dt(0)
    w_pc, w_rgb_s = ref.get("w_pc", 1.0), ref.get("w_rgb_s", 1.0)
    rl, rg = ref_stage(img, ref["img"], dpt, ref["dpt"], c2w, c2w_ref, scale_eff, shift, s_ref, h_ref, cam_id == V - 1, kx, ky,
                       w_pc=w_pc, w_rgb_s=w_rgb_s, cfg=refcfg)
    ld["loss_pc"] = rl["loss_pc"]; ld["loss_rgb_s"] = rl["loss_rgb_s"]
    ld["loss"] = ld["loss"] + dt(w_pc) * rl["loss_pc"] + dt(w_rgb_s) * rl["loss_rgb_s"]
    g_c2w = g_c2w + rg["c2w"]
    g_scale = g_scale + (rg["scale"] if live else dt(0)); g_shift = g_shift + rg["shift"]
    G = {k: np.zeros_like(state[k]) for k in ("r", "t", "scales", "shifts")}
    G["r"][cam_id], G["t"][cam_id] = O.make_c2w_bwd(state["r"][cam_id], state["t"][cam_id], None, g_c2w)
    G["scales"][cam_id, 0] = g_scale; G["shifts"][cam_id, 0] = g_shift
    if "c2w_ref" in rg:
        gr_r, gr_t = O.make_c2w_bwd(state["r"][ri], state["t"][ri], None, rg["c2w_ref"])
        G["r"][ri] += gr_r; G["t"][ri] += gr_t
        G["scales"][ri, 0] += rg["scale_ref"] if live_ref else dt(0); G["shifts"][ri, 0] += rg["shift_ref"]
    state["step"] = state.get("step", 0) + 1
    ad = state.setdefault("adam", {})
    for n in O.PARAM_NAMES:
        m = ad.setdefault("m." + n, np.zeros_like(P[n])); v = ad.setdefault("v." + n, np.zeros_like(P[n]))
        O.adam_step(P[n], gr["params"][n].astype(P[n].dtype), m, v, state["step"], lrs[0])
    for key, lr in (("r", lrs[1]), ("t", lrs[1]), ("scales", lrs[2]), ("shifts", lrs[2])):
        m = ad.setdefault("m." + key, np.zeros_like(state[key])); v = ad.setdefault("v." + key, np.zeros_like(state[key]))
        O.adam_step(state[key], G[key], m, v, state["step"], lr)
    return ld, dict(P=gr["params"], **G)

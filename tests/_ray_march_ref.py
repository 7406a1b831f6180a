"""numpy restatement of Renderer.ray_marching's bracket search and Renderer.secant on given values: every product, sum and quotient is
one float32 numpy operation, i.e. rounded on its own like the torch code's.  tests/test_ray_march_ref.py pins it against the torch body;
tests/test_gpu_ray_march.py uses it for the outputs the torch body does not return (first, bracket)."""
import numpy as np


def depths(near, far, frac):
    """t [N, S] = near (1 - frac) + far frac in float32"""
    frac = frac.astype(np.float32)[None, :]
    return np.float32(near) * (np.float32(1) - frac) + far.astype(np.float32)[:, None] * frac


def first_and_bracket(val, t):
    """val, t [N, S] float32 -> first [N] (index of the first negative rounded product val[i] val[i+1], -1 if none), hit [N],
    v0neg [N], bracket [N, 4] = (d_low, d_high, f_low, f_high) (meaningful where hit)"""
    N, S = val.shape
    neg = (val[:, :-1] * val[:, 1:]) < 0
    has = neg.any(1)
    first = np.where(has, neg.argmax(1), -1).astype(np.int32)
    ar = np.arange(N)
    lo = np.maximum(first, 0)
    hi = np.minimum(lo + 1, S - 1)
    v0neg = val[:, 0] < 0
    hit = has & (val[ar, lo] < 0) & v0neg
    bracket = np.stack([t[ar, lo], t[ar, hi], val[ar, lo], val[ar, hi]], 1).astype(np.float32)
    return first, hit, v0neg, bracket


def secant(bracket, n_secant, f_mid_of):
    """n_secant steps on bracket [K, 4]; f_mid_of(d [K] float32) -> occupancy - tau at depth d of each ray.  Returns d [K]"""
    d_low, d_high, f_low, f_high = (bracket[:, i].copy() for i in range(4))
    step = lambda: -f_low * (d_high - d_low) / (f_high - f_low) + d_low
    d = step()
    for _ in range(n_secant):
        f_mid = f_mid_of(d).astype(np.float32)
        low = f_mid < 0
        d_low = np.where(low, d, d_low); f_low = np.where(low, f_mid, f_low)
        d_high = np.where(low, d_high, d); f_high = np.where(low, f_high, f_mid)
        d = step()
    return d.astype(np.float32)


def depth_out(hit, v0neg, d_hit):
    """the march's output encoding: refined depth on a hit, inf without one, 0 where the first sample is occupied"""
    out = np.full(hit.shape, np.inf, np.float32)
    out[hit] = d_hit
    out[~v0neg] = 0
    return out

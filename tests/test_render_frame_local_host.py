"""Host side of test_gpu_render_frame_local.py (no device): the Python mirror of the frame backward's workspace layout, the float64
end-to-end reference against the numpy oracle, the wrong answers of the reverse rounds on host data, and the planting of translucent and
scattered fields."""
import numpy as np
import pytest
import torch

from nope_nerf_b200 import _lib as L
from oracle import nerf_oracle as O
import test_gpu_ray_local as RL
import test_gpu_render_frame_local as FL

REF_GATE = 1e-12   # the float64 reference against the numpy oracle, |a - b|max / |b|max per tensor


def test_layout_mirror_matches_the_library():
    for engine, e in (("tc", L.ENGINE_TC), ("simt", L.ENGINE_SIMT)):
        for N in (1, 3, 5, 127, 4096):
            for S in (2, 15, 16, 31, 32, 33, 48, 1000, 1024):
                if engine == "tc" and S < 16:
                    continue
                for D in L.HIDDEN_DIMS:
                    assert FL.frame_layout(N, S, D, engine)["total"] == L.lib.nnb_render_frame_bwd_workspace_bytes_engine(N, S, D, e), \
                        (engine, N, S, D)


def _host_case(name, S=None, N=5, D=64, seed=1, noise=True):
    c = dict(FL.CASES[name])
    if S is not None:
        c["S"] = S
    c["N"] = N
    inp = FL.inputs(name, seed, case=c)
    flags = FL._flags(c)
    P = O.init_params(seed=7, D=D, hf_damp=True, dtype=np.float64)
    if not noise or flags & L.NDC:
        inp["noise"] = None
    return inp, flags, P, D


def _oracle(P, inp, flags):
    """numpy oracle forward + backward in float64 at the case's inputs"""
    cfg = FL._cfg(flags, inp["S"])
    pix = O.pixels_from_idx(inp["ray_idx"], FL.H, FL.W, np.float64)
    depth = inp["depth"].astype(np.float64) if "depth" in inp else inp["raw"].astype(np.float64) * float(inp["scale"]) + float(inp["shift"])
    kx, ky = float(inp["cam"][0, 0]), float(inp["cam"][1, 1])
    out, cache = O.render_forward(P, pix, depth, inp["c2w"].astype(np.float64), kx, ky, cfg,
                                  noise=None if inp["noise"] is None else inp["noise"].astype(np.float64), eval_=bool(flags & L.EVAL))
    g = O.render_backward(P, cache, inp["g_rgb"].astype(np.float64), inp["g_dp"].astype(np.float64), inp["g_dg"].astype(np.float64))
    return out, cache, g


def _gates(cache):
    mc = cache["mcache"]
    g = [torch.from_numpy((y > 0).astype(np.float64)) for y in mc["Y"]] + [torch.from_numpy((mc["yr"] > 0).astype(np.float64))]
    return g, torch.from_numpy((mc["s"] > 0).astype(np.float64))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize("name,S,noise", [("t33", 33, True), ("t33", 33, False), ("t100", 100, True), ("t100-ndc", 100, False),
                                          ("t48-dist", 33, True), ("t100-white", 100, True), ("t100-eval", 100, False),
                                          ("t100-depth", 100, True), ("t100-relu-dist", 33, True), ("t100-nonorm", 33, True)])
def test_reference_matches_oracle(name, S, noise):
    """the float64 autograd reference (test_gpu_ray_local's ray and compositing references, the MLP with fixed gates) equals the numpy
    oracle's render_forward / render_backward, given the oracle's own ReLU gates"""
    inp, flags, P, D = _host_case(name, S, noise=noise)
    out, cache, g = _oracle(P, inp, flags)
    gates, s_gate = _gates(cache)
    outs, G, wrong, T = FL.reference(P, inp, flags, gates, s_gate, inp["noise"], dev="cpu")
    assert _rel(outs["rgb"], out["rgb"]) <= REF_GATE
    assert _rel(outs["depth_pred"], out["depth_pred_full"]) <= REF_GATE
    assert _rel(outs["depth_gt"], out["depth_gt_full"]) <= REF_GATE
    for k in O.PARAM_NAMES:
        assert _rel(G[k], g["params"][k]) <= REF_GATE, k
    assert _rel(G["g_c2w"][:3], g["c2w"][:3]) <= REF_GATE
    assert _rel([G["g_cam"][0, 0], G["g_cam"][1, 1]], g["kxy"]) <= REF_GATE
    if "depth" in inp:
        assert _rel(G["g_depth"], g["depth"]) <= REF_GATE
    else:   # depth = raw scale + shift
        gd = g["depth"]
        assert _rel([G["g_scale"], G["g_shift"]], [(gd * inp["raw"]).sum(), gd.sum()]) <= REF_GATE
    assert _rel(T[:, 1:].numpy(), np.cumprod(cache["om"], 1)) <= REF_GATE


@pytest.mark.parametrize("name,S", [("t33", 33), ("t100", 100), ("t48-dist", 48), ("t100-depth", 100)])
def test_wrong_answers_on_translucent_host_data(name, S):
    """on a translucent host field every wrong answer of the reverse rounds moves some gradient by at least 10x the largest end-to-end
    gate; dropping the rounds k >= 1 moves every non-zero dW tensor that much"""
    inp, flags, P, D = _host_case(name, S, N=37)
    s, z = FL.oracle_logits(P, inp, flags)
    P = FL.plant(P, s, z, flags, "translucent")
    P = {k: np.asarray(v, np.float64) for k, v in P.items()}
    out, cache, g = _oracle(P, inp, flags)
    gates, s_gate = _gates(cache)
    outs, G, wrong, T = FL.reference(P, inp, flags, gates, s_gate, inp["noise"], dev="cpu")
    FL._check_coverage("t33" if S == 33 else name, T) if S == FL.CASES[name]["S"] else None
    ref = FL._grad_tensors(G)
    gate = FL.E2E_GATES["translucent"]["tc"]
    for bug in FL.BUGS:
        if not FL._applies(bug, inp, flags):
            continue
        w = FL._grad_tensors(wrong(bug))
        sc = {k: _rel(w[k], ref[k]) if float(ref[k].abs().max()) > 0 else 0.0 for k in ref}
        print(name, bug, "%.3g" % max(sc.values()))
        if bug not in FL.REPORT_ONLY:   # frame_ray_acc's answers: scored on the rayacc stage below
            assert max(sc.values()) >= 10 * gate, (name, bug, sc)
        if bug == "drop_late" and S > 33:
            low = {k: v for k, v in sc.items() if k in O.PARAM_NAMES and float(ref[k].abs().max()) > 0 and v < 10 * gate}
            assert not low, (name, low)


@pytest.mark.parametrize("S", [48, 256, 1024])
def test_planting_puts_the_field_in_band(S):
    """the translucent planting puts the oracle's float64 transmittance into the last chunk at 0.05 .. 0.6 for every ray, and the
    scattered planting at the scattered cases' sizes makes rays lose their transmittance in at least 4 different chunks (S >= 256)"""
    inp, flags, P, D = _host_case("t100", S, N=301 if S == 256 else 37, D=256, noise=False)
    s, z = FL.oracle_logits(P, inp, flags, noise=False)
    P1 = FL.plant(P, s, z, flags, "translucent")
    s1, z1 = FL.oracle_logits({k: np.asarray(v, np.float64) for k, v in P1.items()}, inp, flags, noise=False)
    t_last = FL.transmittance_np(s1, z1, flags)[:, 32 * ((S - 1) // 32)]
    print(S, "translucent: T into the last chunk %.3g .. %.3g" % (t_last.min(), t_last.max()))
    assert t_last.min() >= FL.T_LAST_MIN and t_last.max() <= 0.6
    if S >= 256:
        P2 = FL.plant(P, s, z, flags, "scattered")
        s2, z2 = FL.oracle_logits({k: np.asarray(v, np.float64) for k, v in P2.items()}, inp, flags, noise=False)
        drop = FL.first_drop(FL.transmittance_np(s2, z2, flags), FL.DROP_T)
        print(S, "scattered: first chunk below %g:" % FL.DROP_T, np.bincount(drop))
        assert len(set(drop[drop < (S + 31) // 32].tolist())) >= 4


EMU_GATE = 4.0   # the float32 emulation of the reverse rounds against their float64 references and first-order scales


def emulate_frame(name, S, N=37, seed=3):
    """the frame's reverse-round state as the kernels would leave it, from the float32 emulation of every stage (CPU): the case's inputs,
    random records (logits ~ N(-4, 2), so that the rays stay translucent, a few near-opaque samples planted), random gp / gv"""
    c = dict(FL.CASES[name], S=S, N=N)
    inp = FL.inputs(name, seed, case=c)
    flags = FL._flags(c)
    rng = np.random.default_rng(seed)
    A = RL.Arith(f32=True)
    q_in = FL._qin(inp)
    noise = None if flags & L.NDC else torch.from_numpy(inp["noise"])
    _, z, _, _ = RL.ray_stage(A, RL._rowq(A, q_in, (N, S), "cpu"), flags, S, noise)
    s = torch.from_numpy(rng.normal(-4, 2, (N, S)).astype(np.float32))
    s.view(-1)[rng.choice(N * S, N * S // 200, replace=False)] = 200.0 if flags & L.DIST_ALPHA else 17.0
    sig = torch.where(s > 20, s, torch.log1p(torch.exp(s)))
    a = sig if flags & L.DIST_ALPHA else 1.0 - torch.exp(-sig)
    col = torch.sigmoid(torch.from_numpy(rng.normal(0, 1, (N, S, 3)).astype(np.float32)))
    rec = dict(r=col[..., 0], g=col[..., 1], b=col[..., 2], a=a, z=z)
    seeds = {k: torch.from_numpy(inp[k]) for k in ("g_rgb", "g_dp", "g_dg")}
    q = RL._rowq(A, q_in, (N,), "cpu")
    ray = RL._ray_scalars(RL.setup_ray(A, q, flags), q)
    _, _, dp, _ = RL.composite_fwd_ref(A, rec, ray, flags)
    om, T = RL.transmittance(A, RL.alpha_of(A, rec, flags))
    gs, suf = RL.composite_bwd_ref(A, rec, ray, seeds, flags, want_suffix=True)
    gp = torch.from_numpy(rng.normal(0, 1e-2, (N, S, 3)).astype(np.float32))
    gv = torch.from_numpy(rng.normal(0, 1e-3, (N, S, 3)).astype(np.float32))
    part = FL.frame_lanes_ref(A, gp, gv, z)
    sums = [[RL.warp_sum(A, part[:, 3 * j + c]) for c in range(3)] for j in range(3)]
    red, gdep = RL.ray_adjoint_ref(A, dict(ray, depth_sign=torch.sign(ray["depth"])), *sums, dp, seeds, flags, "depth" in inp)
    tot = RL.reduce_ref(A, red, torch.zeros(16))
    d = dict(rec={k: v.double() for k, v in rec.items()}, gp=gp.double(), gv=gv.double(), ckpt=T[:, 1:, 0].T.double(),
             suffix=suf.double(), gs0=gs[:, :min(S, 32)].double(), raypart=part.double(), rayred=red.double(), depth_pred=dp.double(),
             g_depth=gdep.double(), red=tot.double())
    return d, inp, flags


@pytest.mark.parametrize("name,S", [("t33", 33), ("t48-dist", 48), ("t100", 100), ("t100-ndc", 100), ("t100-eval", 100),
                                    ("t100-depth", 100), ("t100-white", 100), ("t1024", 1024)])
def test_emulation_of_the_reverse_rounds_within_model(name, S):
    """the float32 emulation of the checkpoints, suffix carry, chunk adjoint, lane partials, ray finish and reduction scores within
    EMU_GATE of its float64 reference, and every stage-local wrong answer scores at least 10x the stage's gate on the same data"""
    d, inp, flags = emulate_frame(name, S)
    out = FL.measure_stages(d, inp, flags, dev="cpu")
    print(name, {s: round(out[s]["err"], 2) for s in FL.STAGES},
          {(s, k): "%.3g" % t for s in FL.STAGES for k, t in list(out[s]["teeth"].items()) + list(out[s]["detect"].items())})
    for s in FL.STAGES:
        assert out[s]["err"] <= EMU_GATE, (name, s, out[s]["err"])
        for kind, t in out[s]["teeth"].items():
            assert t >= 10 * FL.STAGE_GATES[s], (name, s, kind, t)
    expect = {("cbwd0", "drop_late"), ("cbwd0", "carry_one"), ("cbwd0", "suffix_reset"), ("suffix", "drop_late"),
              ("suffix", "suffix_reset"), ("rayacc", "z_prev_chunk"), ("rayacc", "last_partial_twice"), ("rayacc", "skip_round1"),
              ("reduce", "skip32")}
    if S > 64:
        expect |= {("cbwd0", "carry"), ("suffix", "carry")}
    have = {(s, k) for s in FL.STAGES for k in out[s]["teeth"]}
    assert expect <= have, expect - have

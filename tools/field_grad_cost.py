#!/usr/bin/env python
"""Cost of training the field on explicit points: forward + backward of OfficialStaticNerf.forward(p, d) under autograd, with the
gradient to every parameter and to p, on the exact-fp32 engine (grad_engine=None: nnb_field_fwd with NNB_STASH + nnb_field_bwd) and on
tensor cores (engine='tc', grad_engine='tc': nnb_field_fwd + nnb_field_grad), and of the occupancy-only infer_occ(p) on both engines,
for M points x model.hidden_dim D.

CUDA events around each forward + backward.  Every configuration is warmed up first; then every configuration is timed in each of
--rounds rounds, the configurations alternating within a round, and the JSON line gives the median [min-max] over the rounds.  The
card's name and power limit are read in the same run (nvidia-smi query, read-only).  There is no CPU path: without a CUDA device the
tool fails."""
import argparse, json, os, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SIZES = (4096, 16384, 131072, 524288)
DIMS = (64, 128, 256)


def step_fn(net, p0, d0, g, occ, tc):
    """forward + backward of one query under autograd: the gradient to p and to every parameter (and to d unless occ)"""
    kw = dict(engine="tc", grad_engine="tc") if tc else {}

    def step():
        p = p0.detach().requires_grad_(True)
        if occ:
            _, s = net.infer_occ(p, **kw)
            loss = (s[:, 0] * g[:, 3]).sum()
        else:
            rgb, a = net(p, d0, return_addocc=True, **kw)
            loss = (rgb * g[:, :3]).sum() + (a[:, 0] * g[:, 3]).sum()
        loss.backward()
        return p.grad
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sizes", type=int, nargs="*", default=list(SIZES))
    ap.add_argument("--dims", type=int, nargs="*", default=list(DIMS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("field_grad_cost: needs a CUDA device (there is no CPU path and a CPU timing would say nothing about the GPU)")
    from field_query_cost import card, rounds_of, summary
    import nope_nerf_b200.model as mdl
    from oracle import nerf_oracle as O
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import _fullsize_cases as FC
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rounds": args.rounds, "reps": args.reps, "cases": []}
    gen = torch.Generator().manual_seed(0)
    for D in args.dims:
        cfg = FC.default_cfg(); cfg["model"]["hidden_dim"] = D
        net = mdl.OfficialStaticNerf(cfg).cuda()
        P = O.init_params(seed=1, D=D, hf_damp=True)
        net.load_state_dict({k: torch.from_numpy(np.asarray(P[k], np.float32)).reshape(v.shape) for k, v in net.state_dict().items()})
        for M in args.sizes:
            p = (torch.rand(M, 3, generator=gen) * 3 - 1.5).cuda()
            d = torch.nn.functional.normalize(torch.randn(M, 3, generator=gen), dim=1).cuda()
            g = torch.randn(M, 4, generator=gen).cuda()
            fns = {"exact": step_fn(net, p, d, g, False, False), "tc": step_fn(net, p, d, g, False, True),
                   "exact_occ": step_fn(net, p, d, g, True, False), "tc_occ": step_fn(net, p, d, g, True, True)}

            def timed(f):
                def call():
                    net.zero_grad(set_to_none=True)
                    f()
                return call
            ts = rounds_of({k: timed(f) for k, f in fns.items()}, args.warmup, args.reps, args.rounds)
            row = {"D": D, "M": M, **{k: summary(v) for k, v in ts.items()}}
            row["exact_over_tc"] = row["exact"]["median_ms"] / row["tc"]["median_ms"]
            row["exact_occ_over_tc_occ"] = row["exact_occ"]["median_ms"] / row["tc_occ"]["median_ms"]
            res["cases"].append(row)
            fmt = lambda s: "%.3f [%.3f-%.3f]" % (s["median_ms"], s["min_ms"], s["max_ms"])
            print("D=%3d M=%7d  exact %s ms  tc %s ms (x%.2f)  infer_occ exact %s ms  tc %s ms (x%.2f)"
                  % (D, M, fmt(row["exact"]), fmt(row["tc"]), row["exact_over_tc"], fmt(row["exact_occ"]), fmt(row["tc_occ"]),
                     row["exact_occ_over_tc_occ"]), file=sys.stderr)
            del fns, p, d, g
            net.zero_grad(set_to_none=True)
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

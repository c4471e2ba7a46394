#!/usr/bin/env python
"""Trust-region Thompson sampling (TuRBO / SCBO, DESIGN.md 4.18): one JSON line.

    python tools/trust_region_bench.py [--m 1048576] [--features 4096] [--steps 3] [--warmup 1]
                                       [--seeds 5] [--q 8] [--init 16] [--batches 10] [--parts select,optimize]

(a) select: the selection of m device candidates by q = 1 and 16 posterior sample paths (k = 10), the plain Philox
    source over the whole box (b200bo_paths_argmin_topk_philox) against the trust-region source
    (b200bo_paths_argmin_topk_philox_tr, a box of half the span around a centre, p = perturb_probability(d)), at C3
    (N = 4096, d = 16), C5 (N = 8192, d = 32) and N = 4096, d = 64.  CUDA events around each call (the call returns
    with the winners' rows on the host), after warm-up, mean and min over the steps.
(b) optimize: the best value after a fixed budget (--init random points, then --batches batches of --q points) on
    seeded synthetic objectives, --seeds seeds each, median and range:
      * Ackley, d = 20, and Levy, d = 32, on [-5, 10]^d (maximising -f): TrustRegionThompsonSampling, ThompsonSampling
        and LogExpectedImprovement (batches through KrigingBeliever);
      * Ackley, d = 10, with SCBO's two constraints sum(x) <= 0 and ||x|| <= 5: TrustRegionThompsonSampling (SCBO)
        against ConstrainedThompsonSampling; the value is the best feasible -f (None while no point is feasible).
    Every method uses device_philox candidates and analytic refinement, n_random = 10 000, n_smart = 10.
The GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
_REF = os.path.join(ROOT, "oracle", "_ref")  # the reference package, vendored by build()
if os.path.isdir(os.path.join(_REF, "bayes_opt")) and _REF not in sys.path:
    sys.path.insert(0, _REF)

import numpy as np  # noqa: E402

from thompson_bench import device_info, timed  # noqa: E402

SELECT = {"C3": (4096, 16), "C5": (8192, 32), "D64": (4096, 64)}


def select_leg(bo, args):
    from sklearn.gaussian_process.kernels import Matern

    from bayesianoptimization_b200.trust_region import perturb_probability

    out = {}
    for name, (n, d) in SELECT.items():
        rs = np.random.RandomState(0)
        X = rs.uniform(size=(n, d))
        y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
        gp = bo.B200GaussianProcessRegressor(kernel=Matern(0.5 * np.sqrt(d), nu=2.5), alpha=1e-6, normalize_y=True,
                                             optimizer=None).fit(X, y)
        bounds = np.stack([np.zeros(d), np.ones(d)], axis=1)
        center = X[int(np.argmax(y))]
        lo, hi = np.maximum(center - 0.25, 0.0), np.minimum(center + 0.25, 1.0)
        p = perturb_probability(d)
        res = {"N": n, "d": d, "p": p}
        for q in (1, 16):
            paths = gp.sample_paths(q, args.features, random_state=1)
            mean, best = timed(lambda: paths.argmin_topk_philox(7, bounds, args.m, 10), args.steps, args.warmup)
            res[f"philox_q{q}_ms"], res[f"philox_q{q}_min_ms"] = mean, best
            mean, best = timed(lambda: paths.argmin_topk_philox_tr(7, lo, hi, center, p, args.m, 10), args.steps,
                               args.warmup)
            res[f"tr_q{q}_ms"], res[f"tr_q{q}_min_ms"] = mean, best
            res[f"tr_vs_philox_q{q}"] = res[f"tr_q{q}_ms"] / res[f"philox_q{q}_ms"]
            del paths
        out[name] = res
        del gp
    return out


def ackley(x):
    a, b, c = 20.0, 0.2, 2 * np.pi
    return -a * np.exp(-b * np.sqrt(np.mean(x**2))) - np.exp(np.mean(np.cos(c * x))) + a + np.e


def levy(x):
    w = 1 + (x - 1) / 4
    t = np.sin(np.pi * w[0]) ** 2 + ((w[-1] - 1) ** 2) * (1 + np.sin(2 * np.pi * w[-1]) ** 2)
    return t + np.sum((w[:-1] - 1) ** 2 * (1 + 10 * np.sin(np.pi * w[:-1] + 1) ** 2))


def _make(bo, ref, method, d, seed, constrained):
    from scipy.optimize import NonlinearConstraint

    pb = {f"x{i:02d}": (-5.0, 10.0) for i in range(d)}
    acq = {"turbo": lambda: bo.TrustRegionThompsonSampling(), "ts": lambda: bo.ThompsonSampling(),
           "cts": lambda: bo.ConstrainedThompsonSampling(),
           "logei": lambda: bo.KrigingBeliever(bo.LogExpectedImprovement(xi=0.0))}[method]()
    con = None
    if constrained:
        def cfun(**kw):
            x = np.array([kw[k] for k in sorted(kw)])
            return np.array([x.sum(), np.linalg.norm(x)])

        con = NonlinearConstraint(cfun, [-np.inf, -np.inf], [0.0, 5.0])
    opt = ref.BayesianOptimization(f=None, pbounds=pb, constraint=con, random_state=seed, verbose=0,
                                   acquisition_function=acq)
    return bo.enable(opt, candidate_source="device_philox", refine="analytic"), pb


def run_one(bo, ref, fn, d, method, seed, args, constrained=False):
    opt, pb = _make(bo, ref, method, d, seed, constrained)
    keys = sorted(pb)
    rs = np.random.RandomState(1000 + seed)  # the same initial design for every method

    def evaluate(params):
        x = np.array([params[k] for k in keys])
        if constrained:
            opt.register(params=params, target=-fn(x), constraint_value=np.array([x.sum(), np.linalg.norm(x)]))
        else:
            opt.register(params=params, target=-fn(x))

    for x in rs.uniform(-5.0, 10.0, size=(args.init, d)):
        evaluate(dict(zip(keys, x)))
    t = time.perf_counter()
    for _ in range(args.batches):
        for params in bo.suggest_batch(opt, args.q):
            evaluate(params)
    secs = time.perf_counter() - t
    tgt = opt.space.target
    if constrained:
        feas = opt.space.mask
        best = float(tgt[feas].max()) if feas.any() else None
    else:
        best = float(tgt.max())
    return best, secs


def optimize_leg(bo, ref, args):
    problems = [("ackley20", ackley, 20, ["turbo", "ts", "logei"], False),
                ("levy32", levy, 32, ["turbo", "ts", "logei"], False),
                ("ackley10_scbo", ackley, 10, ["turbo", "cts"], True)]
    out = {"q": args.q, "init": args.init, "batches": args.batches, "seeds": args.seeds,
           "budget": args.init + args.q * args.batches, "value": "best -f (feasible only for the constrained problem)"}
    for name, fn, d, methods, constrained in problems:
        res = {}
        for method in methods:
            vals, secs = [], []
            for seed in range(args.seeds):
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    v, s = run_one(bo, ref, fn, d, method, seed, args, constrained)
                vals.append(v)
                secs.append(s)
            ok = [v for v in vals if v is not None]
            res[method] = {"best": vals, "median": float(np.median(ok)) if ok else None,
                           "min": float(min(ok)) if ok else None, "max": float(max(ok)) if ok else None,
                           "runs_with_a_feasible_point": len(ok), "mean_run_s": float(np.mean(secs))}
        out[name] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1 << 20)
    ap.add_argument("--features", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seeds", type=int, default=5)
    ap.add_argument("--q", type=int, default=8)
    ap.add_argument("--init", type=int, default=16)
    ap.add_argument("--batches", type=int, default=10)
    ap.add_argument("--parts", default="select,optimize")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("trust_region_bench needs a CUDA device")
    import bayesianoptimization_b200 as bo

    out = {"bench": "trust_region", "device": device_info(), "m": args.m, "n_features": args.features, "k": 10,
           "steps": args.steps, "warmup": args.warmup}
    parts = args.parts.split(",")
    if "select" in parts:
        out["select"] = select_leg(bo, args)
    if "optimize" in parts:
        import bayes_opt as ref

        out["optimize"] = optimize_leg(bo, ref, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

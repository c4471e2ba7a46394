#!/usr/bin/env python
"""Stencil against analytic refinement (DESIGN.md 4.10): one JSON object.

    python tools/refine_grad_bench.py [--shapes c3,c5] [--steps 5] [--warmup 1] [--m 1048576]

On one GP per shape (C3: N = 4096, d = 16; C5: N = 8192, d = 32; fixed hyper-parameters, seeded data), the same
seeds for both modes, the modes alternated in one process after a warm-up of each:
  round     one lockstep round of S = 10 runs, host clock around the call (it returns host values, so the device
            work is complete): the stencil's S (d + 1) rows through b200bo_acq_eval (as the refinement issues it,
            B200BO_PATH_STABLE) against S rows through b200bo_acq_value_grad;
  runs      the 10 L-BFGS-B runs of an EI refinement: per run nit, nfev, success and the final value, and the fraction
            of runs dropped for success = False;
  suggest   wall time of suggest() without refit for ExpectedImprovement and ThompsonSampling, and of
            ThompsonSampling.suggest_batch(q = 16)  (C3 only; M host candidates).
Means and minima over the steps.  The GPU name and power limit are read in the same run.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
_REF = os.path.join(ROOT, "oracle", "_ref")  # the reference package, vendored by build()
if os.path.isdir(os.path.join(_REF, "bayes_opt")) and _REF not in sys.path:
    sys.path.insert(0, _REF)

import numpy as np  # noqa: E402

from tools.thompson_bench import device_info  # noqa: E402

SHAPES = {"c3": (4096, 16), "c5": (8192, 32)}
S = 10
MODES = ("stencil", "analytic")


def _stats(ts):
    return {"mean_ms": 1e3 * float(np.mean(ts)), "min_ms": 1e3 * float(np.min(ts))}


def _alternate(fns, steps, warmup):
    """fns: {mode: callable}; every step runs each mode once, in turn."""
    out = {k: [] for k in fns}
    for i in range(warmup + steps):
        for k, fn in fns.items():
            t0 = time.perf_counter()
            fn()
            if i >= warmup:
                out[k].append(time.perf_counter() - t0)
    return {k: _stats(v) for k, v in out.items()}


def bench_shape(bo, name, args):
    from bayes_opt.target_space import TargetSpace
    from bayesianoptimization_b200.fused import _predicted_stencil, lockstep_lbfgsb
    from sklearn.gaussian_process.kernels import Matern

    n, d = SHAPES[name]
    rs = np.random.RandomState(0)
    X = rs.uniform(size=(n, d))
    y = np.sin(3 * X.sum(1) / np.sqrt(d)) + 0.5 * np.cos(2 * X[:, 0]) + 0.05 * rs.randn(n)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.3 * np.sqrt(d)), alpha=1e-6,
                                         normalize_y=True, optimizer=None).fit(X, y)
    space = TargetSpace(None, {f"x{j:02d}": (0.0, 1.0) for j in range(d)})
    lb, ub = space.bounds[:, 0], space.bounds[:, 1]
    ei = bo.ExpectedImprovement(xi=0.01)
    ei.y_max = float(y.max())
    acq = ei._get_acq(gp)
    x_tries = rs.uniform(size=(20000, d))
    _, _, top = acq.argmin_topk(x_tries, S)
    seeds = x_tries[top]
    res = {"n": n, "d": d, "rows_per_round": {"stencil": S * (d + 1), "analytic": S}}

    stencil_rows = np.vstack([np.vstack([s[None, :], _predicted_stencil(s, lb, ub)]) for s in seeds])

    def round_stencil():
        with acq.refine_mode():
            acq(stencil_rows)

    res["round"] = _alternate({"stencil": round_stencil, "analytic": lambda: acq.value_and_grad(seeds)},
                              args.steps * 4, args.warmup)

    runs = {}
    for mode in MODES:
        with acq.refine_mode():
            out = lockstep_lbfgsb(acq, seeds, space.bounds, grad=(mode == "analytic"))
        runs[mode] = {"nit": [int(r.nit) for r in out], "nfev": [int(r.nfev) for r in out],
                      "success": [bool(r.success) for r in out], "fun": [float(np.squeeze(r.fun)) for r in out],
                      "dropped_fraction": float(np.mean([not r.success for r in out]))}
    res["runs"] = runs

    def refine(mode):
        ei.b200_refine = mode
        return lambda: ei._smart_minimize(acq, space, seeds, np.random.RandomState(0))

    res["refine_10_runs"] = _alternate({m: refine(m) for m in MODES}, args.steps, args.warmup)

    if name == "c3":
        for x_, y_ in zip(X, y):
            space.register(x_, y_)
        ts = bo.ThompsonSampling(n_features=4096)

        def suggest(a, mode, q=None):
            def run():
                a.b200_refine = mode
                kw = dict(n_random=args.m, n_smart=S, fit_gp=False, random_state=np.random.RandomState(1))
                return a.suggest(gp, space, **kw) if q is None else a.suggest_batch(gp, space, q, **kw)

            return run

        res["suggest"] = {
            "ei": _alternate({m: suggest(ei, m) for m in MODES}, args.steps, args.warmup),
            "thompson_q1": _alternate({m: suggest(ts, m) for m in MODES}, args.steps, args.warmup),
            "thompson_batch_q16": _alternate({m: suggest(ts, m, 16) for m in MODES}, args.steps, args.warmup),
        }
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c3,c5")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--m", type=int, default=1 << 20)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("refine_grad_bench needs a CUDA device")
    import bayesianoptimization_b200 as bo

    out = {"device": device_info(), "S": S}
    for name in args.shapes.split(","):
        out[name] = bench_shape(bo, name, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

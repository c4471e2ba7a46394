#!/usr/bin/env python
"""Batch Thompson sampling against the other ways of getting q points per decision: one JSON line.

    python tools/batch_thompson_bench.py [--m 1048576] [--features 4096] [--steps 2] [--warmup 1]

At C3 (N = 4096 registered points, d = 16, fixed hyper-parameters, M host candidates, L features, n_smart = 10) it
times, wall clock around each call (every call returns its points on the host):
  * batch_q{1,4,16}     ThompsonSampling.suggest_batch(q): q paths, one candidate set ranked once, q x n_smart
                        L-BFGS-B runs in lockstep through the row-mode evaluation;
  * seq_q{1,4,16}       q calls of ThompsonSampling.suggest() (one path, its own candidate set, each);
  * liar_q{1,4,16}      q calls of ConstantLiar(ExpectedImprovement).suggest(): each copies the space, registers the
                        pending dummies and refits the GP (sklearn's optimizer, 5 restarts) before its EI pass;
  * round_q{4,16}       one lockstep refinement round of q x n_smart runs, q n_smart (d + 1) rows: the row-mode
                        evaluation (rows_ms) against the full q-path evaluation plus a column pick (full_ms).
The legs alternate inside every step, in one process; means and minima over the steps after the warm-up.  The TS
legs take the GP as fitted (fit_gp=False); fit_ms is one fit of that GP for reference.  The GPU name and power limit
are read in the same run.
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
_REF = os.path.join(ROOT, "oracle", "_ref")  # the reference package, vendored by build()
if os.path.isdir(os.path.join(_REF, "bayes_opt")) and _REF not in sys.path:
    sys.path.insert(0, _REF)

import numpy as np  # noqa: E402

from tools.thompson_bench import device_info  # noqa: E402

N, D = 4096, 16
QS = (1, 4, 16)
N_SMART = 10


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1 << 20)
    ap.add_argument("--features", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("batch_thompson_bench needs a CUDA device")
    import bayesianoptimization_b200 as bo
    from bayes_opt.target_space import TargetSpace
    from sklearn.gaussian_process.kernels import Matern

    rs = np.random.RandomState(0)
    space = TargetSpace(None, {f"x{j:02d}": (0.0, 1.0) for j in range(D)})
    X = rs.uniform(size=(N, D))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(N)
    for x, t in zip(X, y):
        space.register(x, float(t))
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(0.5 * np.sqrt(D), nu=2.5), alpha=1e-6, normalize_y=True,
                                         optimizer=None)
    t = time.perf_counter()
    gp.fit(space.params, space.target)
    fit_ms = 1e3 * (time.perf_counter() - t)
    liar_gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), alpha=1e-6, normalize_y=True,
                                              n_restarts_optimizer=5, random_state=np.random.RandomState(1))
    ts = bo.ThompsonSampling(n_features=args.features)
    kw = dict(n_random=args.m, n_smart=N_SMART)
    leg_rs = np.random.RandomState(2)

    def batch(q):
        return ts.suggest_batch(gp, space, q, fit_gp=False, random_state=leg_rs, **kw)

    def seq(q):
        return [ts.suggest(gp, space, fit_gp=False, random_state=leg_rs, **kw) for _ in range(q)]

    def liar(q):
        cl = bo.ConstantLiar(bo.ExpectedImprovement(xi=0.01))
        return [cl.suggest(liar_gp, space, fit_gp=True, random_state=leg_rs, **kw) for _ in range(q)]

    round_legs = {}
    for q in (4, 16):
        paths = gp.sample_paths(q, args.features, random_state=3)
        rows = rs.uniform(size=(q * N_SMART * (D + 1), D))
        pidx = np.repeat(np.arange(q), N_SMART * (D + 1)).astype(np.int32)
        assert np.array_equal(paths.eval_rows(rows, pidx), paths(rows)[np.arange(len(rows)), pidx])
        round_legs[q] = (lambda p=paths, r=rows, i=pidx: p.eval_rows(r, i),
                         lambda p=paths, r=rows, i=pidx: p(r)[np.arange(len(r)), i])

    legs = {}
    for q in QS:
        legs[f"batch_q{q}"] = lambda q=q: batch(q)
        legs[f"seq_q{q}"] = lambda q=q: seq(q)
        legs[f"liar_q{q}"] = lambda q=q: liar(q)
    for q, (rows_fn, full_fn) in round_legs.items():
        legs[f"round_q{q}_rows"] = rows_fn
        legs[f"round_q{q}_full"] = full_fn
    times = {k: [] for k in legs}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for step in range(args.warmup + args.steps):
            for name, fn in legs.items():  # alternate the legs inside every step
                torch.cuda.synchronize()
                t = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                if step >= args.warmup:
                    times[name].append(1e3 * (time.perf_counter() - t))
    res = {k: {"mean_ms": float(np.mean(v)), "min_ms": float(np.min(v))} for k, v in times.items()}
    for q in QS:
        res[f"batch_q{q}"]["speedup_vs_seq"] = res[f"seq_q{q}"]["mean_ms"] / res[f"batch_q{q}"]["mean_ms"]
        res[f"batch_q{q}"]["speedup_vs_liar"] = res[f"liar_q{q}"]["mean_ms"] / res[f"batch_q{q}"]["mean_ms"]
    for q in round_legs:
        res[f"round_q{q}_rows"]["speedup_vs_full"] = (res[f"round_q{q}_full"]["mean_ms"] /
                                                     res[f"round_q{q}_rows"]["mean_ms"])
    out = {"bench": "batch_thompson", "device": device_info(), "N": N, "d": D, "m": args.m,
           "n_features": args.features, "n_smart": N_SMART, "steps": args.steps, "warmup": args.warmup,
           "fit_ms": fit_ms, "legs": res}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

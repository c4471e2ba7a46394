#!/usr/bin/env python
"""Kriging-believer batches against the other ways of getting q points per decision: one JSON line.

    python tools/kriging_believer_bench.py [--configs C3,C5] [--m 1048576] [--steps 1] [--warmup 1]

Per configuration (C3: N = 4096 registered points, d = 16; C5: N = 8192, d = 32; fixed hyper-parameters, M host
candidates, n_smart = 10) it times, wall clock around each call (every call returns its points on the host):
  * kb_{ei,ucb}_q{4,16}  KrigingBeliever(EI / UCB).suggest_batch(q): one fork of the fitted GP, one candidate set, q
                         greedy rounds of fused selection + lockstep refinement, an O(N^2) conditioning between rounds;
  * ts_q{4,16}           ThompsonSampling.suggest_batch(q) (batch Thompson sampling);
  * liar_q{4,16}         q calls of ConstantLiar(ExpectedImprovement).suggest(): each copies the space, registers the
                         dummies and refits the GP (sklearn's optimizer, 5 restarts) before its EI pass.  Timed once,
                         without a warm-up run of its own (the other legs warm the same kernels up).
The kb / ts legs take the GP as fitted (fit_gp=False).  ``rounds`` breaks one kb_ei_q16 call down per round: the
conditioning (condition_on_pending), the fused kernel (b200bo_last_kernel_ms) with its prune statistics
(b200bo_last_prune_stats) and the refinement (_smart_minimize).  The GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
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

CONFIGS = {"C3": (4096, 16), "C5": (8192, 32)}
QS = (4, 16)
N_SMART = 10


def _round_breakdown(bo, gp, space, kw, rs):
    """Per-round timings of one KrigingBeliever(EI).suggest_batch(16)."""
    import torch

    from bayesianoptimization_b200 import _lib as B

    kb = bo.KrigingBeliever(bo.ExpectedImprovement(xi=0.01))
    base = kb.base_acquisition
    rounds, cur = [], {}
    cls = type(gp)
    orig_cond, orig_sel, orig_smart = cls.condition_on_pending, bo.FusedAcquisition.argmin_topk, type(base)._smart_minimize

    def cond(self, X, extra_rows=0):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = orig_cond(self, X, extra_rows)
        cur["condition_ms"] = 1e3 * (time.perf_counter() - t)
        return out

    def sel(self, x, k):
        t = time.perf_counter()
        out = orig_sel(self, x, k)
        ms, ev, tot = C.c_float(), C.c_int64(), C.c_int64()
        B.check(B.lib().b200bo_last_kernel_ms(C.byref(ms)))
        B.check(B.lib().b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
        rounds.append(cur.copy())
        cur.clear()
        rounds[-1].update(select_ms=1e3 * (time.perf_counter() - t), kernel_ms=float(ms.value),
                          evaluated=int(ev.value), total=int(tot.value))
        return out

    def smart(self, *a, **k):
        t = time.perf_counter()
        out = orig_smart(self, *a, **k)
        rounds[-1]["refine_ms"] = 1e3 * (time.perf_counter() - t)
        return out

    cls.condition_on_pending, bo.FusedAcquisition.argmin_topk, type(base)._smart_minimize = cond, sel, smart
    try:
        kb.suggest_batch(gp, space, 16, fit_gp=False, random_state=rs, **kw)
    finally:
        cls.condition_on_pending, bo.FusedAcquisition.argmin_topk, type(base)._smart_minimize = (
            orig_cond, orig_sel, orig_smart)
    return rounds


def run_config(bo, name, m, steps, warmup):
    import torch
    from bayes_opt.target_space import TargetSpace
    from sklearn.gaussian_process.kernels import Matern

    N, D = CONFIGS[name]
    rs = np.random.RandomState(0)
    space = TargetSpace(None, {f"x{j:02d}": (0.0, 1.0) for j in range(D)})
    X = rs.uniform(size=(N, D))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(N)
    for x, t in zip(X, y):
        space.register(x, float(t))
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(0.5 * np.sqrt(D), nu=2.5), alpha=1e-6, normalize_y=True,
                                         optimizer=None)
    gp.fit(space.params, space.target)
    liar_gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), alpha=1e-6, normalize_y=True,
                                              n_restarts_optimizer=5, random_state=np.random.RandomState(1))
    ts = bo.ThompsonSampling()
    kw = dict(n_random=m, n_smart=N_SMART)
    leg_rs = np.random.RandomState(2)

    def kb(base, q):
        return bo.KrigingBeliever(base).suggest_batch(gp, space, q, fit_gp=False, random_state=leg_rs, **kw)

    def liar(q):
        cl = bo.ConstantLiar(bo.ExpectedImprovement(xi=0.01))
        return [cl.suggest(liar_gp, space, fit_gp=True, random_state=leg_rs, **kw) for _ in range(q)]

    legs = {}
    for q in QS:
        legs[f"kb_ei_q{q}"] = lambda q=q: kb(bo.ExpectedImprovement(xi=0.01), q)
        legs[f"kb_ucb_q{q}"] = lambda q=q: kb(bo.UpperConfidenceBound(kappa=2.576), q)
        legs[f"ts_q{q}"] = lambda q=q: ts.suggest_batch(gp, space, q, fit_gp=False, random_state=leg_rs, **kw)
    times = {k: [] for k in legs}
    for step in range(warmup + steps):
        for leg, fn in legs.items():  # alternate the legs inside every step
            torch.cuda.synchronize()
            t = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if step >= warmup:
                times[leg].append(1e3 * (time.perf_counter() - t))
    for q in QS:
        torch.cuda.synchronize()
        t = time.perf_counter()
        liar(q)
        torch.cuda.synchronize()
        times[f"liar_q{q}"] = [1e3 * (time.perf_counter() - t)]
    res = {k: {"mean_ms": float(np.mean(v)), "min_ms": float(np.min(v))} for k, v in times.items()}
    for q in QS:
        res[f"kb_ei_q{q}"]["speedup_vs_liar"] = res[f"liar_q{q}"]["mean_ms"] / res[f"kb_ei_q{q}"]["mean_ms"]
    rounds = _round_breakdown(bo, gp, space, kw, np.random.RandomState(4))
    return {"N": N, "d": D, "legs": res, "rounds": rounds}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C3,C5")
    ap.add_argument("--m", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("kriging_believer_bench needs a CUDA device")
    import bayesianoptimization_b200 as bo

    out = {"bench": "kriging_believer", "device": device_info(), "m": args.m, "n_smart": N_SMART,
           "steps": args.steps, "warmup": args.warmup, "configs": {}}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for name in args.configs.split(","):
            out["configs"][name] = run_config(bo, name, args.m, args.steps, args.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

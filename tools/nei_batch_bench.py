#!/usr/bin/env python
"""Batches of noisy EI with pending points (PendingNEI) against Kriging-believer batches of LogEI: one JSON line.

    python tools/nei_batch_bench.py [--configs C3,C5] [--qs 4,16] [--m 1048576] [--reps 2] [--study-seeds 10] [--out FILE]

(a) Per configuration (C3: N = 4096 registered points, d = 16; C5: N = 8192, d = 32; Matern 2.5, length scale 0.7, +
    WhiteKernel(1e-2) at fixed hyper-parameters, alpha = 1e-10, normalize_y; M host candidates, n_smart = 10) and q:
    one warm-up call, then --reps timed calls (wall time) of ``PendingNEI(LogNoisyExpectedImprovement(n_samples=16)).suggest_batch``
    and of ``KrigingBeliever(LogExpectedImprovement()).suggest_batch``, alternating in this one process.  The PendingNEI
    call is split into the fantasy draw (``noiseless_fantasies``), the per-round fantasy extension
    (``NoiselessFantasies.condition_on_pending``: the factor row update, fantasy_row_kernel and the S solves), the
    selection (wall time of ``argmin_topk``, with its chunked host upload; ``select_kernel_per_round`` is
    b200bo_last_kernel_ms after it, CUDA events around the last chunk's fused kernel only), and the refinement.  The share of the
    extension that is the factor row update alone is measured apart: one ``condition_on_pending`` row of the noiseless
    regressor against one row of its fantasies, on forks.
(b) a seeded study on Hartmann-6 with Gaussian observation noise (sd 0.1), tools/nei_bench.py's defaults: per seed, 5
    random points, then batches of q = 4 from PendingNEI(LogNEI, S = 16), KrigingBeliever(LogEI) and batch Thompson
    sampling until 40 evaluations, alpha = 1e-2; reported is the noise-free Hartmann-6 value at each run's final
    recommendation (the registered point with the best posterior mean), whatever the outcome.
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
for p in (ROOT, os.path.join(ROOT, "oracle", "_ref")):
    if os.path.isdir(p) and p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from nei_bench import hartmann6, kernel_ms  # noqa: E402
from thompson_bench import device_info  # noqa: E402

CONFIGS = {"C3": (4096, 16), "C5": (8192, 32)}


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


def _setup(bo, name):
    from bayes_opt.target_space import TargetSpace
    from sklearn.gaussian_process.kernels import Matern, WhiteKernel

    n, d = CONFIGS[name]
    rs = np.random.RandomState(0)
    X = rs.uniform(size=(n, d))
    y = -np.sum((X - 0.5) ** 2, axis=1) + 0.1 * rs.randn(n)
    space = TargetSpace(None, {f"x{j:02d}": (0.0, 1.0) for j in range(d)}, random_state=1)
    for x, t in zip(X, y):
        space.register(x, float(t))

    def gp():
        return bo.B200GaussianProcessRegressor(kernel=Matern(length_scale=0.7, nu=2.5) + WhiteKernel(1e-2),
                                               alpha=1e-10, normalize_y=True, optimizer=None)

    return space, gp


class _Timed:
    """Wall time (device-synchronised: every timed call returns host arrays) of a bound method, accumulated."""

    def __init__(self, obj, name, log):
        self.fn, self.log, self.name = getattr(obj, name), log, name
        setattr(obj, name, self)

    def __call__(self, *a, **k):
        t0 = time.perf_counter()
        out = self.fn(*a, **k)
        self.log.setdefault(self.name, []).append(time.perf_counter() - t0)
        return out


def batch(bo, B, name, q, m, reps):
    import bayesianoptimization_b200.gpr as G

    space, make_gp = _setup(bo, name)
    res = {"pending_nei_s": [], "kb_logei_s": [], "split_ms": None}
    for rep in range(reps + 1):  # rep 0 warms up both
        base = bo.LogNoisyExpectedImprovement(n_samples=16)
        pn = bo.PendingNEI(base)
        log = {}
        kms = []
        draw = G.B200GaussianProcessRegressor.noiseless_fantasies

        def timed_draw(self, *a, **k):
            t0 = time.perf_counter()
            fant = draw(self, *a, **k)
            log.setdefault("draw", []).append(time.perf_counter() - t0)
            _Timed(fant, "condition_on_pending", log)
            return fant

        def timed_closure(*a, _orig=base._closure, **k):
            acq = _orig(*a, **k)
            sel = acq.argmin_topk

            def argmin_topk(*aa, **kk):
                t0 = time.perf_counter()
                out = sel(*aa, **kk)
                log.setdefault("select", []).append(time.perf_counter() - t0)
                kms.append(kernel_ms(B))
                return out

            acq.argmin_topk = argmin_topk
            return acq

        G.B200GaussianProcessRegressor.noiseless_fantasies = timed_draw
        base._closure = timed_closure
        _Timed(base, "_smart_minimize", log)
        try:
            t0 = time.perf_counter()
            _quiet(pn.suggest_batch, make_gp(), space, q, n_random=m, n_smart=10, fit_gp=True, random_state=rep)
            t_pn = time.perf_counter() - t0
        finally:
            G.B200GaussianProcessRegressor.noiseless_fantasies = draw
        kb = bo.KrigingBeliever(bo.LogExpectedImprovement(xi=0.0))
        t0 = time.perf_counter()
        _quiet(kb.suggest_batch, make_gp(), space, q, n_random=m, n_smart=10, fit_gp=True, random_state=rep)
        t_kb = time.perf_counter() - t0
        if rep == 0:
            continue
        res["pending_nei_s"].append(t_pn)
        res["kb_logei_s"].append(t_kb)
        res["split_ms"] = {
            "fantasy_draw": 1e3 * sum(log.get("draw", [])),
            "extension_per_round": 1e3 * float(np.mean(log.get("condition_on_pending", [np.nan]))),
            "select_per_round": 1e3 * float(np.mean(log["select"])),
            "select_kernel_per_round": float(np.mean(kms)),
            "refine_per_round": 1e3 * float(np.mean(log["_smart_minimize"])),
        }
    # the factor row update alone against one row of fantasies: two forks of the noiseless regressor per repetition
    gp = make_gp().fit(space.params, space.target)
    t_row, t_fant = [], []
    for r in range(4):
        x = np.random.RandomState(r).uniform(size=(1, space.dim))
        fork = gp.noiseless_fantasies(16, random_state=r, extra_rows=1).gp
        t0 = time.perf_counter()
        fork.condition_on_pending(x)  # in place: a Kriging-believer row, no fantasies
        t_row.append(time.perf_counter() - t0)
        fant = gp.noiseless_fantasies(16, random_state=r, extra_rows=1)
        t0 = time.perf_counter()
        fant.condition_on_pending(x)
        t_fant.append(time.perf_counter() - t0)
    res["row_update_ms"] = 1e3 * float(np.mean(t_row[1:]))
    res["fantasy_row_ms"] = 1e3 * float(np.mean(t_fant[1:]))
    return res


def study(bo, ref, seeds, q=4, init=5, evals=40):
    from bayesianoptimization_b200.acquisition import suggest_batch

    out = {}
    for name, make in (("pending_lognei", lambda: bo.PendingNEI(bo.LogNoisyExpectedImprovement(n_samples=16))),
                       ("kb_logei", lambda: bo.KrigingBeliever(bo.LogExpectedImprovement(xi=0.0))),
                       ("batch_ts", lambda: bo.ThompsonSampling())):
        vals = []
        for seed in range(seeds):
            noise = np.random.RandomState(1000 + seed)

            def f(x):
                return float(hartmann6(x)[0] + 0.1 * noise.randn())

            opt = ref.BayesianOptimization(f=None, pbounds={f"x{j}": (0.0, 1.0) for j in range(6)},
                                           acquisition_function=make(), random_state=seed, verbose=0)
            opt.set_gp_params(alpha=1e-2)
            bo.enable(opt)
            for p in opt.random_sample(init):
                opt.register(params=p, target=f(opt._space.params_to_array(p)))
            while len(opt.space) < evals:
                for p in _quiet(suggest_batch, opt, min(q, evals - len(opt.space))):
                    opt.register(params=p, target=f(opt._space.params_to_array(p)))
            X = opt.space.params
            opt._gp.fit(X, opt.space.target)
            mu = opt._gp.predict(X)
            vals.append(float(hartmann6(X[int(np.argmax(mu))])[0]))
        out[name] = {"noise_free_at_recommendation": vals, "mean": float(np.mean(vals)),
                     "median": float(np.median(vals))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C3,C5")
    ap.add_argument("--qs", default="4,16")
    ap.add_argument("--m", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--study-seeds", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bayes_opt as ref

    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import _lib as B

    res = {"device": device_info(), "m": a.m}
    for name in filter(None, a.configs.split(",")):
        for q in map(int, filter(None, a.qs.split(","))):
            res[f"{name}_q{q}"] = batch(bo, B, name, q, a.m, a.reps)
    if a.study_seeds > 0:
        res["hartmann6_noisy_batch_study"] = study(bo, ref, a.study_seeds)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

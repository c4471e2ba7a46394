#!/usr/bin/env python
"""Constrained noisy expected improvement against NEI x constraints and EI x constraints: one JSON line.

    python tools/cnei_bench.py [--m 524288] [--rounds 3] [--study-seeds 10] [--study-iters 30] [--out FILE]

(a) C4: N = 2048, d = 16, a target and 2 constraint GPs, each Matern 2.5 (length scale 0.7) + WhiteKernel(1e-2) at
    fixed hyper-parameters, alpha = 1e-10, normalize_y; M = 2^19 Philox candidates, k = 10.  Per round, alternating in
    this one process: EI x constraints, then for S = 1, 4 and 16 NEI x constraints and CNEI, and LogCNEI at S = 16 - the
    fused kernel time (b200bo_last_kernel_ms, CUDA events on the launch's stream).  None of them is pruned.
(b) one full ``BayesianOptimization.suggest()`` (GP and constraint fits included) at C4 with 10 000 candidates and 10
    refinements: ConstrainedNoisyExpectedImprovement against NoisyExpectedImprovement, S = 16.
(c) a seeded study on Hartmann-6 with a noisy objective (sd 0.1) and a noisy constraint sum(x) <= 3 (sd 0.1): per seed,
    NEI x PoF (the reference's noiseless constraint GP) and CNEI (a WhiteKernel constraint GP), S = 16, each 5 random
    points + --study-iters iterations through bayes_opt.BayesianOptimization with alpha = 1e-2.  Reported per run: the
    noise-free value and the true feasibility of the recommendation, the registered point with the largest target
    posterior mean among those whose constraint posterior mean is feasible (the largest mean overall when none is).
    The global maximum is 3.32237.
The GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import types
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "_ref")):
    if os.path.isdir(p) and p not in sys.path:
        sys.path.insert(0, p)

import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from nei_bench import hartmann6, kernel_ms, stats  # noqa: E402
from thompson_bench import device_info  # noqa: E402


def _gp(bo, X, y):
    from sklearn.gaussian_process.kernels import Matern, WhiteKernel

    gp = bo.B200GaussianProcessRegressor(kernel=Matern(length_scale=0.7, nu=2.5) + WhiteKernel(1e-2), alpha=1e-10,
                                         normalize_y=True, optimizer=None)
    return gp.fit(X, y)


def c4(bo, B, m, rounds):
    rs = np.random.RandomState(0)
    n, d = 2048, 16
    X = rs.uniform(size=(n, d))
    gp = _gp(bo, X, -np.sum((X - 0.5) ** 2, axis=1) + 0.1 * rs.randn(n))
    cons = [_gp(bo, X, X.sum(1) - 8.0 + 0.1 * rs.randn(n)), _gp(bo, X, np.sin(X[:, 0] * 3) + 0.1 * rs.randn(n))]
    con = types.SimpleNamespace(model=cons, lb=np.array([-np.inf, -0.5]), ub=np.array([0.5, 0.8]))
    y_max = float(gp._y_raw.max())
    bounds = np.array([[0.0, 1.0]] * d)

    def cnei(S, log=False):
        r = np.random.RandomState(S)
        fant = gp.noiseless_fantasies(S, random_state=r)
        cf = [c.noiseless_fantasies(S, random_state=r) for c in cons]
        from bayesianoptimization_b200.acquisition import cnei_eligible

        ok = np.ascontiguousarray(cnei_eligible(np.ones(n, bool), [f.F for f in cf], con.lb, con.ub), dtype=np.uint8)
        best = np.empty(S)
        B.check(B.lib().b200bo_gp_set_fantasy_incumbent(fant.handle.ptr, ok.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                        B.as_dp(best)))
        fant.best = best
        return bo.FusedAcquisition(B.ACQ_LOGCNEI if log else B.ACQ_CNEI, gp, con, xi=0.01, fantasies=fant,
                                   constraint_fantasies=cf)

    def nei(S):
        return bo.FusedAcquisition(B.ACQ_NEI, gp, con, xi=0.01, fantasies=gp.noiseless_fantasies(S, random_state=S))

    cases = [("ei_x_constraints", lambda: bo.FusedAcquisition(B.ACQ_EI, gp, con, xi=0.01, y_max=y_max))]
    for S in (1, 4, 16):
        cases += [(f"nei_x_constraints_S{S}", lambda S=S: nei(S)), (f"cnei_S{S}", lambda S=S: cnei(S))]
    cases += [("logcnei_S16", lambda: cnei(16, log=True))]
    times = {name: [] for name, _ in cases}
    os.environ["B200BO_PRUNE"] = "0"
    for r in range(rounds + 1):  # round 0 warms up
        for name, make in cases:
            acq = make()  # the fantasies of every noiseless handle are redrawn for each case
            acq.argmin_topk_philox(1234 + r, bounds, m, 10)
            if r:
                times[name].append(kernel_ms(B))
    os.environ.pop("B200BO_PRUNE", None)
    return {name: stats(v) for name, v in times.items()}


def suggest_cost(bo, ref):
    from scipy.optimize import NonlinearConstraint
    from sklearn.gaussian_process.kernels import Matern, WhiteKernel

    rs = np.random.RandomState(1)
    n, d = 2048, 16
    X = rs.uniform(size=(n, d))
    out = {}
    for name, make in (("nei_x_pof_S16", lambda: bo.NoisyExpectedImprovement(xi=0.01)),
                       ("cnei_S16", lambda: bo.ConstrainedNoisyExpectedImprovement(xi=0.01))):
        con = NonlinearConstraint(lambda **kw: 0.0, -np.inf, 8.5)
        opt = ref.BayesianOptimization(f=None, pbounds={f"x{j:02d}": (0.0, 1.0) for j in range(d)}, constraint=con,
                                       acquisition_function=make(), random_state=1, verbose=0)
        opt.set_gp_params(alpha=1e-2, optimizer=None)
        bo.enable(opt)
        for m in opt.constraint.model:
            m.set_params(kernel=Matern(length_scale=0.7, nu=2.5) + WhiteKernel(1e-2), optimizer=None)
        for x in X:
            opt.register(params=x, target=float(-np.sum((x - 0.5) ** 2) + 0.1 * rs.randn()),
                         constraint_value=float(x.sum() + 0.1 * rs.randn()))
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                opt.suggest()
            ts.append(time.perf_counter() - t0)
        out[name] = stats(ts[1:])
    return out


def study(bo, ref, seeds, iters):
    from scipy.optimize import NonlinearConstraint
    from sklearn.gaussian_process.kernels import Matern, WhiteKernel

    out = {}
    for name in ("nei_x_pof", "cnei"):
        vals, feas = [], []
        for seed in range(seeds):
            noise = np.random.RandomState(1000 + seed)

            def f(**kw):
                x = np.array([kw[f"x{j}"] for j in range(6)])
                return float(hartmann6(x)[0] + 0.1 * noise.randn())

            def c(**kw):
                return float(sum(kw[f"x{j}"] for j in range(6)) + 0.1 * noise.randn())

            acq = (bo.NoisyExpectedImprovement(xi=0.0, n_samples=16) if name == "nei_x_pof"
                   else bo.ConstrainedNoisyExpectedImprovement(xi=0.0, n_samples=16))
            opt = ref.BayesianOptimization(f=f, pbounds={f"x{j}": (0.0, 1.0) for j in range(6)},
                                           constraint=NonlinearConstraint(c, -np.inf, 3.0), acquisition_function=acq,
                                           random_state=seed, verbose=0)
            opt.set_gp_params(alpha=1e-2)
            bo.enable(opt)
            if name == "cnei":
                for m in opt.constraint.model:
                    m.set_params(kernel=Matern(nu=2.5) + WhiteKernel(1e-2))
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                try:
                    opt.maximize(init_points=5, n_iter=iters)
                except Exception as e:  # NEI x PoF raises without a feasible registered point
                    vals.append(None)
                    feas.append(None)
                    out.setdefault(f"{name}_errors", []).append(type(e).__name__)
                    continue
            X = opt.space.params
            mu = opt._gp.predict(X)
            cm = opt.constraint.model[0].predict(X)
            ok = cm <= 3.0
            i = int(np.argmax(np.where(ok, mu, -np.inf))) if ok.any() else int(np.argmax(mu))
            vals.append(float(hartmann6(X[i])[0]))
            feas.append(bool(X[i].sum() <= 3.0))
        done = [v for v in vals if v is not None]
        out[name] = {"noise_free_at_recommendation": vals, "truly_feasible": feas,
                     "mean": float(np.mean(done)) if done else None,
                     "feasible_fraction": float(np.mean([x for x in feas if x is not None])) if done else None}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1 << 19)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--study-seeds", type=int, default=10)
    ap.add_argument("--study-iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bayes_opt as ref

    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import _lib as B

    res = {"device": device_info()}
    res["c4_kernel_ms"] = c4(bo, B, a.m, a.rounds)
    res["c4_suggest_s"] = suggest_cost(bo, ref)
    if a.study_seeds > 0:
        res["hartmann6_noisy_constraint_study"] = study(bo, ref, a.study_seeds, a.study_iters)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

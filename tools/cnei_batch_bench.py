#!/usr/bin/env python
"""Batches of constrained noisy expected improvement against batch constrained Thompson sampling: one JSON line.

    python tools/cnei_batch_bench.py [--m 524288] [--qs 4,16] [--rounds 2] [--study-seeds 10] [--study-batches 6]
                                     [--out FILE]

(a) C4: N = 2048, d = 16, a target and 2 constraint GPs, each Matern 2.5 (length scale 0.7) + WhiteKernel(1e-2) at
    fixed hyper-parameters, alpha = 1e-10 (the reference's alpha = 1e-6 on the constraint GPs), normalize_y.  Per q and
    round, alternating in this one process: ``PendingNEI(LogConstrainedNoisyExpectedImprovement(n_samples=16))
    .suggest_batch`` and ``ConstrainedThompsonSampling().suggest_batch``, each with M = 2^19 Philox candidates,
    10 refinements on the device gradient, fit_gp=False and no dummies.  The wall time of each call (every stage ends
    in a device synchronise) and, for PendingNEI, its split: the fantasy draw of the J + 1 GPs (forks included), the
    per-round extension of the J + 1 handles, the incumbents, the selection (the fused kernel over M candidates per
    round) and the refinement.
(b) a seeded study on Hartmann-6 with a noisy objective (sd 0.1) and a noisy constraint sum(x) <= 3 (sd 0.1): per seed
    and method, 5 random points, then --study-batches batches of q = 4 through ``suggest_batch(optimizer, 4)``, with
    alpha = 1e-2 and a WhiteKernel constraint GP.  Reported per run: the noise-free value and the true feasibility of
    the recommendation (cnei_bench.py's rule).  The global maximum is 3.32237.
The GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import warnings
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "_ref")):
    if os.path.isdir(p) and p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from nei_bench import hartmann6, stats  # noqa: E402
from thompson_bench import device_info  # noqa: E402

STAGES = defaultdict(float)


def _timed(owner, name, stage):
    """Wraps owner.name so that its wall time adds to STAGES[stage] (every wrapped call returns host results)."""
    fn = getattr(owner, name)

    def wrapper(*a, **k):
        t0 = time.perf_counter()
        try:
            return fn(*a, **k)
        finally:
            STAGES[stage] += time.perf_counter() - t0

    setattr(owner, name, wrapper)


def _instrument(bo):
    from bayesianoptimization_b200 import acquisition as A
    from bayesianoptimization_b200 import fused, gpr

    _timed(gpr.B200GaussianProcessRegressor, "noiseless_fantasies", "draw")
    _timed(A._ConstrainedNoisyEI, "condition_on_pending", "extension")
    _timed(A._ConstrainedNoisyEI, "_set_incumbent", "incumbent")
    _timed(fused.FusedAcquisition, "argmin_topk_philox", "selection")
    _timed(A.DeviceHooks, "_smart_minimize", "refinement")


def _c4_space(bo, rs):
    from bayes_opt.target_space import TargetSpace
    from scipy.optimize import NonlinearConstraint
    from sklearn.gaussian_process.kernels import Matern, WhiteKernel

    from bayesianoptimization_b200.gpr import to_b200_gp

    n, d = 2048, 16
    space = TargetSpace(None, {f"x{j:02d}": (0.0, 1.0) for j in range(d)},
                        constraint=NonlinearConstraint(lambda *a: 0.0, np.array([-np.inf, -0.5]), np.array([0.5, 0.8])))
    cm = space.constraint
    cm._model = [to_b200_gp(m) for m in cm.model]  # as enable(optimizer) does
    for m in cm.model:
        m.set_params(kernel=Matern(length_scale=0.7, nu=2.5) + WhiteKernel(1e-2), optimizer=None)
    X = rs.uniform(size=(n, d))
    for x in X:
        space.register(x, float(-np.sum((x - 0.5) ** 2) + 0.1 * rs.randn()),
                       constraint_value=np.array([x.sum() - 8.0, np.sin(3 * x[0])]) + 0.1 * rs.randn(2))
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(length_scale=0.7, nu=2.5) + WhiteKernel(1e-2), alpha=1e-10,
                                         normalize_y=True, optimizer=None)
    gp.fit(space.params, space.target)
    cm.fit(space.params, space._constraint_values)
    return gp, space


def c4(bo, m, qs, rounds):
    gp, space = _c4_space(bo, np.random.RandomState(0))
    nei = bo.PendingNEI(bo.LogConstrainedNoisyExpectedImprovement(n_samples=16))
    ts = bo.ConstrainedThompsonSampling()
    for a in (nei.base_acquisition, ts):
        a.b200_candidate_source, a.b200_refine = "device_philox", "analytic"
    out = {}
    for q in qs:
        wall = {"pending_logcnei": [], "constrained_ts": []}
        split = defaultdict(list)
        for r in range(rounds + 1):  # round 0 warms up
            for name, acq in (("pending_logcnei", nei), ("constrained_ts", ts)):
                if name == "pending_logcnei":
                    acq.dummies = []
                STAGES.clear()
                t0 = time.perf_counter()
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    acq.suggest_batch(gp, space, q, n_random=m, n_smart=10, fit_gp=False, random_state=100 + r)
                dt = time.perf_counter() - t0
                if r:
                    wall[name].append(dt)
                    if name == "pending_logcnei":
                        for k, v in STAGES.items():
                            split[k].append(v)
        out[f"q{q}"] = {"wall_s": {k: stats(v) for k, v in wall.items()},
                        "pending_logcnei_split_s": {k: stats(v) for k, v in split.items()}}
    return out


def study(bo, ref, seeds, batches):
    from scipy.optimize import NonlinearConstraint
    from sklearn.gaussian_process.kernels import Matern, WhiteKernel

    out = {}
    for name in ("pending_logcnei", "constrained_ts"):
        vals, feas = [], []
        for seed in range(seeds):
            noise = np.random.RandomState(1000 + seed)

            def f(**kw):
                x = np.array([kw[f"x{j}"] for j in range(6)])
                return float(hartmann6(x)[0] + 0.1 * noise.randn())

            def c(**kw):
                return float(sum(kw[f"x{j}"] for j in range(6)) + 0.1 * noise.randn())

            acq = (bo.PendingNEI(bo.LogConstrainedNoisyExpectedImprovement(xi=0.0, n_samples=16))
                   if name == "pending_logcnei" else bo.ConstrainedThompsonSampling())
            opt = ref.BayesianOptimization(f=f, pbounds={f"x{j}": (0.0, 1.0) for j in range(6)},
                                           constraint=NonlinearConstraint(c, -np.inf, 3.0), acquisition_function=acq,
                                           random_state=seed, verbose=0)
            opt.set_gp_params(alpha=1e-2)
            bo.enable(opt)
            for m in opt.constraint.model:
                m.set_params(kernel=Matern(nu=2.5) + WhiteKernel(1e-2))
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                opt.maximize(init_points=5, n_iter=0)
                for _ in range(batches):
                    for p in bo.suggest_batch(opt, 4):
                        opt.probe(p, lazy=False)
            X = opt.space.params
            mu = opt._gp.predict(X)
            ok = opt.constraint.model[0].predict(X) <= 3.0
            i = int(np.argmax(np.where(ok, mu, -np.inf))) if ok.any() else int(np.argmax(mu))
            vals.append(float(hartmann6(X[i])[0]))
            feas.append(bool(X[i].sum() <= 3.0))
        out[name] = {"noise_free_at_recommendation": vals, "truly_feasible": feas, "mean": float(np.mean(vals)),
                     "feasible_fraction": float(np.mean(feas))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1 << 19)
    ap.add_argument("--qs", default="4,16")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--study-seeds", type=int, default=10)
    ap.add_argument("--study-batches", type=int, default=6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bayes_opt as ref

    import bayesianoptimization_b200 as bo

    _instrument(bo)
    res = {"device": device_info()}
    res["c4"] = c4(bo, a.m, [int(q) for q in a.qs.split(",")], a.rounds)
    if a.study_seeds > 0:
        res["hartmann6_noisy_constraint_batch_study"] = study(bo, ref, a.study_seeds, a.study_batches)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

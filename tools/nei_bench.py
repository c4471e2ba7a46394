#!/usr/bin/env python
"""Noisy expected improvement against EI: one JSON line.

    python tools/nei_bench.py [--m 1048576] [--rounds 3] [--study-seeds 10] [--study-iters 40] [--out FILE]

(a) C3: N = 4096, d = 16, Matern 2.5 (length scale 0.7) + WhiteKernel(1e-2) at fixed hyper-parameters, alpha = 1e-10,
    normalize_y; M = 2^20 Philox candidates, k = 10.  Per round, alternating in this one process: unpruned EI
    (B200BO_PRUNE=0), NEI at S = 1, 4 and 16, LogNEI at S = 16, and pruned EI for scale - the fused kernel time
    (b200bo_last_kernel_ms, CUDA events on the launch's stream).
(b) the cost of the noiseless GP's factorisation plus b200bo_gp_set_fantasies (``noiseless_fantasies``, S = 16, wall
    time, first call and a call that refits the cached noiseless handle), and of one full ``suggest()`` of
    NoisyExpectedImprovement against ExpectedImprovement at C3 (10 000 candidates, 10 refinements).
(c) a seeded study on Hartmann-6 with Gaussian observation noise (sd 0.1): per seed, EI, NEI and LogNEI (S = 16) each run
    5 random points + --study-iters iterations through bayes_opt.BayesianOptimization with alpha = 1e-2; reported is the
    noise-free Hartmann-6 value at each run's final recommendation (the registered point with the best posterior
    mean), whatever the outcome.  The global maximum is 3.32237.
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

import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from thompson_bench import device_info  # noqa: E402


def stats(v):
    return {"mean": float(np.mean(v)), "min": float(np.min(v)), "n": len(v)}


def kernel_ms(B):
    ms = C.c_float()
    B.check(B.lib().b200bo_last_kernel_ms(C.byref(ms)))
    return float(ms.value)


def c3(bo, B, m, rounds):
    from sklearn.gaussian_process.kernels import Matern, WhiteKernel

    rs = np.random.RandomState(0)
    n, d = 4096, 16
    X = rs.uniform(size=(n, d))
    y = -np.sum((X - 0.5) ** 2, axis=1) + 0.1 * rs.randn(n)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(length_scale=0.7, nu=2.5) + WhiteKernel(1e-2), alpha=1e-10,
                                         normalize_y=True, optimizer=None)
    gp.fit(X, y)
    bounds = np.array([[0.0, 1.0]] * d)
    t0 = time.perf_counter()
    fants = {S: gp.noiseless_fantasies(S, random_state=S) for S in (1, 4, 16)}
    first_fant_s = time.perf_counter() - t0
    fants = {S: gp.noiseless_fantasies(S, random_state=S) for S in (1, 4, 16)}  # the cached handle refitted
    ei = bo.FusedAcquisition(B.ACQ_EI, gp, xi=0.01, y_max=float(y.max()))
    cases = [("ei_unpruned", ei, "0")]
    cases += [(f"nei_S{S}", None, "0") for S in (1, 4, 16)]
    cases += [("lognei_S16", None, "0"), ("ei_pruned", ei, "1")]
    times = {name: [] for name, _, _ in cases}
    for r in range(rounds + 1):  # round 0 warms up
        for name, acq, prune in cases:
            os.environ["B200BO_PRUNE"] = prune
            if acq is None:
                S = int(name.split("S")[1])
                fant = gp.noiseless_fantasies(S, random_state=S)
                code = B.ACQ_LOGNEI if name.startswith("log") else B.ACQ_NEI
                acq = bo.FusedAcquisition(code, gp, xi=0.01, fantasies=fant)
            acq.argmin_topk_philox(1234 + r, bounds, m, 10)
            if r:
                times[name].append(kernel_ms(B))
    os.environ.pop("B200BO_PRUNE", None)
    fant_s = []
    for _ in range(3):
        t0 = time.perf_counter()
        gp.noiseless_fantasies(16, random_state=0)
        fant_s.append(time.perf_counter() - t0)
    return gp, {name: stats(v) for name, v in times.items()}, {"first_three_calls_s": first_fant_s,
                                                             "refit_and_fantasies_S16_s": stats(fant_s)}


def suggest_cost(bo, ref, gp):
    from bayes_opt.target_space import TargetSpace

    d = gp.X_train_.shape[1]
    space = TargetSpace(None, {f"x{j:02d}": (0.0, 1.0) for j in range(d)}, random_state=1)
    for x, t in zip(gp.X_train_, gp._y_raw):
        space.register(x, float(t))
    out = {}
    for name, acq in (("ei", bo.ExpectedImprovement(xi=0.01)), ("nei_S16", bo.NoisyExpectedImprovement(xi=0.01))):
        ts = []
        for r in range(3):
            t0 = time.perf_counter()
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                acq.suggest(gp, space, n_random=10_000, n_smart=10, fit_gp=False, random_state=r)
            ts.append(time.perf_counter() - t0)
        out[name] = stats(ts[1:])
    return out


_H6_A = np.array([[10, 3, 17, 3.5, 1.7, 8], [0.05, 10, 17, 0.1, 8, 14], [3, 3.5, 1.7, 10, 17, 8],
                  [17, 8, 0.05, 10, 0.1, 14]])
_H6_P = 1e-4 * np.array([[1312, 1696, 5569, 124, 8283, 5886], [2329, 4135, 8307, 3736, 1004, 9991],
                         [2348, 1451, 3522, 2883, 3047, 6650], [4047, 8828, 8732, 5743, 1091, 381]])
_H6_ALPHA = np.array([1.0, 1.2, 3.0, 3.2])


def hartmann6(x):
    x = np.atleast_2d(x)
    return np.sum(_H6_ALPHA * np.exp(-np.sum(_H6_A * (x[:, None, :] - _H6_P) ** 2, axis=2)), axis=1)


def study(bo, ref, seeds, iters):
    out = {}
    for name, make in (("ei", lambda: bo.ExpectedImprovement(xi=0.0)),
                       ("nei", lambda: bo.NoisyExpectedImprovement(xi=0.0, n_samples=16)),
                       ("lognei", lambda: bo.LogNoisyExpectedImprovement(xi=0.0, n_samples=16))):
        vals = []
        for seed in range(seeds):
            noise = np.random.RandomState(1000 + seed)

            def f(**kw):
                x = np.array([kw[f"x{j}"] for j in range(6)])
                return float(hartmann6(x)[0] + 0.1 * noise.randn())

            opt = ref.BayesianOptimization(f=f, pbounds={f"x{j}": (0.0, 1.0) for j in range(6)},
                                           acquisition_function=make(), random_state=seed, verbose=0)
            opt.set_gp_params(alpha=1e-2)
            bo.enable(opt)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                opt.maximize(init_points=5, n_iter=iters)
            X = opt.space.params
            mu = opt._gp.predict(X)
            vals.append(float(hartmann6(X[int(np.argmax(mu))])[0]))
        out[name] = {"noise_free_at_recommendation": vals, "mean": float(np.mean(vals)),
                     "median": float(np.median(vals))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1 << 20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--study-seeds", type=int, default=10)
    ap.add_argument("--study-iters", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bayes_opt as ref

    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import _lib as B

    res = {"device": device_info()}
    gp, res["c3_kernel_ms"], res["c3_fantasies"] = c3(bo, B, a.m, a.rounds)
    res["c3_suggest_s"] = suggest_cost(bo, ref, gp)
    del gp
    if a.study_seeds > 0:
        res["hartmann6_noisy_study"] = study(bo, ref, a.study_seeds, a.study_iters)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

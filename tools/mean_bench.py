#!/usr/bin/env python
"""The posterior-mean merit (B200BO_ACQ_MEAN) against EI on the same candidates, and recommend(): one JSON line.

    python tools/mean_bench.py [--m 1048576] [--rounds 3] [--out FILE]

(a) Selection (k = 10) over M = 2^20 candidates, host-drawn (uploaded) and Philox (generated in the kernel), at
    C3: N = 4096, d = 16, one GP;  C5: N = 8192, d = 32, one GP;  C4: N = 2048, d = 16, a target and 2 constraint GPs.
    Every GP is Matern 2.5 (length scale 0.7) + WhiteKernel(1e-2) at fixed hyper-parameters, alpha = 1e-10,
    normalize_y.  Per round, alternating in this one process: MEAN, EI with B200BO_PRUNE=0 and EI pruned (the default;
    with constraint GPs EI is never pruned, so C4's two EI rows are the same kernel).  Reported: the kernel time
    (b200bo_last_kernel_ms, CUDA events on the launch's stream; the pruned EI time includes its bound pass and sort)
    of the Philox launch and the wall time of each call (a synchronising host entry point; host candidates are uploaded
    chunk by chunk behind the kernels, which then run as several launches, so only their wall time is reported).
(b) recommend() on a BayesianOptimization with 1024 registered noisy points in d = 16 (C3's GP, one constraint GP at
    C4's bounds): in_sample=True and in_sample=False (10 000 candidates, 10 L-BFGS-B refinements), each with the
    optimizer's GPs stale (clones fitted, at fixed hyper-parameters) and fitted (used read-only).
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

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from nei_bench import kernel_ms, stats  # noqa: E402
from thompson_bench import device_info  # noqa: E402

CONFIGS = {"C3": dict(n=4096, d=16, J=0), "C5": dict(n=8192, d=32, J=0), "C4": dict(n=2048, d=16, J=2)}


def _kernel():
    from sklearn.gaussian_process.kernels import Matern, WhiteKernel

    return Matern(length_scale=0.7, nu=2.5, length_scale_bounds="fixed") + WhiteKernel(1e-2, "fixed")


def _gp(bo, X, y):
    return bo.B200GaussianProcessRegressor(kernel=_kernel(), alpha=1e-10, normalize_y=True, optimizer=None).fit(X, y)


def _setup(bo, cfg, seed):
    rs = np.random.RandomState(seed)
    n, d = cfg["n"], cfg["d"]
    X = rs.uniform(size=(n, d))
    gp = _gp(bo, X, -np.sum((X - 0.5) ** 2, axis=1) + 0.1 * rs.randn(n))
    con = None
    if cfg["J"]:
        cons = [_gp(bo, X, X.sum(1) - d / 2 + 0.1 * rs.randn(n)), _gp(bo, X, np.sin(X[:, 0] * 3) + 0.1 * rs.randn(n))]
        con = types.SimpleNamespace(model=cons, lb=np.array([-np.inf, -0.5]), ub=np.array([0.5, 0.8]))
    return rs, gp, con


def selection(bo, B, m, rounds):
    out = {}
    for name, cfg in CONFIGS.items():
        rs, gp, con = _setup(bo, cfg, 0)
        d = cfg["d"]
        xt = rs.uniform(size=(m, d))
        bounds = np.array([[0.0, 1.0]] * d)
        y_max = float(gp._y_raw.max())
        acqs = {"mean": (bo.FusedAcquisition(B.ACQ_MEAN, gp, con), None),
                "ei_unpruned": (bo.FusedAcquisition(B.ACQ_EI, gp, con, xi=0.01, y_max=y_max), "0"),
                "ei_pruned": (bo.FusedAcquisition(B.ACQ_EI, gp, con, xi=0.01, y_max=y_max), "1")}
        res = {k: {"host_wall_ms": [], "philox_kernel_ms": [], "philox_wall_ms": []} for k in acqs}
        for r in range(rounds + 1):  # round 0 warms every shape up
            for k, (acq, prune) in acqs.items():
                if prune is None:
                    os.environ.pop("B200BO_PRUNE", None)
                else:
                    os.environ["B200BO_PRUNE"] = prune
                t0 = time.perf_counter()
                acq.argmin_topk(xt, 10)
                t1 = time.perf_counter()
                acq.argmin_topk_philox(1234 + r, bounds, m, 10)
                t2 = time.perf_counter()
                kp = kernel_ms(B)
                if r:
                    res[k]["host_wall_ms"].append(1e3 * (t1 - t0))
                    res[k]["philox_kernel_ms"].append(kp)
                    res[k]["philox_wall_ms"].append(1e3 * (t2 - t1))
        os.environ.pop("B200BO_PRUNE", None)
        out[name] = {k: {kk: stats(vv) for kk, vv in v.items()} for k, v in res.items()}
        print(name, json.dumps({k: {kk: round(vv["mean"], 3) for kk, vv in v.items()} for k, v in out[name].items()}),
              file=sys.stderr)
    return out


def recommend_times(bo, rounds):
    import bayes_opt
    from scipy.optimize import NonlinearConstraint

    d, n = 16, 1024
    keys = [f"x{i:02d}" for i in range(d)]
    out = {}
    for constrained in (False, True):
        rs = np.random.RandomState(5)
        con = NonlinearConstraint(lambda **p: sum(p.values()) - d / 2, -np.inf, 0.5) if constrained else None
        opt = bayes_opt.BayesianOptimization(f=None, pbounds={k: (0.0, 1.0) for k in keys}, constraint=con,
                                             random_state=1, verbose=0, allow_duplicate_points=True)
        opt.set_gp_params(kernel=_kernel(), alpha=1e-10)
        bo.enable(opt)
        if constrained:
            for g in opt.constraint.model:
                g.set_params(kernel=_kernel(), alpha=1e-10)
        X = rs.uniform(size=(n, d))
        for x in X:
            kw = {"constraint_value": float(x.sum() - d / 2 + 0.1 * rs.randn())} if constrained else {}
            opt.register(params=dict(zip(keys, x)), target=float(-np.sum((x - 0.5) ** 2) + 0.1 * rs.randn()), **kw)
        tag = "constrained" if constrained else "unconstrained"
        for fitted in (False, True):
            if fitted:
                opt.acquisition_function._fit_gp(opt._gp, opt.space)
            for ins in (True, False):
                ts = []
                for r in range(rounds + 1):
                    t0 = time.perf_counter()
                    bo.recommend(opt, in_sample=ins, random_state=r)
                    if r:
                        ts.append(1e3 * (time.perf_counter() - t0))
                key = f"{tag}_{'fitted' if fitted else 'stale'}_{'in_sample' if ins else 'domain'}_ms"
                out[key] = stats(ts)
                print(key, round(out[key]["mean"], 2), file=sys.stderr)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1 << 20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import _lib as B

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        res = {"device": device_info(), "m": a.m, "rounds": a.rounds, "selection": selection(bo, B, a.m, a.rounds),
               "recommend": recommend_times(bo, a.rounds)}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

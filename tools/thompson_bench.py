#!/usr/bin/env python
"""Thompson sampling vs EI on the same candidates: one JSON line.

    python tools/thompson_bench.py [--m 1048576] [--features 4096] [--steps 3] [--warmup 1]

For C3 (N = 4096, d = 16) and C5 (N = 8192, d = 32), fixed hyper-parameters, it times
  * ts_q1/4/16       PosteriorPaths.argmin_topk (b200bo_paths_argmin_topk, k = 10) of 1, 4 and 16 paths, L features,
  * ei               FusedAcquisition.argmin_topk (b200bo_acq_argmin_topk, k = 10),
on the same M host candidates: CUDA events on the default stream around each call (the calls return with their
results on the host, so a window includes the streamed H2D copy of the batch), after warm-up, mean over the steps.
The C4 leg (N = 2048, d = 16, two constraint GPs, --m-c4 = 2^19 candidates) times
  * cts_q1           ConstrainedPaths.argmin_topk (b200bo_cpaths_argmin_topk, k = 10): one path of the target and one of
                     each constraint GP, ranked feasible-first,
  * ts_q1            the target's path alone (PosteriorPaths.argmin_topk), for the cost of the joint ranking,
  * poi_constrained  FusedAcquisition PoI x probability of feasibility (b200bo_acq_argmin_topk, k = 10).
Also reported: the one-off path creation (draws on the host + one O(N^2) solve per path).  Rates: cand/s = M / time,
path*cand/s = q M / time.  The GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

CONFIGS = {"C3": (4096, 16), "C5": (8192, 32)}
C4 = (2048, 16, 2)  # N, d, constraint GPs


def device_info():
    import torch

    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.split(",")[0])
    except Exception:
        info["power_limit_w"] = None
    return info


def timed(fn, steps, warmup):
    import torch

    for _ in range(warmup):
        fn()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(steps):
        t0.record()
        fn()
        t1.record()
        t1.synchronize()
        ms.append(t0.elapsed_time(t1))
    return float(np.mean(ms)), float(np.min(ms))


def c4_leg(bo, args):
    from types import SimpleNamespace

    from sklearn.gaussian_process.kernels import Matern

    from bayesianoptimization_b200.paths import ConstrainedPaths

    n, d, J = C4
    m = args.m_c4
    rs = np.random.RandomState(0)
    X = rs.uniform(size=(n, d))
    Xc = rs.uniform(size=(m, d))
    mk = lambda y: bo.B200GaussianProcessRegressor(kernel=Matern(0.5 * np.sqrt(d), nu=2.5), alpha=1e-6,  # noqa: E731
                                                   normalize_y=True, optimizer=None).fit(X, y)
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    gp = mk(y)
    cgps = [mk(np.cos(X[:, j::J].sum(1)) + 0.1 * rs.randn(n)) for j in range(J)]
    lb, ub = np.array([-np.inf, -0.5]), np.array([0.3, np.inf])
    res = {"N": n, "d": d, "constraint_gps": J, "m": m}
    t = time.perf_counter()
    path_rs = np.random.RandomState(1)
    target = gp.sample_paths(1, args.features, random_state=path_rs)
    cp = ConstrainedPaths(target, [g.sample_paths(1, args.features, random_state=path_rs) for g in cgps], lb, ub)
    res["cts_q1_create_ms"] = 1e3 * (time.perf_counter() - t)
    mean, best = timed(lambda: cp.argmin_topk(Xc, 10), args.steps, args.warmup)
    res["cts_q1_ms"], res["cts_q1_min_ms"], res["cts_q1_cand_per_s"] = mean, best, m / (mean * 1e-3)
    mean, best = timed(lambda: target.argmin_topk(Xc, 10), args.steps, args.warmup)
    res["ts_q1_ms"], res["ts_q1_min_ms"] = mean, best
    acq = bo.FusedAcquisition(bo._lib.ACQ_POI, gp, SimpleNamespace(model=cgps, lb=lb, ub=ub), xi=0.01,
                              y_max=float(y.max()))
    mean, best = timed(lambda: acq.argmin_topk(Xc, 10), args.steps, args.warmup)
    res["poi_constrained_ms"], res["poi_constrained_min_ms"] = mean, best
    res["poi_constrained_cand_per_s"] = m / (mean * 1e-3)
    res["cts_q1_vs_ts_q1"] = res["cts_q1_ms"] / res["ts_q1_ms"]
    res["cts_q1_speedup_vs_poi_constrained"] = res["poi_constrained_ms"] / res["cts_q1_ms"]
    feas = np.mean(cp(Xc[:65536])[:, 0] == cp.raw(Xc[:65536])[:, 0, 0])
    res["cts_feasible_fraction_first_65536"] = float(feas)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1 << 20)
    ap.add_argument("--features", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--m-c4", type=int, default=1 << 19)
    ap.add_argument("--configs", default="C3,C5,C4")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("thompson_bench needs a CUDA device")
    import bayesianoptimization_b200 as bo
    from sklearn.gaussian_process.kernels import Matern

    B = bo._lib
    out = {"bench": "thompson_vs_ei", "device": device_info(), "m": args.m, "n_features": args.features, "k": 10,
           "steps": args.steps, "warmup": args.warmup, "configs": {}}
    for name in args.configs.split(","):
        if name == "C4":
            out["configs"][name] = c4_leg(bo, args)
            continue
        n, d = CONFIGS[name]
        rs = np.random.RandomState(0)
        X = rs.uniform(size=(n, d))
        y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
        Xc = rs.uniform(size=(args.m, d))
        gp = bo.B200GaussianProcessRegressor(kernel=Matern(0.5 * np.sqrt(d), nu=2.5), alpha=1e-6, normalize_y=True,
                                             optimizer=None).fit(X, y)
        res = {"N": n, "d": d}
        for q in (1, 4, 16):
            t = time.perf_counter()
            paths = gp.sample_paths(q, args.features, random_state=1)
            res[f"ts_q{q}_create_ms"] = 1e3 * (time.perf_counter() - t)
            mean, best = timed(lambda: paths.argmin_topk(Xc, 10), args.steps, args.warmup)
            res[f"ts_q{q}_ms"], res[f"ts_q{q}_min_ms"] = mean, best
            res[f"ts_q{q}_cand_per_s"] = args.m / (mean * 1e-3)
            res[f"ts_q{q}_path_cand_per_s"] = q * args.m / (mean * 1e-3)
        acq = bo.FusedAcquisition(B.ACQ_EI, gp, xi=0.01, y_max=float(y.max()))
        mean, best = timed(lambda: acq.argmin_topk(Xc, 10), args.steps, args.warmup)
        res["ei_ms"], res["ei_min_ms"], res["ei_cand_per_s"] = mean, best, args.m / (mean * 1e-3)
        res["ts_q1_speedup_vs_ei"] = res["ei_ms"] / res["ts_q1_ms"]
        out["configs"][name] = res
        del gp, paths, acq
    print(json.dumps(out))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Thompson sampling vs EI on the same candidates: one JSON line.

    python tools/thompson_bench.py [--m 1048576] [--features 4096] [--steps 3] [--warmup 1]

For C3 (N = 4096, d = 16) and C5 (N = 8192, d = 32), fixed hyper-parameters, it times
  * ts_q1/4/16       PosteriorPaths.argmin_topk (b200bo_paths_argmin_topk, k = 10) of 1, 4 and 16 paths, L features,
  * ei               FusedAcquisition.argmin_topk (b200bo_acq_argmin_topk, k = 10),
on the same M host candidates: CUDA events on the default stream around each call (the calls return with their
results on the host, so a window includes the streamed H2D copy of the batch), after warm-up, mean over the steps.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1 << 20)
    ap.add_argument("--features", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--configs", default="C3,C5")
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

#!/usr/bin/env python
"""Max-value entropy search vs EI at C3: one JSON line.

    python tools/mes_bench.py [--m 1048576] [--rounds 3] [--features 4096] [--out FILE]

C3: N = 4096 training points, d = 16, Matern 2.5 at fixed hyper-parameters, M = 2^20 candidates, k = 10.
  * kernel_ms        the fused predict kernel alone (b200bo_last_kernel_ms: CUDA events around the launch) of EI and of
                     MES with K = 1, 10 and 16 samples y*, on the same device-resident candidates (b200bo_acq_eval_dev
                     with fused top-10 selection), alternated EI, K1, K10, K16 in every round; mean and min over rounds
  * call_ms          FusedAcquisition.argmin_topk on the same candidates in host memory (streamed upload included),
                     alternated the same way; CUDA events on the default stream, the call returns with its results
  * ystar_ms         MaxValueEntropySearch's y* sampling with K = 10: sample_paths (host draws + one O(N^2 q) solve)
                     and mes_max_values (host candidate draws, path maxima over them and the training inputs) for
                     several candidate-set sizes n_max_candidates
  * suggest_ms       a full suggest() (fit_gp=False, n_random = M, n_smart = 10) of MaxValueEntropySearch (K = 10,
                     default n_max_candidates) and of ExpectedImprovement on the same target space
The GPU name and power limit are read in the same run.
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
for p in (ROOT, os.path.join(ROOT, "oracle", "_ref")):  # the reference package, where build() vendored it
    if os.path.isdir(p) and p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from thompson_bench import device_info  # noqa: E402


def stats(v):
    return {"mean": float(np.mean(v)), "min": float(np.min(v)), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1 << 20)
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--d", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--features", type=int, default=4096)
    ap.add_argument("--ystar-sizes", default="16384,65536,262144,1048576")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("mes_bench needs a CUDA device")
    import bayesianoptimization_b200 as bo
    from bayes_opt.target_space import TargetSpace
    from sklearn.gaussian_process.kernels import Matern

    from bayesianoptimization_b200.acquisition import MES_MAX_CANDIDATES, mes_max_values

    B = bo._lib
    L = B.lib()
    n, d, m = args.n, args.d, args.m
    rs = np.random.RandomState(0)
    X = rs.uniform(size=(n, d))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    Xc = rs.uniform(size=(m, d))
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(0.5 * np.sqrt(d), nu=2.5), alpha=1e-6, normalize_y=True,
                                         optimizer=None).fit(X, y)
    out = {"bench": "mes_vs_ei", "device": device_info(), "config": "C3", "N": n, "d": d, "m": m, "k": 10,
           "n_features": args.features, "rounds": args.rounds}

    # y* of the kernel legs: K samples above the data (what mes_max_values returns is of this kind)
    ystar = {K: float(y.max()) + float(np.std(y)) * np.linspace(0.05, 1.0, K) for K in (1, 10, 16)}
    legs = {"ei": bo.FusedAcquisition(B.ACQ_EI, gp, xi=0.01, y_max=float(y.max()))}
    for K, v in ystar.items():
        legs[f"mes_k{K}"] = bo.FusedAcquisition(B.ACQ_MES, gp, max_values=v)

    x_dev = torch.from_numpy(Xc).cuda()
    sel = torch.empty(16 * 11, dtype=torch.uint8, device="cuda")

    def kernel_once(f):
        spec = f.spec  # sets this closure's samples on the handle
        B.check(L.b200bo_acq_eval_dev(C.byref(spec), x_dev.data_ptr(), m, None, None, None, 10, sel.data_ptr(), 0,
                                      None))
        ms = C.c_float()
        B.check(L.b200bo_last_kernel_ms(C.byref(ms)))
        return float(ms.value)

    def call_once(f):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        f.argmin_topk(Xc, 10)
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1)

    kern, call, sel_out = {k: [] for k in legs}, {k: [] for k in legs}, {}
    for f in legs.values():  # warm-up of every leg
        kernel_once(f)
        call_once(f)
    for _ in range(args.rounds):
        for name, f in legs.items():
            kern[name].append(kernel_once(f))
        for name, f in legs.items():
            call[name].append(call_once(f))
    for name, f in legs.items():
        idx, val, top = f.argmin_topk(Xc, 10)
        sel_out[name] = {"argmin": int(idx), "value": float(val)}
    out["kernel_ms"] = {k: stats(v) for k, v in kern.items()}
    out["call_ms"] = {k: stats(v) for k, v in call.items()}
    out["kernel_vs_ei"] = {k: out["kernel_ms"][k]["mean"] / out["kernel_ms"]["ei"]["mean"] for k in legs}
    out["selection"] = sel_out

    # y* sampling (K = 10) over candidate sets of several sizes
    space = TargetSpace(None, {f"x{j:02d}": (0.0, 1.0) for j in range(d)})
    for i in range(n):
        space.register(X[i], float(y[i]))
    ys_ms = {}
    for size in [int(s) for s in args.ystar_sizes.split(",")]:
        v = []
        for r in range(args.rounds + 1):
            torch.cuda.synchronize()
            t = time.perf_counter()
            srs = np.random.RandomState(100 + r)
            paths = gp.sample_paths(10, args.features, random_state=srs)
            t_paths = time.perf_counter() - t
            mes_max_values(gp, paths, space, srs, size)
            v.append((1e3 * t_paths, 1e3 * (time.perf_counter() - t)))
        v = v[1:]  # the first round warms up
        ys_ms[str(size)] = {"sample_paths_ms": stats([a for a, _ in v]), "total_ms": stats([b for _, b in v])}
    out["ystar_k10_ms"] = ys_ms

    # full suggest() of both policies on the same space (fit_gp=False: the GP above)
    sug = {"ei": [], "mes_k10": []}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for r in range(args.rounds + 1):
            for name in sug:
                acq = bo.ExpectedImprovement(xi=0.01) if name == "ei" else bo.MaxValueEntropySearch(
                    n_samples=10, n_features=args.features)
                torch.cuda.synchronize()
                t = time.perf_counter()
                acq.suggest(gp, space, n_random=m, n_smart=10, fit_gp=False, random_state=np.random.RandomState(r))
                if r > 0:
                    sug[name].append(1e3 * (time.perf_counter() - t))
    out["suggest_ms"] = {k: stats(v) for k, v in sug.items()}
    out["mes_default_n_max_candidates"] = MES_MAX_CANDIDATES
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

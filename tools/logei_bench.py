#!/usr/bin/env python
"""LogEI / LogPoI against EI: one JSON line.

    python tools/logei_bench.py [--m 1048576] [--rounds 3] [--out FILE]

(a) C3: N = 4096, d = 16, Matern 2.5 at fixed hyper-parameters, M = 2^20 device-resident candidates, k = 10, y_max = the
    largest target.  Per kind (EI, LogEI, LogPoI, alternated in every round): the fused selection time
    (b200bo_last_kernel_ms: CUDA events around the bound pass, the sort and the evaluation) and the fraction of the
    candidates that went through phase B under pruning (b200bo_last_prune_stats), with pruning on (the default) and
    off (B200BO_PRUNE=0).
(b) the late-stage study: a training set with a fifth of the rows uniform and the rest clustered around the optimum
    of -|x - 0.6|^2 with a spread shrinking from 1e-1 to 1e-3, at d = 2 (N = 60), d = 16 (N = 600) and the C3 shape
    (N = 4096, d = 16), seeded and generated here; Matern 2.5, length scale 1 (fixed), normalize_y, alpha = 1e-6,
    xi = 0.01; 10 000 uniform candidates.  Reports the fraction of candidates whose EI is exactly 0 or below 1e-12 of
    the largest EI, and for the top-5 seeds of each of EI and LogEI the L-BFGS-B runs of the refinement (the lockstep
    driver, SciPy's default gtol 1e-5): nit, distance moved and final closure value.
The GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "_ref")):
    if os.path.isdir(p) and p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from thompson_bench import device_info  # noqa: E402


def stats(v):
    return {"mean": float(np.mean(v)), "min": float(np.min(v)), "n": len(v)}


def late_stage(d, n, seed):
    rs = np.random.RandomState(seed)
    opt = np.full(d, 0.6)
    n_u = n // 5
    spread = np.logspace(-1, -3, n - n_u)[:, None]
    X = np.vstack([rs.uniform(size=(n_u, d)), np.clip(opt + spread * rs.randn(n - n_u, d), 0.0, 1.0)])
    return X, -np.sum((X - opt) ** 2, axis=1), rs


def part_a(bo, args):
    import torch
    from sklearn.gaussian_process.kernels import Matern

    B = bo._lib
    L = B.lib()
    n, d, m = 4096, 16, args.m
    rs = np.random.RandomState(0)
    X = rs.uniform(size=(n, d))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(0.5 * np.sqrt(d), nu=2.5), alpha=1e-6, normalize_y=True,
                                         optimizer=None).fit(X, y)
    x_dev = torch.from_numpy(rs.uniform(size=(m, d))).cuda()
    sel = torch.empty(16 * 11, dtype=torch.uint8, device="cuda")
    legs = {name: bo.FusedAcquisition(code, gp, xi=0.01, y_max=float(y.max()))
            for name, code in (("ei", B.ACQ_EI), ("logei", B.ACQ_LOGEI), ("logpoi", B.ACQ_LOGPOI))}

    def once(f):
        B.check(L.b200bo_acq_eval_dev(C.byref(f.spec), x_dev.data_ptr(), m, None, None, None, 10, sel.data_ptr(), 0,
                                      None))
        ms, ev, tot = C.c_float(), C.c_int64(), C.c_int64()
        B.check(L.b200bo_last_kernel_ms(C.byref(ms)))
        B.check(L.b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
        rec = sel.view(torch.int64).view(11, 2)[0].cpu().numpy()
        return float(ms.value), ev.value / tot.value, (int(rec[1]), float(np.int64(rec[0]).view(np.float64)))

    out = {"config": "C3", "N": n, "d": d, "m": m, "k": 10}
    for prune in ("1", "0"):
        os.environ["B200BO_PRUNE"] = prune
        for f in legs.values():
            once(f)
        ms, frac, best = {k: [] for k in legs}, {}, {}
        for _ in range(args.rounds):
            for name, f in legs.items():
                t, fr, b = once(f)
                ms[name].append(t)
                frac[name], best[name] = fr, b
        out["prune_on" if prune == "1" else "prune_off"] = {
            "kernel_ms": {k: stats(v) for k, v in ms.items()}, "evaluated_fraction": frac, "argmin": best,
            "vs_ei": {k: float(np.mean(ms[k]) / np.mean(ms["ei"])) for k in legs}}
    os.environ.pop("B200BO_PRUNE", None)
    return out


def part_b(bo, args):
    from sklearn.gaussian_process.kernels import Matern

    from bayesianoptimization_b200.fused import lockstep_lbfgsb

    B = bo._lib
    res = {}
    for d, n in ((2, 60), (16, 600), (16, 4096)):
        X, y, rs = late_stage(d, n, 1)
        gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=1.0, length_scale_bounds="fixed"),
                                             alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)
        xc = rs.uniform(size=(10_000, d))
        bounds = np.column_stack([np.zeros(d), np.ones(d)])
        y_max = float(np.max(y))
        ei = -bo.FusedAcquisition(B.ACQ_EI, gp, xi=0.01, y_max=y_max)(xc)
        row = {"N": n, "d": d, "ei_max": float(ei.max()), "frac_ei_zero": float(np.mean(ei == 0.0)),
               "frac_ei_below_1e-12_max": float(np.mean(ei < 1e-12 * ei.max()))}
        for name, code in (("ei", B.ACQ_EI), ("logei", B.ACQ_LOGEI)):
            f = bo.FusedAcquisition(code, gp, xi=0.01, y_max=y_max)
            _, _, top = f.argmin_topk(xc, 5)
            seeds = xc[top]
            runs = lockstep_lbfgsb(f, seeds, bounds)
            le = bo.FusedAcquisition(B.ACQ_LOGEI, gp, xi=0.01, y_max=y_max)
            row[name] = [{"nit": int(r.nit), "moved": float(np.linalg.norm(r.x - s)), "fun": float(np.squeeze(r.fun)),
                          "logei_at_x": float(-le(r.x)[0])} for r, s in zip(runs, seeds)]
        res[f"d{d}_n{n}"] = row
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1 << 20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("logei_bench needs a CUDA device")
    import bayesianoptimization_b200 as bo

    out = {"bench": "logei_vs_ei", "device": device_info(), "rounds": args.rounds,
           "selection": part_a(bo, args), "late_stage": part_b(bo, args)}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

"""A/B of the Gram bound passes of pruning (B200BO_PRUNE_BOUND=f64/f32, DESIGN.md 4.9, 6) in one process, on both
sides of the rule that picks between them (A1 constv 2^-24 <= 1e-3); the fp32 pass with both of its kernels (f32: the
default, predict_bound_gram_reg_kernel at d <= 16; f32-ring: B200BO_PRUNE_GRAM_KERNEL=ring).

  python tools/prune_bound_ab.py [--reps 3] [--calls 3] [--legs c3,b_m25_c3,b_rbf_long]

c3: tools/prune_ab.py's leg (2^20 uniform candidates, EI, argmin + top-10).  b_*: the ill-conditioned fixtures of
tests/golden/illbig_*.npz with their candidates tiled eight times, EI.  Per leg and pass: b200bo_last_kernel_ms mean
(min-max), the stage split of b200bo_last_prune_stage_ms, the evaluated and refined counts, the pass auto picks, and
whether the records (value bits and indices) equal those of the fp64 pass.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from predict_pipe_ab import Sampler, card  # noqa: E402
from prune_ab import ALPHA, K, LEGS, XI  # noqa: E402

STAGES = ("bound", "sort", "lead", "refine", "final", "tiles")
PASSES = ("f64", "f32", "f32-ring")
SWITCHES = ("B200BO_PRUNE_BOUND", "B200BO_PRUNE_GRAM_KERNEL")


def apply_pass(p):
    for v in SWITCHES:
        os.environ.pop(v, None)
    if p:
        os.environ["B200BO_PRUNE_BOUND"] = p.split("-")[0]
        if p.endswith("-ring"):
            os.environ["B200BO_PRUNE_GRAM_KERNEL"] = "ring"


def problem(name):
    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import _lib as B
    from sklearn.gaussian_process.kernels import Matern

    if name in LEGS:
        d, n, ls, kind, kappa, m, source = LEGS[name]
        rs = np.random.RandomState(0)
        X = rs.uniform(size=(n, d))
        y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
        gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=ls), alpha=ALPHA, normalize_y=True,
                                             optimizer=None, device=0).fit(X, y)
        acq = bo.FusedAcquisition(B.ACQ_EI, gp, xi=XI, y_max=float(y.max()))
        return gp, acq, np.random.RandomState(1000).uniform(size=(m, d))
    from oracle import make_illcond as MI
    from oracle import make_illcond_big as MB

    c, r = MB.CASES[name], MB.load(name)
    gp = bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True, optimizer=None,
                                         device=0).fit(r["X"], r["y"])
    acq = bo.FusedAcquisition(B.ACQ_EI, gp, xi=MI.XI, y_max=float(np.max(r["y"])))
    return gp, acq, np.tile(r["xt"], (8, 1))


def leg(name, reps, calls):
    import torch

    from bayesianoptimization_b200 import _lib as B

    L = B.lib()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    gp, acq, x = problem(name)
    spec = acq.spec
    m = x.shape[0]
    xc = torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    sel = torch.zeros((K + 1, 2), dtype=torch.int64, device=dev)
    apply_pass(None)
    auto = C.c_int()
    B.check(L.b200bo_acq_prune_bound_pass(C.byref(spec), C.byref(auto), stream.cuda_stream))

    def call():
        B.check(L.b200bo_acq_eval_dev(C.byref(spec), xc.data_ptr(), m, None, None, None, K, sel.data_ptr(), 0,
                                      stream.cuda_stream))
        ms, ev, tot, ref = C.c_float(), C.c_int64(), C.c_int64(), C.c_int64()
        st = (C.c_float * 6)()
        B.check(L.b200bo_last_kernel_ms(C.byref(ms)))
        B.check(L.b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
        B.check(L.b200bo_last_prune_stage_ms(st, C.byref(ref)))
        return ms.value, list(st), ev.value, ref.value, tot.value, sel.cpu().numpy().copy()

    res = {p: {"ms": [], "st": [], "clocks": []} for p in PASSES}
    for _ in range(reps):
        for p in PASSES:
            apply_pass(p)
            call()
            with Sampler() as smp:
                for _ in range(calls):
                    ms, st, ev, ref, tot, rec = call()
                    res[p]["ms"].append(ms)
                    res[p]["st"].append(st)
            res[p]["clocks"].extend(smp.samples)
            res[p].update(evaluated=ev, refined=ref, total=tot, sel=rec)
    apply_pass(None)
    for p in PASSES:
        t, c, st = np.array(res[p]["ms"]), np.array(res[p]["clocks"]), np.array(res[p]["st"]).mean(0)
        print(json.dumps({
            "leg": name, "B200BO_PRUNE_BOUND": p, "auto_picks": {1: "f64", 2: "f32"}.get(auto.value, "direct"),
            "kernel_ms_mean": round(float(t.mean()), 3),
            "kernel_ms_min_max": [round(float(t.min()), 3), round(float(t.max()), 3)],
            "stage_ms": {k: round(float(v), 3) for k, v in zip(STAGES, st)},
            "evaluated": res[p]["evaluated"], "refined": res[p]["refined"], "total": res[p]["total"],
            "sm_clock_mhz_median": float(np.median(c[:, 0])) if len(c) else None,
            "power_w_median": float(np.median(c[:, 1])) if len(c) else None,
            "records_equal_f64": bool(np.array_equal(res[p]["sel"], res[PASSES[0]]["sel"])),
        }), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--legs", default="c3,b_m25_c3,b_rbf_long")
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for name in filter(None, args.legs.split(",")):
        leg(name, args.reps, args.calls)


if __name__ == "__main__":
    main()

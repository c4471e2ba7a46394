"""Interleaved A/B of selection-only pruning (B200BO_PRUNE=0/1, DESIGN.md 4.9) in one process, then bench.py per
setting, alternated.

  python tools/prune_ab.py [--reps 3] [--calls 3] [--bench-runs 2] [--bench-steps 5] [--bench-warmup 3]

Legs (argmin + top-10 through b200bo_acq_eval_dev unless noted; Matern-2.5, alpha 1e-6, normalize_y):
  c3        d=16, N=4096, l=0.7, EI xi=0.01, 2^20 candidates: reps x (calls per setting), settings alternated
  c2        d=8,  N=1024, l=0.5, EI, 2^20
  c5        d=32, N=8192, l=1.0, UCB kappa=2.576, 2^22 (one call per setting: the unpruned call takes seconds)
  philox    c3 through b200bo_acq_select_philox_dev (candidates generated in the kernel)
  worst     c3 with UCB kappa=100: sigma dominates the value, so the bound prunes little
Per leg and setting: kernel time (b200bo_last_kernel_ms: with pruning the bound pass + sort + evaluation, without the
selection merge), the candidates that went through the N^2 term (b200bo_last_prune_stats), the median SM clock and
power draw sampled read-only by nvidia-smi, and whether the records (value bits and indices) equal those of
B200BO_PRUNE=0.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from predict_pipe_ab import Sampler, card  # noqa: E402

K, ALPHA, XI = 10, 1e-6, 0.01
LEGS = {  # name: d, N, length scale, acquisition, kappa, candidates, source
    "c3": (16, 4096, 0.7, "ei", 0.0, 1 << 20, "dev"),
    "c2": (8, 1024, 0.5, "ei", 0.0, 1 << 20, "dev"),
    "c5": (32, 8192, 1.0, "ucb", 2.576, 1 << 22, "dev"),
    "philox": (16, 4096, 0.7, "ei", 0.0, 1 << 20, "philox"),
    "worst": (16, 4096, 0.7, "ucb", 100.0, 1 << 20, "dev"),
}


def leg(name, reps, calls):
    import torch

    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import _lib as B
    from sklearn.gaussian_process.kernels import Matern

    d, n, ls, kind, kappa, m, source = LEGS[name]
    L = B.lib()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    rs = np.random.RandomState(0)
    X = rs.uniform(size=(n, d))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=ls), alpha=ALPHA, normalize_y=True,
                                         optimizer=None, device=0).fit(X, y)
    code = B.ACQ_EI if kind == "ei" else B.ACQ_UCB
    acq = bo.FusedAcquisition(code, gp, kappa=kappa, xi=XI, y_max=float(y.max()))
    spec = acq.spec
    sel = torch.zeros((K + 1, 2), dtype=torch.int64, device=dev)
    xc = None if source == "philox" else torch.from_numpy(np.random.RandomState(1000).uniform(size=(m, d))).to(dev)
    lo, hi = np.zeros(d), np.ones(d)

    def call():
        if source == "philox":
            B.check(L.b200bo_acq_select_philox_dev(C.byref(spec), 12345, B.as_dp(lo), B.as_dp(hi), m, 0, K,
                                                   sel.data_ptr(), stream.cuda_stream))
        else:
            B.check(L.b200bo_acq_eval_dev(C.byref(spec), xc.data_ptr(), m, None, None, None, K, sel.data_ptr(), 0,
                                          stream.cuda_stream))
        ms, ev, tot = C.c_float(), C.c_int64(), C.c_int64()
        B.check(L.b200bo_last_kernel_ms(C.byref(ms)))
        B.check(L.b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
        return ms.value, ev.value, tot.value, sel.cpu().numpy().copy()

    res = {s: {"ms": [], "clocks": [], "sel": None, "evaluated": None} for s in ("0", "1")}
    for _ in range(reps):
        for s in ("0", "1"):
            os.environ["B200BO_PRUNE"] = s
            call()  # warm-up of this setting
            with Sampler() as smp:
                for _ in range(calls):
                    ms, ev, tot, rec = call()
                    res[s]["ms"].append(ms)
            res[s]["clocks"].extend(smp.samples)
            res[s]["evaluated"], res[s]["total"], res[s]["sel"] = ev, tot, rec
    os.environ.pop("B200BO_PRUNE", None)
    base = float(np.mean(res["0"]["ms"]))
    for s in ("0", "1"):
        t, c = np.array(res[s]["ms"]), np.array(res[s]["clocks"])
        print(json.dumps({
            "leg": name, "B200BO_PRUNE": int(s), "kernel_ms_mean": round(float(t.mean()), 2),
            "kernel_ms": [round(x, 2) for x in t.tolist()], "speedup_vs_prune0": round(base / float(t.mean()), 3),
            "evaluated": res[s]["evaluated"], "total": res[s]["total"],
            "evaluated_frac": res[s]["evaluated"] / res[s]["total"],
            "sm_clock_mhz_median": float(np.median(c[:, 0])) if len(c) else None,
            "power_w_median": float(np.median(c[:, 1])) if len(c) else None,
            "records_equal_prune0": bool(np.array_equal(res[s]["sel"], res["0"]["sel"])),
        }), flush=True)
    del xc, gp, acq
    torch.cuda.empty_cache()


def bench_ab(args):
    for run in range(args.bench_runs):
        for s in ("0", "1"):
            env = dict(os.environ, B200BO_PRUNE=s)
            cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps),
                   "--warmup", str(args.bench_warmup), "--no-cpu-baseline"]
            with Sampler() as smp:
                r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
            line = None
            for ln in r.stdout.splitlines()[::-1]:
                if ln.startswith("{"):
                    line = json.loads(ln)
                    break
            rec = {"leg": "bench", "run": run, "B200BO_PRUNE": int(s), "rc": r.returncode, **smp.medians()}
            if line is not None:
                rec["line"] = line
            else:
                rec["stderr_tail"] = r.stderr[-2000:]
            print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="alternations of the settings at c3")
    ap.add_argument("--calls", type=int, default=3, help="timed launches per setting and alternation at c3")
    ap.add_argument("--legs", default=",".join(LEGS))
    ap.add_argument("--bench-runs", type=int, default=2, help="bench.py runs per setting, alternated (0: none)")
    ap.add_argument("--bench-steps", type=int, default=5)
    ap.add_argument("--bench-warmup", type=int, default=3)
    args = ap.parse_args()

    import torch

    assert torch.cuda.is_available(), "needs a CUDA device"
    print(json.dumps({"leg": "card", **card()}), flush=True)
    for name in filter(None, args.legs.split(",")):
        if name == "c3":
            leg(name, args.reps, args.calls)
        else:
            leg(name, 1, 1 if name == "c5" else 2)
    bench_ab(args)
    print(json.dumps({"leg": "card_after", **card()}), flush=True)


if __name__ == "__main__":
    main()

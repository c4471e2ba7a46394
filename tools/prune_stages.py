"""Where the kernel time of a pruned selection call goes, stage by stage (DESIGN.md 4.9, 6), and the A/B of the refine
stages' switches in one process, then bench.py per setting, alternated.

  python tools/prune_stages.py [--settings 0,1] [--reps 3] [--calls 3] [--legs c3,c2,c5,philox,worst] [--bench-runs 2]

A setting is a value of B200BO_PRUNE_REFINE, or switches joined by '+' (names without B200BO_PRUNE_), e.g. the two
fp32 Gram bound kernels:  --settings GRAM_KERNEL=ring,GRAM_KERNEL=reg

Legs as in tools/prune_ab.py (argmin + top-10; Matern-2.5, alpha 1e-6, normalize_y).  Per leg and setting:
b200bo_last_kernel_ms mean (min-max), the stage split of b200bo_last_prune_stage_ms (bound pass, sort, lead, refine
with its levels, final, whole-tile kernel; mean over the timed calls), the levels' part of the refine stage and the
candidates the refine stage and each level let through (b200bo_last_prune_levels), the candidates that went through the full N^2 term and through
the refine stage, the median SM clock and power draw sampled read-only by nvidia-smi, and whether the records (value
bits and indices) equal those of B200BO_PRUNE=0 (one extra call; --no-exact skips it: at c5 it takes seconds).
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
from prune_ab import ALPHA, K, LEGS, XI  # noqa: E402

STAGES = ("bound", "sort", "lead", "refine", "final", "tiles")
SWITCHES = ("B200BO_PRUNE_REFINE", "B200BO_PRUNE_GRAM_KERNEL")


def setting_env(s):
    """environment variables of a setting: a bare value of B200BO_PRUNE_REFINE, or NAME=V joined by '+'"""
    if "=" not in s:
        return {"B200BO_PRUNE_REFINE": s}
    return {"B200BO_PRUNE_" + k: v for k, v in (kv.split("=", 1) for kv in s.split("+"))}


def apply_setting(s):
    for v in SWITCHES:
        os.environ.pop(v, None)
    os.environ.update(setting_env(s))


def leg(name, settings, reps, calls, exact):
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
    acq = bo.FusedAcquisition(B.ACQ_EI if kind == "ei" else B.ACQ_UCB, gp, kappa=kappa, xi=XI, y_max=float(y.max()))
    spec = acq.spec
    sel = torch.zeros((K + 1, 2), dtype=torch.int64, device=dev)
    xc = None if source == "philox" else torch.from_numpy(np.random.RandomState(1000).uniform(size=(m, d))).to(dev)
    lo, hi = np.zeros(d), np.ones(d)

    def call(stages=True):
        if source == "philox":
            B.check(L.b200bo_acq_select_philox_dev(C.byref(spec), 12345, B.as_dp(lo), B.as_dp(hi), m, 0, K,
                                                   sel.data_ptr(), stream.cuda_stream))
        else:
            B.check(L.b200bo_acq_eval_dev(C.byref(spec), xc.data_ptr(), m, None, None, None, K, sel.data_ptr(), 0,
                                          stream.cuda_stream))
        ms, ev, tot, ref = C.c_float(), C.c_int64(), C.c_int64(), C.c_int64()
        st, lms, passed, nlev = (C.c_float * 6)(), C.c_float(), (C.c_int64 * 5)(), C.c_int()
        B.check(L.b200bo_last_kernel_ms(C.byref(ms)))
        B.check(L.b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
        if stages:
            B.check(L.b200bo_last_prune_stage_ms(st, C.byref(ref)))
            B.check(L.b200bo_last_prune_levels(C.byref(lms), passed, C.byref(nlev)))
        lev = (lms.value, list(passed)[:nlev.value + 1])
        return ms.value, list(st), ev.value, ref.value, tot.value, sel.cpu().numpy().copy(), lev

    ref_sel = None
    if exact:
        os.environ["B200BO_PRUNE"] = "0"
        ref_sel = call(stages=False)[5]
        os.environ.pop("B200BO_PRUNE")
    res = {s: {"ms": [], "st": [], "lev_ms": [], "clocks": []} for s in settings}
    for _ in range(reps):
        for s in settings:
            apply_setting(s)
            call()  # warm-up of this setting
            with Sampler() as smp:
                for _ in range(calls):
                    ms, st, ev, ref, tot, rec, (lev_ms, passed) = call()
                    res[s]["ms"].append(ms)
                    res[s]["st"].append(st)
                    res[s]["lev_ms"].append(lev_ms)
            res[s]["clocks"].extend(smp.samples)
            res[s].update(evaluated=ev, refined=ref, total=tot, sel=rec, passed=passed)
    apply_setting("1")
    os.environ.pop("B200BO_PRUNE_REFINE")
    base = float(np.mean(res[settings[0]]["ms"]))
    for s in settings:
        t, c, st = np.array(res[s]["ms"]), np.array(res[s]["clocks"]), np.array(res[s]["st"]).mean(0)
        print(json.dumps({
            "leg": name, "setting": s, "kernel_ms_mean": round(float(t.mean()), 3),
            "kernel_ms_min_max": [round(float(t.min()), 3), round(float(t.max()), 3)],
            "speedup_vs_first_setting": round(base / float(t.mean()), 3),
            "stage_ms": {k: round(float(v), 3) for k, v in zip(STAGES, st)},
            "levels_ms": round(float(np.mean(res[s]["lev_ms"])), 3), "passed_refine_then_levels": res[s]["passed"],
            "evaluated": res[s]["evaluated"], "refined": res[s]["refined"], "total": res[s]["total"],
            "evaluated_frac": res[s]["evaluated"] / res[s]["total"],
            "refined_frac": res[s]["refined"] / res[s]["total"],
            "sm_clock_mhz_median": float(np.median(c[:, 0])) if len(c) else None,
            "power_w_median": float(np.median(c[:, 1])) if len(c) else None,
            "records_equal_prune0": None if ref_sel is None else bool(np.array_equal(res[s]["sel"], ref_sel)),
        }), flush=True)
    del xc, gp, acq
    torch.cuda.empty_cache()


def bench_ab(args, settings):
    for run in range(args.bench_runs):
        for s in settings:
            env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
            env.update(setting_env(s))
            cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps),
                   "--warmup", str(args.bench_warmup), "--no-cpu-baseline"]
            with Sampler() as smp:
                r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
            line = None
            for ln in r.stdout.splitlines()[::-1]:
                if ln.startswith("{"):
                    line = json.loads(ln)
                    break
            rec = {"leg": "bench", "run": run, "setting": s, "rc": r.returncode, **smp.medians()}
            if line is not None:
                rec["line"] = line
            else:
                rec["stderr_tail"] = r.stderr[-2000:]
            print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--settings", default="0,1", help="settings of the switches (see above), alternated")
    ap.add_argument("--reps", type=int, default=3, help="alternations of the settings at c3")
    ap.add_argument("--calls", type=int, default=3, help="timed launches per setting and alternation at c3")
    ap.add_argument("--legs", default="c3,c2,c5,philox,worst")
    ap.add_argument("--no-exact", action="store_true", help="skip the B200BO_PRUNE=0 call the records are compared to")
    ap.add_argument("--bench-runs", type=int, default=0, help="bench.py runs per setting, alternated")
    ap.add_argument("--bench-steps", type=int, default=5)
    ap.add_argument("--bench-warmup", type=int, default=3)
    args = ap.parse_args()
    settings = [s for s in args.settings.split(",") if s]
    unknown = [x for x in args.legs.split(",") if x and x not in LEGS]
    if unknown or not settings:
        ap.error(f"unknown legs {unknown} or no settings")

    import torch

    assert torch.cuda.is_available(), "needs a CUDA device"
    print(json.dumps({"leg": "card", **card()}), flush=True)
    for name in filter(None, args.legs.split(",")):
        if name == "c3":
            leg(name, settings, args.reps, args.calls, not args.no_exact)
        else:
            leg(name, settings, 1, 1 if name == "c5" else 2, not args.no_exact)
    bench_ab(args, settings)
    print(json.dumps({"leg": "card_after", **card()}), flush=True)


if __name__ == "__main__":
    main()

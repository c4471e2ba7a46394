"""Interleaved A/B of the phase B data paths of predict_acq16_kernel at C3 (d=16, N=4096, Matern-2.5 l=0.7, EI, 2^20
candidates, argmin + top-10), then bench.py per path, all in one process tree.

  python tools/predict_pipe_ab.py [--reps 3] [--calls 3] [--bench-runs 2] [--bench-steps 5] [--bench-warmup 3]

Paths (B200BO_PREDICT_PIPE, read per launch): cpasync = per-thread cp.async under CTA barriers, bulk_nomc (default)
= two bulk copies per stage from padded stage images, bulk = the same with the L^-1 stages multicast across CTA pairs
(clusters of 2).
Prints JSON lines: the card (name, power limit), per path the kernel time (b200bo_last_kernel_ms, CUDA events around
the one launch) with the median SM clock and power draw sampled read-only by nvidia-smi while it ran, whether mu,
sigma, acq and the selection are bit-equal to cpasync, and `bench.py --no-extra --no-cpu-baseline` runs of the three
paths alternated.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, D, LS, M, K = 4096, 16, 0.7, 1 << 20, 10
ALPHA, XI = 1e-6, 0.01
PIPES = ["cpasync", "bulk_nomc", "bulk"]


def smi(query):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return [s.strip() for s in out.split(",")]
    except Exception as e:  # noqa: BLE001
        return [f"error: {e}"]


def card():
    q = "name,power.limit,clocks.max.sm"
    return dict(zip(q.split(","), smi(q)))


class Sampler:
    """nvidia-smi clocks.sm / power.draw every `period` s while active (read-only queries)."""

    def __init__(self, period=0.5):
        self.period, self.samples, self._stop = period, [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.is_set():
            v = smi("clocks.sm,power.draw")
            try:
                self.samples.append((float(v[0]), float(v[1])))
            except (ValueError, IndexError):
                pass
            self._stop.wait(self.period)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()

    def medians(self):
        if not self.samples:
            return {"sm_clock_mhz": None, "power_w": None, "samples": 0}
        a = np.array(self.samples)
        return {"sm_clock_mhz": float(np.median(a[:, 0])), "power_w": float(np.median(a[:, 1])),
                "samples": len(self.samples)}


def kernel_ab(args):
    import torch

    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import _lib as B
    from sklearn.gaussian_process.kernels import Matern

    L = B.lib()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    rs = np.random.RandomState(0)
    X = rs.uniform(size=(N, D))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(N)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=LS), alpha=ALPHA, normalize_y=True,
                                         optimizer=None, device=0).fit(X, y)
    acq = bo.FusedAcquisition(B.ACQ_EI, gp, xi=XI, y_max=float(y.max()))
    spec = acq.spec
    xc = torch.from_numpy(np.random.RandomState(1000).uniform(size=(M, D))).to(dev)
    sel = torch.zeros((K + 1, 2), dtype=torch.int64, device=dev)

    def launch_select():
        B.check(L.b200bo_acq_eval_dev(C.byref(spec), xc.data_ptr(), M, None, None, None, K, sel.data_ptr(), 0,
                                      stream.cuda_stream))
        ms = C.c_float()
        B.check(L.b200bo_last_kernel_ms(C.byref(ms)))
        return ms.value

    def outputs():
        acq_o, mu, sd = (torch.empty(M, dtype=torch.float64, device=dev) for _ in range(3))
        B.check(L.b200bo_acq_eval_dev(C.byref(spec), xc.data_ptr(), M, acq_o.data_ptr(), mu.data_ptr(),
                                      sd.data_ptr(), K, sel.data_ptr(), 0, stream.cuda_stream))
        ms = C.c_float()
        B.check(L.b200bo_last_kernel_ms(C.byref(ms)))
        s = sel.cpu().numpy()
        return {"acq": acq_o.cpu().numpy(), "mu": mu.cpu().numpy(), "sd": sd.cpu().numpy(),
                "sel": s.copy()}

    times = {p: [] for p in PIPES}
    clocks = {p: [] for p in PIPES}
    outs = {}
    for rep in range(args.reps):
        for p in PIPES:
            os.environ["B200BO_PREDICT_PIPE"] = p
            launch_select()  # warm-up of this path
            with Sampler() as smp:
                t = [launch_select() for _ in range(args.calls)]
            times[p].extend(t)
            clocks[p].extend(smp.samples)
            if rep == 0:
                outs[p] = outputs()
    os.environ.pop("B200BO_PREDICT_PIPE", None)
    ref = outs["cpasync"]
    base = float(np.mean(times["cpasync"]))
    for p in PIPES:
        t = np.array(times[p])
        o = outs[p]
        c = np.array(clocks[p]) if clocks[p] else None
        print(json.dumps({
            "leg": "kernel", "B200BO_PREDICT_PIPE": p, "kernel_ms_mean": round(float(t.mean()), 2),
            "kernel_ms_min": round(float(t.min()), 2), "kernel_ms_max": round(float(t.max()), 2),
            "b200bo_last_kernel_ms": [round(x, 2) for x in t.tolist()],
            "speedup_vs_cpasync": round(base / float(t.mean()), 4),
            "cand_per_s": M / (t.mean() * 1e-3),
            "tflops": (N * N + N * (3 * D + 18)) * M / (t.mean() * 1e-3) / 1e12,
            "sm_clock_mhz_median": float(np.median(c[:, 0])) if c is not None else None,
            "power_w_median": float(np.median(c[:, 1])) if c is not None else None,
            "smi_samples": 0 if c is None else len(c),
            "bit_equal_mu_sd_acq": all(np.array_equal(o[k], ref[k]) for k in ("mu", "sd", "acq")),
            "same_selection": bool(np.array_equal(o["sel"], ref["sel"])),
        }), flush=True)


def bench_ab(args):
    for run in range(args.bench_runs):
        for p in PIPES:
            env = dict(os.environ, B200BO_PREDICT_PIPE=p)
            cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps),
                   "--warmup", str(args.bench_warmup), "--no-extra", "--no-cpu-baseline"]
            with Sampler() as smp:
                r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
            line = None
            for ln in r.stdout.splitlines()[::-1]:
                if ln.startswith("{"):
                    line = json.loads(ln)
                    break
            rec = {"leg": "bench", "run": run, "B200BO_PREDICT_PIPE": p, "rc": r.returncode, **smp.medians()}
            if line is not None:
                rec.update({"value": line.get("value"), "kernel_ms": line.get("kernel_ms"),
                            "result": line.get("result")})
            else:
                rec["stderr_tail"] = r.stderr[-2000:]
            print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="alternations of the paths")
    ap.add_argument("--calls", type=int, default=3, help="timed launches per path and alternation")
    ap.add_argument("--bench-runs", type=int, default=2, help="bench.py runs per path, alternated (0: none)")
    ap.add_argument("--bench-steps", type=int, default=5)
    ap.add_argument("--bench-warmup", type=int, default=3)
    args = ap.parse_args()

    import torch

    assert torch.cuda.is_available(), "needs a CUDA device"
    print(json.dumps({"leg": "card", **card()}), flush=True)
    kernel_ab(args)
    bench_ab(args)
    print(json.dumps({"leg": "card_after", **card()}), flush=True)


if __name__ == "__main__":
    main()

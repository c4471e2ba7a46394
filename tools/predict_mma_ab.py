"""Shape table of the fp64 mma.sync instructions (tools/dmma_shapes.cu) and an interleaved A/B of phase B of
predict_acq16_kernel at C3 (d=16, N=4096, Matern-2.5 l=0.7, EI, 2^20 candidates, argmin + top-10), in one process.

  python tools/predict_mma_ab.py [--reps 3] [--calls 3] [--l2]

Phase B variants (B200BO_PREDICT_MMA, read per launch): 884 = the sm_80 shape m8n8k4, 1684 = m16n8k4 (default).
--l2 adds an A/B of the evict_last fraction of the L^-1 loads (B200BO_PREDICT_L2).
Prints JSON lines; the kernel time is b200bo_last_kernel_ms (CUDA events around the one launch).
"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, D, LS, M, K = 4096, 16, 0.7, 1 << 20, 10
ALPHA, XI = 1e-6, 0.01


def shape_table():
    from bayesianoptimization_b200._build import NVCC_FLAGS

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    gencode = NVCC_FLAGS[:2]  # the library's -gencode arch=compute_90a,code=sm_90a
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "dmma_shapes")
        subprocess.run([nvcc, *gencode, "-O3", "-o", exe, os.path.join(ROOT, "tools", "dmma_shapes.cu")], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    rows = [json.loads(line) for line in out.splitlines() if line.strip()]
    for r in rows:
        print(json.dumps({"leg": "shapes", **r}), flush=True)


def card():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="alternations of the variants")
    ap.add_argument("--calls", type=int, default=3, help="timed launches per variant and alternation")
    ap.add_argument("--l2", action="store_true", help="also A/B the evict_last fraction of the L^-1 loads")
    ap.add_argument("--no-shapes", action="store_true")
    args = ap.parse_args()

    import torch

    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import _lib as B
    from sklearn.gaussian_process.kernels import Matern

    assert torch.cuda.is_available(), "needs a CUDA device"
    print(json.dumps({"leg": "card", **card()}), flush=True)
    if not args.no_shapes:
        shape_table()

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
        stream.synchronize()
        s = sel.cpu().numpy()
        return {"acq": acq_o.cpu().numpy(), "mu": mu.cpu().numpy(), "sd": sd.cpu().numpy(),
                "argmin": int(s[0, 1]), "top": [int(t) for t in s[1:, 1]]}

    def ab(var, values, label):
        times = {v: [] for v in values}
        outs = {}
        for rep in range(args.reps):
            for v in values:
                if v is None:
                    os.environ.pop(var, None)
                else:
                    os.environ[var] = v
                launch_select()  # warm-up of this variant
                t = [launch_select() for _ in range(args.calls)]
                times[v].extend(t)
                if rep == 0:
                    outs[v] = outputs()
        os.environ.pop(var, None)
        ref = outs[values[0]]
        for v in values:
            t = np.array(times[v])
            o = outs[v]
            print(json.dumps({
                "leg": label, var: v, "kernel_ms_mean": round(float(t.mean()), 2),
                "kernel_ms_min": round(float(t.min()), 2), "kernel_ms_max": round(float(t.max()), 2),
                "b200bo_last_kernel_ms": [round(x, 2) for x in t.tolist()],
                "cand_per_s": M / (t.mean() * 1e-3),
                "tflops": (N * N + N * (3 * D + 18)) * M / (t.mean() * 1e-3) / 1e12,
                "vs": values[0],
                "max_abs_dmu": float(np.max(np.abs(o["mu"] - ref["mu"]))),
                "max_abs_dsd": float(np.max(np.abs(o["sd"] - ref["sd"]))),
                "max_abs_dacq": float(np.max(np.abs(o["acq"] - ref["acq"]))),
                "same_argmin_top10": o["argmin"] == ref["argmin"] and o["top"] == ref["top"],
            }), flush=True)

    ab("B200BO_PREDICT_MMA", ["884", "1684"], "phase_b_shape")
    if args.l2:
        ab("B200BO_PREDICT_L2", ["1.0", "0.75", "0.5", "none"], "linv_l2_evict_last")
    print(json.dumps({"leg": "card_after", **card()}), flush=True)


if __name__ == "__main__":
    main()

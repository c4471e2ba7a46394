"""Outputs of the Gram bound passes of pruning (DESIGN.md 4.9), written for a byte-for-byte comparison between builds.

  python tools/prune_bound_bits.py --out OUT.npz [--legs c3,c2,c5,b_m25_c3,b_m15_d17,b_rbf_long]
  python tools/prune_bound_bits.py --compare a.npz b.npz

Per leg (the problems of tools/prune_bound_ab.py, EI; the c* legs on the first 2^18 of their candidates), the keys,
(mu_lo, mu_hi) and kmax_lb of b200bo_acq_prune_bound_gram32_dev and of b200bo_acq_prune_bound_gram_dev.  For each fp32
covariance (Matern-1.5, Matern-2.5, RBF), b200bo_cov_f32_dev over every fp32 argument from +0 to twice the clamp, kept
as two position-weighted 64-bit digests of the (k~, z~) bits per 2^26 arguments (the values themselves are GBs).
--compare prints which arrays differ between two such files and exits non-zero if any does.
"""
import argparse
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

M_LEG = 1 << 18
COVS = {"m15": (1, 2300.0), "m25": (2, 1400.0), "rbf": (3, 166.0)}  # code, CovF32::r2max (predict16.cuh)


def bound_outputs(name, out):
    import torch

    from bayesianoptimization_b200 import _lib as B
    from prune_bound_ab import problem

    gp, acq, x = problem(name)
    x = np.ascontiguousarray(x[:M_LEG])
    m = x.shape[0]
    xd = torch.from_numpy(x).cuda()
    s = torch.cuda.current_stream()
    L = B.lib()
    for tag, entry in (("f32", L.b200bo_acq_prune_bound_gram32_dev), ("f64", L.b200bo_acq_prune_bound_gram_dev)):
        key = torch.empty(m, dtype=torch.int64, device="cuda")
        mu = torch.empty((m, 2), dtype=torch.float64, device="cuda")
        kmax_lb = torch.empty(m, dtype=torch.float64, device="cuda")
        B.check(entry(C.byref(acq.spec), xd.data_ptr(), m, key.data_ptr(), mu.data_ptr(), kmax_lb.data_ptr(),
                      s.cuda_stream))
        s.synchronize()
        out[f"{name}/{tag}/key"] = key.cpu().numpy().view(np.uint64)
        out[f"{name}/{tag}/mu"] = mu.cpu().numpy()
        out[f"{name}/{tag}/kmax_lb"] = kmax_lb.cpu().numpy()
    print(f"{name}: m={m}", flush=True)


def cov_digests(cov, out):
    import torch

    from bayesianoptimization_b200 import _lib as B

    code, r2max = COVS[cov]
    fam, nu = {1: (B.KERNEL_MATERN, B.NU_15), 2: (B.KERNEL_MATERN, B.NU_25), 3: (B.KERNEL_RBF, B.NU_25)}[code]
    L, s = B.lib(), torch.cuda.current_stream()
    hi = int(np.float32(2 * r2max).view(np.int32))
    chunk = 1 << 26
    k = torch.empty(chunk, dtype=torch.float32, device="cuda")
    z = torch.empty(chunk, dtype=torch.float32, device="cuda")
    dig = []
    for b0 in range(0, hi + 1, chunk):
        n = min(chunk, hi + 1 - b0)
        bits = torch.arange(b0, b0 + n, dtype=torch.int32, device="cuda")
        B.check(L.b200bo_cov_f32_dev(fam, nu, bits.view(torch.float32).data_ptr(), n, k.data_ptr(), z.data_ptr(),
                                     s.cuda_stream))
        v = (k[:n].view(torch.int32).long() << 32) | (z[:n].view(torch.int32).long() & 0xFFFFFFFF)
        i = bits.long()
        dig.append([int((v * (i * 0x9E3779B97F4A7C1 + 1)).sum()), int((v ^ (i * 0x2545F4914F6CDD1D)).sum())])
    out[f"cov_f32/{cov}"] = np.array(dig, dtype=np.int64)
    print(f"cov_f32 {cov}: {hi + 1} arguments", flush=True)


def compare(a, b):
    A, Bz = np.load(a), np.load(b)
    bad = sorted(set(A.files) ^ set(Bz.files))
    for f in sorted(set(A.files) & set(Bz.files)):
        if A[f].dtype != Bz[f].dtype or A[f].shape != Bz[f].shape or A[f].tobytes() != Bz[f].tobytes():
            bad.append(f)
    print(f"{len(A.files)} / {len(Bz.files)} arrays; differing: {bad if bad else 'none'}")
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="the .npz to write (required unless --compare)")
    ap.add_argument("--legs", default="c3,c2,c5,b_m25_c3,b_m15_d17,b_rbf_long")
    ap.add_argument("--compare", nargs=2, metavar="NPZ")
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not args.out:
        ap.error("--out is required")
    out = {}
    for name in filter(None, args.legs.split(",")):
        bound_outputs(name, out)
    for cov in COVS:
        cov_digests(cov, out)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    np.savez(args.out, **out)
    print(f"wrote {args.out}: {len(out)} arrays", flush=True)


if __name__ == "__main__":
    main()

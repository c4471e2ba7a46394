"""Double-double reference of NEI with pending points (include/b200bo.h b200bo_gp_condition_fantasies, DESIGN.md 4.14)
at production sizes and on ill-conditioned noiseless factors.

Three cases of oracle/make_nei_big.py (c_m25_d3: N = 121, d = 3; b_m15_d17: N = 1000, d = 17; b_m25_c3: N = 4096,
d = 16; each with its WhiteKernel(2^-13) noisy GP and the noiseless GP K0 = c k + tau I, tau = 1e-6), S = 4 draws from
RandomState(SEED) in the order of noiseless_fantasies(pending=..., extra_rows=...): Z, E, then 15 z rows.  The 15
pending rows are, in order: the incumbent's input (the training row of largest y), then a row 1e-3 from a random
training row every third row (4 in all, a quarter), and uniform rows over the box of X between them; p = 1, 7 and 15
take the first p of them (the device runs pending=P[:p], extra_rows=15 - p, so every p sees the same z rows).

Everything is evaluated in double-double arithmetic (oracle/dd.py) in the order of the definition:

  F, W = K^-1 R and best_s of the registered rows as oracle/make_nei_big.py forms them; the factor of K0 extended by the
  pending rows (dd.Fit.extend: the Cholesky rows of K0 over X u P, independent of the device's L^-1 row updates);
  F_js = L0'[n + j, :n + j + 1] [Z; z_1 .. z_j]_s + c k(x_j, X)^T W_s; per p, A' = K0'^-1 F' by substitution with the
  leading n + p block and best_s' = max(best_s, max_{j<p} (s_y F_js + ybar)); at every candidate (the case's candidate
  set, the 15 pending rows and their 1e-7 neighbours) sigma0'^2 = c - |L0'^-1 k*|^2 over the n + p rows,
  mu_s = s_y k*^T a'_s + ybar, and NEI / LogNEI at 50 digits (mpmath's Phi and phi).

The inputs are not stored again: load() rebuilds X, y and the candidates with make_nei_big.inputs() and checks them
against the SHA-256 digests the fixture keeps; P and the neighbours are rebuilt from their seed here.  The fixture,
tests/golden/neibatch_<case>.npz, stores the truth rounded to fp64 and, as the referee, tests/nei_batch_oracle.py's fp64
results on the same draws (keys "sk_*").

Regenerate with

    python -m oracle.make_nei_batch                   # every case of CASES
    python -m oracle.make_nei_batch --only c_m25_d3   # some of them

About four and a half minutes on 8 CPU cores for the three cases (measured: c_m25_d3 15 s, b_m15_d17 58 s, b_m25_c3
3 min 18 s); nothing here needs a GPU.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import mpmath as mp
import numpy as np

from oracle import dd
from oracle import make_illcond as MI
from oracle import make_nei_big as NB

sys.path.insert(0, os.path.join(MI.ROOT, "tests"))
import nei_batch_oracle as NBO  # noqa: E402

CASES = ("c_m25_d3", "b_m15_d17", "b_m25_c3")
S = 4
SEED = 32
P_MAX = 15
PS = (1, 7, 15)
XI = NB.XI


def draws(n):
    """Z, E, then the P_MAX z rows of the pending points."""
    return NBO.draws(np.random.RandomState(SEED), n, S, P_MAX)


def pending(X, y, seed):
    """The P_MAX pending rows (module docstring) and their 1e-7 neighbours."""
    rs = np.random.RandomState(3000 + seed)
    d = X.shape[1]
    lo, hi = X.min(axis=0), X.max(axis=0)
    P = np.empty((P_MAX, d))
    for j in range(P_MAX):
        if j == 0:
            P[j] = X[int(np.argmax(y))]
        elif j % 3 == 1 and j < 12:
            u = rs.randn(d)
            P[j] = X[rs.randint(len(X))] + 1e-3 * u / np.linalg.norm(u)
        else:
            P[j] = lo + (hi - lo) * rs.uniform(size=d)
    u = rs.randn(P_MAX, d)
    return P, P + 1e-7 * u / np.linalg.norm(u, axis=1, keepdims=True)


def _seed(name):
    c = NB.CASES[name]
    base = c["base"]
    return (NB.MB.CASES if base in NB.MB.CASES else MI.CASES)[base]["seed"]


def candidates(name, X, y, xt):
    P, Pn = pending(X, y, _seed(name))
    return P, np.vstack([xt, P, Pn])


def _ei(a, sd):
    z = a / sd
    return a * mp.ncdf(z) + sd * mp.npdf(z)


def truth(name, X, y, xc, P):
    """The double-double pipeline, rounded to fp64 (module docstring)."""
    mp.mp.dps = 50
    noisy, nl, tau = NB.gp_cases(name)
    n = len(X)
    fit0 = dd.Fit(nl, X, y, extra=P_MAX)
    fit = dd.Fit(noisy, X, y)
    ds = mp.mpf(noisy.get("white") or 0.0) + mp.mpf(noisy["alpha"]) - mp.mpf(tau)
    assert ds > 0
    sqp, dsp = dd.from_mp(mp.sqrt(ds)), dd.from_mp(ds)
    yh, yl = fit0.yn
    Z, E, Zp = draws(n)
    Zt, Et = np.ascontiguousarray(Z.T), np.ascontiguousarray(E.T)
    Fp = dd.lower_rows(fit0.L[0], fit0.L[1], Zt, np.zeros_like(Zt), n)
    R = NB._residual(yh, yl, Fp[0], Fp[1], sqp[0], sqp[1], Et)
    W = dd.solve_rows(fit, *R)
    F = NB._combine(yh, yl, sqp[0], sqp[1], Et, dsp[0], dsp[1], *W)
    best = [max(dd.to_mp(F[0][s, i], F[1][s, i]) for i in range(n)) * fit0.y_std + fit0.y_mean for s in range(S)]
    Ps = dd.scaled(nl, P)
    _, Kp = fit0.extend(Ps)
    L0h, L0l = fit0.L
    Za = np.ascontiguousarray(np.vstack([Z, Zp]).T)  # (S, n + P_MAX)
    Fh = np.zeros((S, n + P_MAX))
    Fl = np.zeros((S, n + P_MAX))
    Fh[:, :n], Fl[:, :n] = F
    zl = np.zeros(n + P_MAX)
    for j in range(P_MAX):
        for s in range(S):
            ah, al = dd._dot(L0h[n + j], L0l[n + j], Za[s], zl, 0, n + j + 1)
            bh, bl = dd._dot(Kp[0][j], Kp[1][j], W[0][s], W[1][s], 0, n)
            Fh[s, n + j], Fl[s, n + j] = dd.dd_add(ah, al, bh, bl)
    xs = dd.scaled(nl, xc)
    Ks = fit0.cross(xs, np.vstack([fit0.Xs, Ps]))
    var = fit0.variance(Ks, [n + p for p in PS])
    ys, ym = fit0.y_std, fit0.y_mean
    out = dict(tau=tau, y_std=float(ys))
    for q, p in enumerate(PS):
        m = n + p
        B = (np.ascontiguousarray(Fh[:, :m]), np.ascontiguousarray(Fl[:, :m]))
        V = dd.forward_rows(L0h, L0l, B[0], B[1], m)
        A = dd.backward_rows(L0h, L0l, V[0], V[1], m)
        fP = [[dd.to_mp(Fh[s, n + j], Fl[s, n + j]) * ys + ym for s in range(S)] for j in range(p)]
        bp = [max([best[s]] + [fP[j][s] for j in range(p)]) for s in range(S)]
        K0h, K0l = np.ascontiguousarray(Ks[0][:, :m]), np.ascontiguousarray(Ks[1][:, :m])
        cols = [dd._matvec(K0h, K0l, np.ascontiguousarray(A[0][s]), np.ascontiguousarray(A[1][s])) for s in range(S)]
        nei = []
        for t, v in enumerate(var[q]):
            sd = mp.sqrt(v)
            nei.append(mp.fsum(_ei(dd.to_mp(cols[s][0][t], cols[s][1][t]) * ys + ym - bp[s] - mp.mpf(XI), sd)
                               for s in range(S)) / S)
        out[f"p{p}_F"] = np.array([[float(v) for v in r] for r in fP])
        out[f"p{p}_best"] = np.array([float(v) for v in bp])
        out[f"p{p}_sd0"] = np.array([float(mp.sqrt(v)) for v in var[q]])
        out[f"p{p}_nei"] = np.array([float(v) for v in nei])
        out[f"p{p}_lognei"] = np.array([float(mp.log(v)) if v > 0 else -np.inf for v in nei])
    return out


def referee(name, X, y, xc, P):
    """tests/nei_batch_oracle.py's fp64 results on the same draws."""
    noisy, nl, tau = NB.gp_cases(name)
    kc = MI.sk_kernel(dict(nl, white=None))
    ym, ys = float(np.mean(y)), float(np.std(y)) or 1.0
    yn = (y - ym) / ys
    s2 = float(noisy["alpha"]) + float(noisy.get("white") or 0.0)
    Z, E, Zp = draws(len(X))
    n = len(X)
    out = {}
    for p in PS:
        Fa, A, best = NBO.pending_fantasies(kc, X, P[:p], yn, s2, tau, Z, E, Zp, np.ones(n, bool), ym, ys)
        Xa = np.vstack([X, P[:p]])
        out[f"sk_p{p}_F"] = ys * Fa[n:] + ym
        out[f"sk_p{p}_best"] = best
        out[f"sk_p{p}_sd0"] = NBO.grown_sd(kc, Xa, tau, xc, ys)
        for kind, log in (("nei", False), ("lognei", True)):
            with np.errstate(all="ignore"):
                out[f"sk_p{p}_{kind}"] = NBO.nei(kc, Xa, A, best, tau, xc, XI, ym, ys, log=log)
    return out


def make_case(name):
    X, y, xt, _ = NB.inputs(name)
    P, xc = candidates(name, X, y, xt)
    res = truth(name, X, y, xc, P)
    res.update(referee(name, X, y, xc, P))
    res.update(X_sha256=np.array(NB._digest(X)), y_sha256=np.array(NB._digest(y)),
               xt_sha256=np.array(NB._digest(xt)), P_sha256=np.array(NB._digest(P)))
    return res


def fixture_path(name):
    return os.path.join(MI.GOLDEN, f"neibatch_{name}.npz")


def load(name, path=None):
    """The fixture of a case with its inputs (X, y, the pending rows P and the candidates xc), checked against the
    digests it keeps."""
    with np.load(path or fixture_path(name)) as z:
        r = {k: z[k] for k in z.files}
    X, y, xt, _ = NB.inputs(name)
    P, xc = candidates(name, X, y, xt)
    for k, v in (("X", X), ("y", y), ("xt", xt), ("P", P)):
        if NB._digest(v) != str(r[f"{k}_sha256"]):
            raise ValueError(f"{name}: the inputs {k} differ from those the fixture was computed on")
    r.update(X=X, y=y, P=P, xc=xc)
    return r


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--only", nargs="*", default=None, help="case names (default: all)")
    ap.add_argument("--out", default=MI.GOLDEN)
    a = ap.parse_args(argv)
    for name in a.only or CASES:
        t0 = time.perf_counter()
        res = make_case(name)
        np.savez_compressed(os.path.join(a.out, f"neibatch_{name}.npz"), **res)
        print(f"{name}: min sd0={np.min(res['p15_sd0']):.1e} ({time.perf_counter() - t0:.0f} s)", flush=True)


if __name__ == "__main__":
    main()

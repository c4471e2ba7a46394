"""Double-double reference of noisy expected improvement (include/b200bo.h B200BO_ACQ_NEI / LOGNEI, DESIGN.md 4.13) at
production sizes and on ill-conditioned noiseless factors.

The noisy GP is a case's kernel plus WhiteKernel(2^-13) (b_m05_ard keeps its own WhiteKernel 1e-5), so
sigma_n^2 = alpha + noise; the noiseless GP has K0 = c k(X, X) + tau I with tau = min(alpha, jitter), cond(K0) from
about 1e6 to 1e11.  Every quantity of the definition is evaluated in double-double arithmetic (oracle/dd.py, about 106
bits), in its order:

  the factors L0 of K0 and L of K = c k + sigma_n^2 I; per sample s, F_prior = L0 z_s, R = (y_n - F_prior) - sq e_s,
  K^-1 R, f_s = (y_n - sq e_s) - ds K^-1 R (sq = sqrt(ds), ds = sigma_n^2 - tau), a_s = K0^-1 f_s and best_s, the
  largest s_y f_s + ybar over the incumbent rows; at every candidate sigma0^2 = c - |L0^-1 k*|^2 and
  mu_s = s_y k*^T a_s + ybar; NEI and LogNEI from those at 50 digits (mpmath's Phi and phi); and on 64 rows (the
  training rows, their 1e-7 neighbours, the incumbent's neighbourhood and uniform rows) the input gradients of NEI and
  LogNEI, through u = K0^-1 k* and dd.cross_cov_grad.

The draws are those of noiseless_fantasies (tests/nei_oracle.draws: Z, then E) from RandomState(SEEDS[S]) for
S = 1, 4, 16 with every row an incumbent (runs "s1", "s4", "s16"), and once more at S = 4 with the tenth of the rows of
largest y left out of the incumbent mask ("s4m"), so that best_s moves.

The inputs are not stored again: load() takes X, y and the candidates of a big case from make_illcond_big.load() (X
and the uniform candidates rebuilt from seeds) and of a small case from its tests/golden/illcond_*.npz fixture, and
checks them against the SHA-256 digests the fixture keeps.  The fixture, tests/golden/neibig_<case>.npz, stores the
truth rounded to fp64 and, as the referee, tests/nei_oracle.py's fp64 results on the same draws (keys "sk_*"): F at
F_rows() (both sides of every 64-row block edge, the incumbent row of y and the argmax row of every best_s), best_s,
sigma0, NEI and LogNEI at every candidate, and the gradients on the 64 rows.

Regenerate with

    python -m oracle.make_nei_big                   # every case of CASES
    python -m oracle.make_nei_big --only c_m25_d3   # some of them

About nine minutes on 8 CPU cores for the whole table (measured 8 min 49 s), six of them for the two b_m25_c3 cases;
nothing here needs a GPU.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import sys
import time

import mpmath as mp
import numpy as np
from numba import njit

from oracle import dd
from oracle import make_illcond as MI
from oracle import make_illcond_big as MB

sys.path.insert(0, os.path.join(MI.ROOT, "tests"))
import grad_oracle as GO  # noqa: E402
import nei_oracle as NO  # noqa: E402

NOISE = 2.0 ** -13  # the WhiteKernel added to every case without one of its own
JITTER = 1e-6  # noiseless_fantasies' default
SEEDS = {1: 31, 4: 32, 16: 33}
RUNS = {"s1": (1, False), "s4": (4, False), "s16": (16, False), "s4m": (4, True)}  # name: (S, masked)
XI = MI.XI
CASES = {
    # the C3 shape (N = 4096, d = 16, np = N: no padding), 32 row blocks, 34 candidate tiles
    "b_m25_c3": dict(base="b_m25_c3"),
    # the same with jitter 2^-27 < alpha: tau = 7.5e-9, cond(K0) near 1e11
    "b_m25_c3_j27": dict(base="b_m25_c3", jitter=2.0 ** -27),
    # d = 17: phase A without candidate registers
    "b_m15_d17": dict(base="b_m15_d17"),
    # tau = alpha = 1e-8, cond(K0) about 1e11
    "b_rbf_long": dict(base="b_rbf_long"),
    # ARD with its own WhiteKernel 1e-5: sigma_n^2 - tau = 1e-5 is small
    "b_m05_ard": dict(base="b_m05_ard"),
    # the sets tests/test_gpu_nei.py checks for finiteness, and d = 17 at N = 130
    "c_m25_d3": dict(base="c_m25_d3"),
    "l_m25_d4": dict(base="l_m25_d4"),
    "c_m15_d17": dict(base="c_m15_d17"),
}
SMALL_CASE = "c_m25_d3"
NU = {"m05": 0.5, "m15": 1.5, "m25": 2.5, "rbf": np.inf}


def gp_cases(name, white=None):
    """(noisy, noiseless, tau): the make_illcond case dicts of the noisy GP (alpha, WhiteKernel) and of the noiseless
    one (no WhiteKernel, alpha = tau).  `white` overrides the noise term (0: none)."""
    c = CASES[name]
    base = (MB.CASES if c["base"] in MB.CASES else MI.CASES)[c["base"]]
    w = white if white is not None else (base.get("white") or NOISE)
    noisy = dict(base, white=w or None)
    tau = min(float(base["alpha"]), float(c.get("jitter", JITTER)))
    return noisy, dict(base, white=None, alpha=tau), tau


def incumbent_mask(y, masked):
    """Every row, or every row but the tenth of largest y."""
    mask = np.ones(len(y), dtype=bool)
    if masked:
        mask[np.argsort(y, kind="stable")[-max(1, len(y) // 10):]] = False
    return mask


def grad_rows(group):
    """The 64 gradient rows: the 16 training rows, their 1e-7 neighbours, the incumbent's neighbourhood and the first
    16 uniform rows of make_illcond.problem()'s groups."""
    out = [np.flatnonzero(group == g)[:16] for g in (MI.G_TRAIN, MI.G_DUP7, MI.G_INC, MI.G_UNIFORM)]
    assert all(len(o) == 16 for o in out)
    return np.concatenate(out)


def draws(n, S):
    return NO.draws(np.random.RandomState(SEEDS[S]), n, S)


# ---------------------------------------------------------------------------------------------------------------
# the double-double pipeline
# ---------------------------------------------------------------------------------------------------------------
@njit(cache=False)
def _residual(yh, yl, Fph, Fpl, sqh, sql, E):
    """R[t, i] = (y_i - Fp[t, i]) - sq e[t, i]."""
    m, n = Fph.shape
    Rh = np.zeros((m, n))
    Rl = np.zeros((m, n))
    for t in range(m):
        for i in range(n):
            ah, al = dd.dd_sub(yh[i], yl[i], Fph[t, i], Fpl[t, i])
            bh, bl = dd.dd_mul_d(sqh, sql, E[t, i])
            Rh[t, i], Rl[t, i] = dd.dd_sub(ah, al, bh, bl)
    return Rh, Rl


@njit(cache=False)
def _combine(yh, yl, sqh, sql, E, dsh, dsl, KRh, KRl):
    """F[t, i] = (y_i - sq e[t, i]) - ds (K^-1 R)[t, i]."""
    m, n = KRh.shape
    Fh = np.zeros((m, n))
    Fl = np.zeros((m, n))
    for t in range(m):
        for i in range(n):
            bh, bl = dd.dd_mul_d(sqh, sql, E[t, i])
            ah, al = dd.dd_sub(yh[i], yl[i], bh, bl)
            ch, cl = dd.dd_mul(dsh, dsl, KRh[t, i], KRl[t, i])
            Fh[t, i], Fl[t, i] = dd.dd_sub(ah, al, ch, cl)
    return Fh, Fl


_solve = dd.solve_rows


def _ei(a, sd):
    z = a / sd
    return a * mp.ncdf(z) + sd * mp.npdf(z), mp.ncdf(z), mp.npdf(z)


class Truth:
    """The double-double NEI pipeline of one case (module docstring).  Unrounded: fit0 / fit (dd.Fit of K0 and K),
    and per run F, A ((S, n) pairs: rows are samples), best (mpmath list), mu (mpmath (m, S)); var0 (mpmath list,
    sigma0^2 in data units), nei / lognei per run (mpmath lists); on the gradient rows gi, g_nei / g_lognei per run
    (mpmath (64, d))."""

    def __init__(self, name, X, y, xt, gi, white=None, runs=RUNS):
        mp.mp.dps = 50
        noisy, nl, self.tau = gp_cases(name, white)
        self.noisy, self.nl = noisy, nl
        n = self.n = len(X)
        self.fit0 = fit0 = dd.Fit(nl, X, y)
        s2 = mp.mpf(noisy.get("white") or 0.0) + mp.mpf(noisy["alpha"])
        ds = s2 - mp.mpf(self.tau)
        self.fit = fit0 if ds == 0 else dd.Fit(noisy, X, y)
        sqp, dsp = dd.from_mp(mp.sqrt(ds)), dd.from_mp(ds)
        yh, yl = fit0.yn
        self.runs = {}
        for run, (S, masked) in runs.items():
            Z, E = draws(n, S)
            if ds > 0:
                Zt = np.ascontiguousarray(Z.T)
                Fp = dd.lower_rows(fit0.L[0], fit0.L[1], Zt, np.zeros_like(Zt), n)
                Et = np.ascontiguousarray(E.T)
                R = _residual(yh, yl, Fp[0], Fp[1], sqp[0], sqp[1], Et)
                KR = _solve(self.fit, *R)
                F = _combine(yh, yl, sqp[0], sqp[1], Et, dsp[0], dsp[1], *KR)
            else:  # sigma_n^2 = tau: F = y_n
                F = (np.tile(yh, (S, 1)), np.tile(yl, (S, 1)))
            A = _solve(fit0, *F)
            mask = incumbent_mask(y, masked)
            rows = np.flatnonzero(mask)
            arg = [int(rows[np.lexsort((F[1][s, rows], F[0][s, rows]))[-1]]) for s in range(S)]
            best = [dd.to_mp(F[0][s, i], F[1][s, i]) * fit0.y_std + fit0.y_mean for s, i in enumerate(arg)]
            self.runs[run] = dict(S=S, mask=mask, F=F, A=A, best=best, best_row=np.array(arg))
        self.xs = dd.scaled(nl, xt)
        Ks = fit0.cross(self.xs)
        self.var0 = fit0.variance(Ks, [n])[0]
        for run, r in self.runs.items():
            S, A = r["S"], r["A"]
            cols = [dd._matvec(Ks[0], Ks[1], np.ascontiguousarray(A[0][s]), np.ascontiguousarray(A[1][s]))
                    for s in range(S)]
            r["mu"] = [[dd.to_mp(cols[s][0][t], cols[s][1][t]) * fit0.y_std + fit0.y_mean for s in range(S)]
                       for t in range(len(xt))]
            r["nei"], r["lognei"] = [], []
            for t, v in enumerate(self.var0):
                e = mp.fsum(_ei(m - b - mp.mpf(XI), mp.sqrt(v))[0] for m, b in zip(r["mu"][t], r["best"])) / S
                r["nei"].append(e)
                r["lognei"].append(mp.log(e))
        self.gi = gi
        self._grad(Ks)

    def _grad(self, Ks):
        """d NEI / dx and d LogNEI / dx on the rows gi: d mu_s = s_y sum_i a_si dk*_i, d sigma0^2 = -2 s_y^2 u . dk*
        with u = K0^-1 k*, d sigma0 = d sigma0^2 / (2 sigma0); NEI's the mean of Phi(z_s) d mu_s + phi(z_s) d sigma0,
        LogNEI's that over NEI."""
        fit0, gi = self.fit0, self.gi
        Kg = (np.ascontiguousarray(Ks[0][gi]), np.ascontiguousarray(Ks[1][gi]))
        order = list(self.runs)
        W = tuple(np.concatenate([self.runs[r]["A"][p] for r in order]) for p in (0, 1))
        q = len(W[0])
        U, G = dd.posterior_grad(fit0, self.xs[gi], Kg, W)
        d = G[0].shape[2]
        ys = fit0.y_std
        self.U = U
        off = 0
        for run in order:
            r = self.runs[run]
            S = r["S"]
            r["g_nei"], r["g_lognei"] = [], []
            for k, t in enumerate(gi):
                sd = mp.sqrt(self.var0[t])
                dsd = [-ys * ys * dd.to_mp(G[0][k, q, j], G[1][k, q, j]) / sd for j in range(d)]
                g = [mp.mpf(0)] * d
                for s in range(S):
                    _, cdf, pdf = _ei(r["mu"][t][s] - r["best"][s] - mp.mpf(XI), sd)
                    for j in range(d):
                        dmu = ys * dd.to_mp(G[0][k, off + s, j], G[1][k, off + s, j])
                        g[j] += cdf * dmu + pdf * dsd[j]
                g = [v / S for v in g]
                r["g_nei"].append(g)
                r["g_lognei"].append([v / r["nei"][t] for v in g])
            off += S

    def rounded(self, f_rows_idx):
        """The truth rounded to fp64, as the fixture keys it."""
        fit0 = self.fit0
        out = dict(sd0=np.array([float(mp.sqrt(v)) for v in self.var0]), tau=self.tau, y_std=float(fit0.y_std),
                   grad_rows=self.gi, F_rows=f_rows_idx)
        for run, r in self.runs.items():
            F = r["F"][0] + r["F"][1]
            out[f"{run}_F"] = float(fit0.y_std) * F.T[f_rows_idx] + float(fit0.y_mean)
            out[f"{run}_best"] = np.array([float(v) for v in r["best"]])
            out[f"{run}_best_row"] = r["best_row"]
            out[f"{run}_nei"] = np.array([float(v) for v in r["nei"]])
            out[f"{run}_lognei"] = np.array([float(v) for v in r["lognei"]])
            out[f"{run}_g_nei"] = np.array([[float(v) for v in g] for g in r["g_nei"]])
            out[f"{run}_g_lognei"] = np.array([[float(v) for v in g] for g in r["g_lognei"]])
        return out


def F_rows(n, y, truth_best_rows):
    """Both sides of every 64-row block edge, the last row, the incumbent row of y and the argmax rows of best_s."""
    rows = {n - 1, int(np.argmax(y))}
    for e in range(64, n, 64):
        rows |= {e - 1, e}
    for b in truth_best_rows:
        rows |= {int(v) for v in b}
    return np.array(sorted(rows), dtype=np.int64)


# ---------------------------------------------------------------------------------------------------------------
# the fp64 referee
# ---------------------------------------------------------------------------------------------------------------
def referee(name, X, y, xt, gi, f_rows_idx):
    """tests/nei_oracle.py's fp64 results on the same draws: F at f_rows_idx, best_s, sigma0, NEI, LogNEI and the
    gradients on the rows gi (nei_oracle.nei_value_grad)."""
    noisy, nl, tau = gp_cases(name)
    kc = MI.sk_kernel(dict(nl, white=None))
    Kc = kc(X)
    ym, ys = float(np.mean(y)), float(np.std(y)) or 1.0
    yn = (y - ym) / ys
    s2 = float(noisy["alpha"]) + float(noisy.get("white") or 0.0)
    c = float(nl.get("const") or 1.0)
    Ks = kc(xt, X)
    out = dict(sk_sd0=NO.noiseless_sd(Kc, tau, Ks, c, ys))
    gp0 = GO.GradGP(X, y, NU[nl["kern"]], dd.ls_vec(nl), const=c, noise=0.0, alpha=tau)
    for run, (S, masked) in RUNS.items():
        Z, E = draws(len(X), S)
        F, A, best = NO.fantasies(Kc, yn, s2, tau, Z, E, incumbent_mask(y, masked), ym, ys)
        out[f"sk_{run}_F"] = ys * F[f_rows_idx] + ym
        out[f"sk_{run}_best"] = best
        for kind, log in (("nei", False), ("lognei", True)):
            out[f"sk_{run}_{kind}"] = NO.nei(Ks, A, best, out["sk_sd0"], XI, ym, ys, log=log)
            out[f"sk_{run}_g_{kind}"] = NO.nei_value_grad(gp0, xt[gi], A, best, XI, log=log)[1]
    ev = np.linalg.eigvalsh(Kc + tau * np.eye(len(X)))
    out["cond0"] = float(ev[-1] / ev[0])
    return out


# ---------------------------------------------------------------------------------------------------------------
# inputs, fixtures
# ---------------------------------------------------------------------------------------------------------------
def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype="<f8").tobytes()).hexdigest()


def inputs(name):
    """X, y, the candidates and their groups of a case, from the fixture its base case already has."""
    base = CASES[name]["base"]
    if base in MB.CASES:
        r = MB.load(base)
    else:
        with np.load(MI.fixture_path(base)) as z:
            r = {k: z[k] for k in ("X", "y", "xt", "group")}
    return r["X"], r["y"], r["xt"], r["group"]


def make_case(name, inputs_=None):
    """Every array of the fixture of one case."""
    X, y, xt, group = inputs_ if inputs_ is not None else inputs(name)
    gi = grad_rows(group)
    tr = Truth(name, X, y, xt, gi)
    fr = F_rows(len(X), y, [r["best_row"] for r in tr.runs.values()])
    res = tr.rounded(fr)
    res.update(referee(name, X, y, xt, gi, fr))
    res.update(X_sha256=np.array(_digest(X)), y_sha256=np.array(_digest(y)), xt_sha256=np.array(_digest(xt)))
    return res


def fixture_path(name):
    return os.path.join(MI.GOLDEN, f"neibig_{name}.npz")


def load(name, path=None):
    """The fixture of a case with its inputs (X, y, xt, group), checked against the digests it keeps."""
    with np.load(path or fixture_path(name)) as z:
        r = {k: z[k] for k in z.files}
    X, y, xt, group = inputs(name)
    for k, v in (("X", X), ("y", y), ("xt", xt)):
        if _digest(v) != str(r[f"{k}_sha256"]):
            raise ValueError(f"{name}: the inputs {k} differ from those the fixture was computed on")
    r.update(X=X, y=y, xt=xt, group=group)
    return r


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--only", nargs="*", default=None, help="case names (default: all)")
    ap.add_argument("--out", default=MI.GOLDEN)
    a = ap.parse_args(argv)
    for name in a.only or sorted(CASES):
        t0 = time.perf_counter()
        res = make_case(name)
        np.savez_compressed(os.path.join(a.out, f"neibig_{name}.npz"), **res)
        print(f"{name}: cond(K0)={res['cond0']:.2e} tau={res['tau']:.1e} "
              f"min sd0={np.min(res['sd0']):.1e} ({time.perf_counter() - t0:.0f} s)", flush=True)


if __name__ == "__main__":
    main()

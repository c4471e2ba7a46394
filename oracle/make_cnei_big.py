"""Double-double reference of constrained noisy expected improvement (include/b200bo.h B200BO_ACQ_CNEI / LOGCNEI,
DESIGN.md 4.15), alone and with pending points (b200bo_gp_set_constrained_incumbent, DESIGN.md 4.16), at production
sizes and on ill-conditioned noiseless factors.

Each case takes a case of oracle/make_nei_big.py (its X, y, candidates and target GP: the kernel plus WhiteKernel 2^-13,
noiseless K0 = c k + tau I) and adds J constraint GPs on the same X (CASES: every covariance code, ARD and isotropic,
noisy and noiseless - sigma_n^2 = tau, so that F_j is the observed values - and every bound shape).  Constraint j's y is
a polynomial in X (exact IEEE arithmetic) plus 0.02 N(0, 1) noise from RandomState(4000 + seed), rebuilt on load and
checked against the SHA-256 digest the fixture keeps.

The draws are the class's: per GP in order (the target, then constraint 0 .. J-1) Z, E (cnei_oracle.draws) for p = 0,
and Z, E, then 15 z rows (cnei_batch_oracle.draws) with pending rows, from make_nei_big.SEEDS[S] and make_nei_batch.SEED,
so that the target's fantasies are those of the neibig / neibatch fixtures.  Runs: "s4" and "s16" (p = 0), "s4f" (s4's
draws with constraint 0's bound tightened so that at least one sample has no eligible row: the floor), and "p1", "p7",
"p15" at S = 4 with make_nei_batch.pending()'s rows.  The in-bounds mask marks the registered row of largest y and the
third pending row (p >= 7) as outside the parameter bounds.

Every quantity of the definition is evaluated in double-double arithmetic (oracle/dd.py) in its order: each GP's F and
F' over X u P (make_nei_batch's pipeline, with dd.Fit.extend), A' = K0'^-1 F'; the eligibility mask, best_s (the largest
eligible target fantasy, or the smallest over every row when none is eligible) and its row; sigma0 of every GP; the
means mu_js and, at 50 digits with mpmath, P_js = Phi(u) - Phi(l) (reflected into the lower tail), CNEI and LogCNEI =
log CNEI, so that deep tails are exact; on make_nei_big.grad_rows' 64 rows (runs s4, s4f, s16) the input gradients of
both kinds, per GP through dd.posterior_grad and the product rule in mpmath.  The candidates are the case's candidate
set (4296 rows on the big cases), the 15 pending rows and their 1e-7 neighbours (make_nei_batch.candidates()).

Bounds without ties: each finite bound starts at a quantile of the observed constraint values (about 40 % of the rows
eligible over all constraints) and moves to the midpoint of the nearest gap of at least 4e-6 y_std_j between the sorted
fantasy values of that constraint over every run; the generator asserts that every fantasy lies at least 1e-6 y_std_j
from every finite bound, so the device's eligibility must equal the truth's exactly.

The fixture, tests/golden/cneibig_<case>.npz, stores the truth rounded to fp64 and, as the referee, tests/cnei_oracle.py's
and tests/cnei_batch_oracle.py's fp64 results on the same draws with their own incumbents (keys "sk_*").  Self-checks:
with every bound at +-inf and every row in bounds, the target's pipeline reproduces the neibig_<case> NEI / LogNEI
(s4, s16) and neibatch_<case> values (p1, p7, p15) bit for bit where those fixtures exist; the floor occurs in s4f; on
c_m25_d3 a pending run has a sample whose incumbent is a pending row (elsewhere the count is stored); the out-of-bounds rows are never eligible.

Regenerate with

    python -m oracle.make_cnei_big                   # every case of CASES
    python -m oracle.make_cnei_big --only c_m25_d3   # some of them

Measured on 8 CPU cores with the four cases run as four processes at once (one --only each): 19 min 20 s wall, of it
c_m25_d3 95 s, b_rbf_long 609 s, b_m15_d17 773 s and b_m25_c3 1157 s; most of the time is the 50-digit mpmath values,
which run on one core per process.  The sequential time of one process over the whole table is not measured.  Nothing
here needs a GPU.
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
from oracle import make_nei_batch as NBB
from oracle import make_nei_big as NB

sys.path.insert(0, os.path.join(MI.ROOT, "tests"))
import cnei_batch_oracle as CBO  # noqa: E402
import cnei_oracle as CO  # noqa: E402
import nei_oracle as NO  # noqa: E402

NOISE = NB.NOISE
JITTER = NB.JITTER
XI = NB.XI
S_PEND = NBB.S
P_MAX = NBB.P_MAX
PS = NBB.PS
PEND_OUT = 2  # the pending row marked outside the parameter bounds (p >= 7)
# name: (S, seed, p); s4f is s4's draws with the tightened bounds
RUNS = {"s4": (4, NB.SEEDS[4], 0), "s16": (16, NB.SEEDS[16], 0), "s4f": (4, NB.SEEDS[4], 0),
        **{f"p{p}": (S_PEND, NBB.SEED, p) for p in PS}}
GRAD_RUNS = ("s4", "s16", "s4f")
ELIGIBLE = 0.4  # the fraction of rows the starting quantiles keep over all finite bounds
MARGIN = 1e-6  # every fantasy at least this times y_std_j from every finite bound
ARD16 = [1.0, 2.0] * 8

# Constraint GPs: kern / ls / const / white as in make_illcond.CASES (ls and const powers of two), alpha (default 1e-6),
# bound: "ub" (-inf, ub], "lb" [lb, +inf), "both" [lb, ub], "none" (-inf, +inf).  white None with alpha = 1e-6 = jitter:
# sigma_n^2 = tau, the GP is its own noiseless GP and F_j is the observed values.
CASES = {
    # N = 4096, d = 16: 32 row blocks, 34 candidate tiles
    "b_m25_c3": [dict(kern="rbf", ls=2.0, const=2.0, white=NOISE, bound="ub"),
                 dict(kern="m15", ls=ARD16, white=NOISE, bound="both")],
    # N = 1000, d = 17: phase A without candidate registers
    "b_m15_d17": [dict(kern="rbf", ls=2.0, white=NOISE, bound="ub"),
                  dict(kern="m25", ls=2.0, white=None, bound="both"),
                  dict(kern="m15", ls=2.0, white=NOISE, bound="lb")],
    # N = 2000, d = 6, the target's cond(K0) about 1e11
    "b_rbf_long": [dict(kern="m25", ls=1.0, white=NOISE, bound="both")],
    # N = 121, d = 3, J = 7 (B200BO_MAX_GPS - 1): every covariance code and bound shape
    "c_m25_d3": [dict(kern="m05", ls=[0.5, 1.0, 2.0], const=4.0, white=1e-5, bound="ub"),
                 dict(kern="m15", ls=1.0, white=None, bound="lb"),
                 dict(kern="m25", ls=1.0, white=NOISE, bound="both"),
                 dict(kern="rbf", ls=1.0, const=2.0, white=None, bound="none"),
                 dict(kern="m05", ls=1.0, white=NOISE, bound="both"),
                 dict(kern="m15", ls=[1.0, 0.5, 2.0], white=NOISE, bound="ub"),
                 dict(kern="rbf", ls=[0.5, 1.0, 1.0], white=None, bound="lb")],
}
SMALL_CASE = "c_m25_d3"


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def _seed(name):
    return NBB._seed(name)


def constraint_y(name, X):
    """(J, n): constraint j's observed values, a polynomial in X (exact IEEE operations, column by column) plus noise."""
    n, d = X.shape
    rs = np.random.RandomState(4000 + _seed(name))
    out = []
    for j in range(len(CASES[name])):
        t = np.zeros(n)
        for k in range(d):
            t = t + (((k + 2 * j) % 5) - 2) * 0.25 * X[:, k]
        out.append(t - 0.3 * t * t + 0.5 * X[:, j % d] + 0.02 * rs.standard_normal(n))
    return np.array(out)


def gp_specs(name, d):
    """Per GP (the target, then every constraint): (noisy case dict, noiseless case dict, tau)."""
    out = [NB.gp_cases(name)]
    for c in CASES[name]:
        noisy = dict(kern=c["kern"], d=d, ls=c["ls"], const=c.get("const"), white=c.get("white"),
                     alpha=c.get("alpha", 1e-6))
        tau = min(float(noisy["alpha"]), JITTER)
        out.append((noisy, dict(noisy, white=None, alpha=tau), tau))
    return out


def inputs(name):
    """X, y, the constraint values Yc (J, n), the candidates xt, the pending rows P and every candidate xc."""
    X, y, xt, group = NB.inputs(name)
    P, xc = NBB.candidates(name, X, y, xt)
    return X, y, constraint_y(name, X), xt, group, P, xc


def in_bounds(n, y):
    """(n + P_MAX,) the in-bounds mask: the registered row of largest y and pending row PEND_OUT are outside."""
    m = np.ones(n + P_MAX, dtype=bool)
    m[int(np.argmax(y))] = False
    m[n + PEND_OUT] = False
    return m


def draws(name, run, n):
    """Per GP (Z, E, Zp) of a run, Zp None for p = 0."""
    S, seed, p = RUNS[run]
    J = len(CASES[name])
    rs = np.random.RandomState(seed)
    if p == 0:
        return [(Z, E, None) for Z, E in CO.draws(rs, n, S, J)]
    return CBO.draws(rs, n, S, J, P_MAX)


# ---------------------------------------------------------------------------------------------------------------
# the double-double pipeline of one GP
# ---------------------------------------------------------------------------------------------------------------
def _mp(pair, *idx):
    return dd.to_mp(pair[0][idx], pair[1][idx])


class GP:
    """One GP's double-double pipeline over every run: per run F (pair, (S, n + p), normalised), the data-unit
    fantasies Fd (mpmath, [s][row]), the means mu ([t][s], data units); var ([p] -> list over candidates);
    on the gradient rows, per p = 0 run dmu ([k][s][j]) and dsd ([k][j])."""

    def __init__(self, spec, X, y, P, xc, gi, run_draws, grad=True):
        mp.mp.dps = 50
        noisy, nl, tau = spec
        n = self.n = len(X)
        self.fit0 = fit0 = dd.Fit(nl, X, y, extra=P_MAX)
        ds = mp.mpf(noisy.get("white") or 0.0) + mp.mpf(noisy["alpha"]) - mp.mpf(tau)
        fit = fit0 if ds == 0 else dd.Fit(noisy, X, y)
        sqp, dsp = dd.from_mp(mp.sqrt(ds)), dd.from_mp(ds)
        yh, yl = fit0.yn
        self.ys, self.ym = ys, ym = fit0.y_std, fit0.y_mean
        Ps = dd.scaled(nl, P)
        _, Kp = fit0.extend(Ps)
        L0h, L0l = fit0.L
        xs = dd.scaled(nl, xc)
        Ks = fit0.cross(xs, np.vstack([fit0.Xs, Ps]))
        ends = [n] + [n + p for p in PS]
        var = fit0.variance(Ks, ends)
        self.var = dict(zip([0, *PS], var))
        self.F, self.Fd, self.mu, self.A = {}, {}, {}, {}
        for run, (Z, E, Zp) in run_draws.items():
            S, _, p = RUNS[run]
            Zt, Et = np.ascontiguousarray(Z.T), np.ascontiguousarray(E.T)
            Fp = dd.lower_rows(L0h, L0l, Zt, np.zeros_like(Zt), n)
            R = NB._residual(yh, yl, Fp[0], Fp[1], sqp[0], sqp[1], Et)
            W = dd.solve_rows(fit, *R)
            F = NB._combine(yh, yl, sqp[0], sqp[1], Et, dsp[0], dsp[1], *W)
            m = n + p
            if p:
                Za = np.ascontiguousarray(np.vstack([Z, Zp[:p]]).T)
                Fh, Fl = np.zeros((S, m)), np.zeros((S, m))
                Fh[:, :n], Fl[:, :n] = F
                zl = np.zeros(m)
                for j in range(p):
                    for s in range(S):
                        ah, al = dd._dot(L0h[n + j], L0l[n + j], Za[s], zl, 0, n + j + 1)
                        bh, bl = dd._dot(Kp[0][j], Kp[1][j], W[0][s], W[1][s], 0, n)
                        Fh[s, n + j], Fl[s, n + j] = dd.dd_add(ah, al, bh, bl)
                F = (Fh, Fl)
            V = dd.forward_rows(L0h, L0l, np.ascontiguousarray(F[0]), np.ascontiguousarray(F[1]), m)
            A = dd.backward_rows(L0h, L0l, V[0], V[1], m)
            K0h, K0l = np.ascontiguousarray(Ks[0][:, :m]), np.ascontiguousarray(Ks[1][:, :m])
            cols = [dd._matvec(K0h, K0l, np.ascontiguousarray(A[0][s]), np.ascontiguousarray(A[1][s]))
                    for s in range(S)]
            self.F[run], self.A[run] = F, A
            self.Fd[run] = [[_mp(F, s, i) * ys + ym for i in range(m)] for s in range(S)]
            self.mu[run] = [[_mp(cols[s], t) * ys + ym for s in range(S)] for t in range(len(xc))]
        self.dmu, self.dsd = {}, {}
        if grad:
            self._grad(xs, Ks, gi, [r for r in GRAD_RUNS if r in run_draws])

    def _grad(self, xs, Ks, gi, runs):
        n, fit0, ys = self.n, self.fit0, self.ys
        Kg = (np.ascontiguousarray(Ks[0][gi, :n]), np.ascontiguousarray(Ks[1][gi, :n]))
        W = tuple(np.ascontiguousarray(np.concatenate([self.A[r][p] for r in runs])) for p in (0, 1))
        q = len(W[0])
        _, G = dd.posterior_grad(fit0, xs[gi], Kg, W)
        d = G[0].shape[2]
        self.dsd = [[-ys * ys * _mp(G, k, q, j) / mp.sqrt(self.var[0][t]) for j in range(d)]
                    for k, t in enumerate(gi)]
        off = 0
        for r in runs:
            S = len(self.A[r][0])
            self.dmu[r] = [[[ys * _mp(G, k, off + s, j) for j in range(d)] for s in range(S)] for k in range(len(gi))]
            off += S


def _ei(a, sd):
    z = a / sd
    return a * mp.ncdf(z) + sd * mp.npdf(z), mp.ncdf(z), mp.npdf(z)


def _factor(lb, ub, m, sd):
    """(P, dP/dm, dP/dsd) of Phi((ub - m)/sd) - Phi((lb - m)/sd), reflected into the lower tail when both bounds lie
    above the mean's upper tail, so that the 50-digit difference keeps its digits."""
    u = (mp.mpf(ub) - m) / sd if ub != np.inf else mp.inf
    l = (mp.mpf(lb) - m) / sd if lb != -np.inf else -mp.inf
    if l > 0:
        p = mp.ncdf(-l) - mp.ncdf(-u)
    else:
        p = mp.ncdf(u) - mp.ncdf(l)
    fu = mp.npdf(u) if ub != np.inf else mp.mpf(0)
    fl = mp.npdf(l) if lb != -np.inf else mp.mpf(0)
    dm = -(fu - fl) / sd
    dsd = -((u * fu if ub != np.inf else 0) - (l * fl if lb != -np.inf else 0)) / sd
    return p, dm, dsd


# ---------------------------------------------------------------------------------------------------------------
# the truth of one case
# ---------------------------------------------------------------------------------------------------------------
def eligibility(gps, run, lb, ub, inb):
    """(n + p, S) eligible mask (truth): in bounds and lb_j <= F_j <= ub_j in every constraint."""
    S, _, p = RUNS[run]
    m = gps[0].n + p
    ok = np.repeat(inb[:m, None], S, axis=1)
    for j, g in enumerate(gps[1:]):
        lo, hi = mp.mpf(lb[j]), mp.mpf(ub[j])
        for s in range(S):
            for i in range(m):
                if ok[i, s] and not (lo <= g.Fd[run][s][i] <= hi):
                    ok[i, s] = False
    return ok


def incumbents(g0, run, ok):
    """best_s (mpmath), its row, and whether sample s fell to the floor."""
    S = len(ok[0])
    best, rows, floor = [], [], []
    for s in range(S):
        v = g0.Fd[run][s]
        cand = np.flatnonzero(ok[:, s])
        if len(cand):
            i = max(cand, key=lambda r: v[r])
            floor.append(False)
        else:
            i = min(range(len(v)), key=lambda r: v[r])
            floor.append(True)
        best.append(v[i])
        rows.append(int(i))
    return best, np.array(rows), np.array(floor)


def values(gps, run, best, lb, ub, rows=None):
    """CNEI and LogCNEI (mpmath lists) at the candidates `rows` (default all)."""
    S, _, p = RUNS[run]
    g0 = gps[0]
    rows = range(len(g0.mu[run])) if rows is None else rows
    cnei, logcnei = [], []
    for t in rows:
        sds = [mp.sqrt(g.var[p][t]) for g in gps]
        terms = []
        for s in range(S):
            v = _ei(g0.mu[run][t][s] - best[s] - mp.mpf(XI), sds[0])[0]
            for j, g in enumerate(gps[1:]):
                if lb[j] == -np.inf and ub[j] == np.inf:
                    continue
                v *= _factor(lb[j], ub[j], g.mu[run][t][s], sds[j + 1])[0]
            terms.append(v)
        e = mp.fsum(terms) / S
        cnei.append(e)
        logcnei.append(mp.log(e) if e > 0 else mp.mpf("-inf"))
    return cnei, logcnei


def gradients(gps, run, best, lb, ub, gi, cnei):
    """d CNEI / dx and d LogCNEI / dx (mpmath, [k][j]) on the gradient rows: per sample the product rule over
    EI_s and the factors P_js, averaged over s; LogCNEI's is that over CNEI."""
    S, _, _ = RUNS[run]
    g0 = gps[0]
    d = len(g0.dsd[0])
    out_c, out_l = [], []
    for k, t in enumerate(gi):
        sds = [mp.sqrt(g.var[0][t]) for g in gps]
        grad = [mp.mpf(0)] * d
        for s in range(S):
            e, cdf, pdf = _ei(g0.mu[run][t][s] - best[s] - mp.mpf(XI), sds[0])
            f = [e] + [mp.mpf(1)] * (len(gps) - 1)
            df = [[cdf * g0.dmu[run][k][s][j] + pdf * g0.dsd[k][j] for j in range(d)]]
            for q, g in enumerate(gps[1:]):
                if lb[q] == -np.inf and ub[q] == np.inf:
                    df.append([mp.mpf(0)] * d)
                    continue
                p, dm, dsd = _factor(lb[q], ub[q], g.mu[run][t][s], sds[q + 1])
                f[q + 1] = p
                df.append([dm * g.dmu[run][k][s][j] + dsd * g.dsd[k][j] for j in range(d)])
            for a in range(len(gps)):
                rest = mp.mpf(1)
                for b in range(len(gps)):
                    if b != a:
                        rest *= f[b]
                for j in range(d):
                    grad[j] += df[a][j] * rest
        grad = [v / S for v in grad]
        out_c.append(grad)
        out_l.append([v / cnei[t] for v in grad])
    return out_c, out_l


def _gap_bound(v, b, scale):
    """The midpoint of the gap of the sorted values v nearest to b that is at least 4 MARGIN scale wide."""
    k = int(np.searchsorted(v, b))
    for step in range(len(v)):
        for q in (k + step, k - step):
            if 0 < q < len(v) and v[q] - v[q - 1] >= 4 * MARGIN * scale:
                return 0.5 * (v[q - 1] + v[q])
    raise AssertionError("no gap wide enough for a bound")


def choose_bounds(name, gps, Yc, inb):
    """(lb, ub, lb_f, ub_f): the bounds from quantiles moved into gaps, and the tightened ones of run s4f."""
    J = len(CASES[name])
    shapes = [c["bound"] for c in CASES[name]]
    nfin = sum(1 for b in shapes if b != "none")
    q = ELIGIBLE ** (1.0 / max(nfin, 1))
    lb, ub = np.full(J, -np.inf), np.full(J, np.inf)
    for j, shape in enumerate(shapes):
        fv = np.sort(np.concatenate([np.array([float(x) for row in gps[j + 1].Fd[r] for x in row])
                                     for r in RUNS if r != "s4f"]))
        sc = float(gps[j + 1].ys)
        if shape in ("lb", "both"):
            lb[j] = _gap_bound(fv, np.quantile(Yc[j], (1 - q) / (2 if shape == "both" else 1)), sc)
        if shape in ("ub", "both"):
            ub[j] = _gap_bound(fv, np.quantile(Yc[j], 1 - (1 - q) / (2 if shape == "both" else 1)), sc)
    # s4f: constraint 0's upper bound between the smallest and second smallest over s of the least F_0 among the rows
    # every other condition admits, so that one sample keeps eligible rows and the others fall to the floor
    ok = eligibility(gps, "s4", np.r_[lb[:0], -np.inf, lb[1:]], np.r_[ub[:0], np.inf, ub[1:]], inb)
    F0 = np.array([[float(x) for x in row] for row in gps[1].Fd["s4"]]).T  # (n, S)
    ok &= F0 >= lb[0]
    least = np.sort(np.where(ok, F0, np.inf).min(axis=0))
    assert np.isfinite(least[1]), name
    fv = np.sort(np.concatenate([np.array([float(x) for row in gps[1].Fd[r] for x in row]) for r in RUNS
                                 if r != "s4f"]))
    ub_f = ub.copy()
    ub_f[0] = _gap_bound(fv, 0.5 * (least[0] + least[1]), float(gps[1].ys))
    assert least[0] < ub_f[0] < least[1], name
    return lb, ub, lb.copy(), ub_f


def run_bounds(run, b):
    lb, ub, lb_f, ub_f = b
    return (lb_f, ub_f) if run == "s4f" else (lb, ub)


class Truth:
    """The double-double CNEI pipeline of one case (module docstring); `cons` False: the target's alone with every
    bound at +-inf (the identity with the NEI fixtures)."""

    def __init__(self, name, X, y, Yc, xc, P, gi, cons=True, runs=RUNS):
        specs = gp_specs(name, X.shape[1])
        if not cons:
            specs = specs[:1]
        n = len(X)
        self.runs = runs
        rd = {r: draws(name, r, n) for r in runs if r != "s4f"}
        ys = [y] + list(Yc)
        self.gps = []
        for g, spec in enumerate(specs):
            self.gps.append(GP(spec, X, ys[g], P, xc, gi, {r: v[g] for r, v in rd.items()}, grad=cons))
            if "s4f" in runs:
                self._alias(self.gps[-1])
        self.inb = in_bounds(n, y)
        J = len(specs) - 1
        self.bounds = choose_bounds(name, self.gps, Yc, self.inb) if J else (np.zeros(0),) * 4
        self.res = {}
        for run in runs:
            lb, ub = run_bounds(run, self.bounds)
            inb = self.inb if J else np.ones_like(self.inb)
            ok = eligibility(self.gps, run, lb, ub, inb)
            best, rows, floor = incumbents(self.gps[0], run, ok)
            cnei, logcnei = values(self.gps, run, best, lb, ub)
            r = dict(ok=ok, best=best, best_row=rows, floor=floor, cnei=cnei, logcnei=logcnei)
            if cons and run in GRAD_RUNS:
                r["g_cnei"], r["g_logcnei"] = gradients(self.gps, run, best, lb, ub, gi, cnei)
            self.res[run] = r

    @staticmethod
    def _alias(g):
        for d in (g.F, g.Fd, g.mu, g.A, g.dmu):
            if "s4" in d:
                d["s4f"] = d["s4"]

    def F_rows(self, y):
        n = self.gps[0].n
        return NB.F_rows(n, y, [r["best_row"][r["best_row"] < n] for r in self.res.values()])

    def rounded(self, y, gi):
        fr = self.F_rows(y)
        n = self.gps[0].n
        out = dict(grad_rows=gi, F_rows=fr, y_std=np.array([float(g.ys) for g in self.gps]),
                   lb=self.bounds[0], ub=self.bounds[1], lb_f=self.bounds[2], ub_f=self.bounds[3], inb=self.inb)
        for run, r in self.res.items():
            p = RUNS[run][2]
            rows = np.concatenate([fr, np.arange(n, n + p)])
            out[f"{run}_F"] = np.array([[[float(g.Fd[run][s][i]) for s in range(len(r["best"]))] for i in rows]
                                        for g in self.gps])
            out[f"{run}_ok"] = r["ok"]
            out[f"{run}_best"] = np.array([float(v) for v in r["best"]])
            out[f"{run}_best_row"] = r["best_row"]
            out[f"{run}_floor"] = r["floor"]
            out[f"{run}_cnei"] = np.array([float(v) for v in r["cnei"]])
            out[f"{run}_logcnei"] = np.array([float(v) for v in r["logcnei"]])
            for k in ("g_cnei", "g_logcnei"):
                if k in r:
                    out[f"{run}_{k}"] = np.array([[float(v) for v in g] for g in r[k]])
        return out


# ---------------------------------------------------------------------------------------------------------------
# the fp64 referee
# ---------------------------------------------------------------------------------------------------------------
def referee(name, X, y, Yc, xc, P, tr):
    """tests/cnei_oracle.py (p = 0) and tests/cnei_batch_oracle.py (pending rows) in fp64 on the same draws, with their
    own fantasies and incumbents: F at the stored rows, best_s, the eligibility mask, CNEI and LogCNEI."""
    n = len(X)
    specs = gp_specs(name, X.shape[1])
    gps = []
    for (noisy, nl, tau), yg in zip(specs, [y] + list(Yc)):
        ym, ys = float(np.mean(yg)), float(np.std(yg)) or 1.0
        gps.append(dict(kc=MI.sk_kernel(dict(nl, white=None)), y_n=(yg - ym) / ys, y_mean=ym, y_std=ys, tau=tau,
                        s2=float(noisy["alpha"]) + float(noisy.get("white") or 0.0), c=float(nl.get("const") or 1.0)))
    fr = tr.F_rows(y)
    out = {}
    for run in RUNS:
        S, _, p = RUNS[run]
        lb, ub = run_bounds(run, tr.bounds)
        dr = draws(name, run, n)
        inb = tr.inb[:n + p]
        if p == 0:
            st = []
            for g, (Z, E, _) in zip(gps, dr):
                Kc = g["kc"](X)
                F, A, _ = NO.fantasies(Kc, g["y_n"], g["s2"], g["tau"], Z, E, np.ones(n, bool), g["y_mean"],
                                       g["y_std"])
                Ks = g["kc"](xc, X)
                st.append((g["y_std"] * F + g["y_mean"], A, Ks, NO.noiseless_sd(Kc, g["tau"], Ks, g["c"], g["y_std"])))
            ok = CO.eligible(inb, [s[0] for s in st[1:]], lb, ub)
            best = CO.incumbents(st[0][0], ok)
            for kind, log in (("cnei", False), ("logcnei", True)):
                with np.errstate(all="ignore"):
                    out[f"sk_{run}_{kind}"] = CO.cnei(
                        st[0][2], st[0][1], best, st[0][3], XI, [s[2] for s in st[1:]], [s[1] for s in st[1:]],
                        [s[3] for s in st[1:]], lb, ub, gps[0]["y_mean"], gps[0]["y_std"],
                        [g["y_mean"] for g in gps[1:]], [g["y_std"] for g in gps[1:]], log=log)
            Fd = [s[0] for s in st]
        else:
            grown = [CBO.grown(g, X, P[:p], Z, E, Zp) for g, (Z, E, Zp) in zip(gps, dr)]
            Fd = [CBO.data_units(F, g) for (F, _), g in zip(grown, gps)]
            best, ok = CBO.incumbents(Fd[0], Fd[1:], inb, lb, ub)
            Xa = np.vstack([X, P[:p]])
            for kind, log in (("cnei", False), ("logcnei", True)):
                with np.errstate(all="ignore"):
                    out[f"sk_{run}_{kind}"] = CBO.cnei(gps, Xa, [A for _, A in grown], best, xc, XI, lb, ub, log=log)
        rows = np.concatenate([fr, np.arange(n, n + p)])
        out[f"sk_{run}_F"] = np.array([F[rows] for F in Fd])
        out[f"sk_{run}_best"] = best
        out[f"sk_{run}_ok"] = ok
    return out


# ---------------------------------------------------------------------------------------------------------------
# self-checks, fixtures
# ---------------------------------------------------------------------------------------------------------------
def identity_check(name, X, y, xt, xc, P, gi):
    """With every bound at +-inf and every row in bounds, the target's pipeline gives the NEI fixtures' values bit for
    bit (runs s4, s16 against neibig_<name> on its candidates; p1, p7, p15 against neibatch_<name>).  Returns the
    number of arrays compared."""
    count = 0
    have_big = os.path.exists(NB.fixture_path(name))
    have_batch = name in NBB.CASES and os.path.exists(NBB.fixture_path(name))
    runs = {r: RUNS[r] for r in RUNS if (r in ("s4", "s16") and have_big) or (r.startswith("p") and have_batch)}
    if not runs:
        return 0
    tr = Truth(name, X, y, np.zeros((0, len(X))), xc, P, gi, cons=False, runs=runs)
    big = NB.load(name) if have_big else None
    batch = NBB.load(name) if have_batch else None
    for run, r in tr.res.items():
        for kind, nk in (("cnei", "nei"), ("logcnei", "lognei")):
            got = np.array([float(v) for v in r[kind]])
            if run.startswith("s"):
                want = big[f"{run}_{nk}"]
                got = got[:len(want)]
            else:
                want = batch[f"{run}_{nk}"]
            assert np.array_equal(got.view(np.int64), want.view(np.int64)), (name, run, kind)
            count += 1
        wb = big[f"{run}_best"] if run.startswith("s") else batch[f"{run}_best"]
        assert np.array_equal(np.array([float(v) for v in r["best"]]), wb), (name, run, "best")
    return count


def coverage_check(name, res, n):
    """The floor occurs in s4f (and in no other p = 0 run), on SMALL_CASE some pending run has a sample whose incumbent
    is a pending row, the out-of-bounds rows are never eligible, and between 5 and 90 % of the registered rows are
    eligible.  Returns the number of (pending run, sample) pairs whose incumbent is a pending row."""
    assert res["s4f_floor"].any() and not res["s4f_floor"].all(), (name, res["s4f_floor"])
    assert not res["s4_floor"].any() and not res["s16_floor"].any(), name
    pend = sum(int(np.sum(res[f"p{p}_best_row"] >= n)) for p in PS)
    assert pend > 0 or name != SMALL_CASE, name
    for run in RUNS:
        ok = res[f"{run}_ok"]
        assert not ok[~res["inb"][:len(ok)]].any(), (name, run)
        frac = ok[:n].mean()
        assert 0.05 <= frac <= 0.9 or run == "s4f", (name, run, frac)
    return pend


def margins(tr):
    """The smallest distance of a constraint fantasy to a finite bound, relative to that constraint's y_std."""
    worst = np.inf
    for j, g in enumerate(tr.gps[1:]):
        v = np.concatenate([np.array([float(x) for row in g.Fd[r] for x in row]) for r in RUNS])
        for b in (tr.bounds[0][j], tr.bounds[1][j], tr.bounds[3][j]):
            if np.isfinite(b):
                worst = min(worst, float(np.min(np.abs(v - b))) / float(g.ys))
    return worst


def make_case(name):
    X, y, Yc, xt, group, P, xc = inputs(name)
    gi = NB.grad_rows(group)
    n = len(X)
    ident = identity_check(name, X, y, xt, xc, P, gi)
    tr = Truth(name, X, y, Yc, xc, P, gi)
    res = tr.rounded(y, gi)
    marg = margins(tr)
    assert marg >= MARGIN, (name, marg)
    res["pending_incumbents"] = coverage_check(name, res, n)
    res.update(referee(name, X, y, Yc, xc, P, tr))
    res.update(X_sha256=np.array(NB._digest(X)), y_sha256=np.array(NB._digest(y)),
               Yc_sha256=np.array(NB._digest(Yc)), xt_sha256=np.array(NB._digest(xt)),
               P_sha256=np.array(NB._digest(P)), margin=marg, identity_arrays=ident)
    return res


def fixture_path(name):
    return os.path.join(MI.GOLDEN, f"cneibig_{name}.npz")


def load(name, path=None):
    """The fixture of a case with its inputs (X, y, Yc, xt, group, P, xc), checked against the digests it keeps."""
    with np.load(path or fixture_path(name)) as z:
        r = {k: z[k] for k in z.files}
    X, y, Yc, xt, group, P, xc = inputs(name)
    for k, v in (("X", X), ("y", y), ("Yc", Yc), ("xt", xt), ("P", P)):
        if NB._digest(v) != str(r[f"{k}_sha256"]):
            raise ValueError(f"{name}: the inputs {k} differ from those the fixture was computed on")
    r.update(X=X, y=y, Yc=Yc, xt=xt, group=group, P=P, xc=xc)
    return r


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--only", nargs="*", default=None, help="case names (default: all)")
    ap.add_argument("--out", default=MI.GOLDEN)
    a = ap.parse_args(argv)
    for name in a.only or list(CASES):
        t0 = time.perf_counter()
        res = make_case(name)
        np.savez_compressed(os.path.join(a.out, f"cneibig_{name}.npz"), **res)
        print(f"{name}: J={len(CASES[name])} margin={float(res['margin']):.1e} identity arrays="
              f"{int(res['identity_arrays'])} ({time.perf_counter() - t0:.0f} s)", flush=True)


if __name__ == "__main__":
    main()

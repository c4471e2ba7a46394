"""Double-double reference of LogEI, LogPoI, MES and the constrained acquisitions (include/b200bo.h B200BO_ACQ_*,
DESIGN.md 4.10 - 4.12), values and input gradients, at production sizes on ill-conditioned training sets.

Problems: the four of oracle/make_illcond_big.py (N = 1000 .. 4096, cond(K) 6e6 .. 2e11) and b_m25_c5, the C5 shape
of bench.py (Matern 2.5, d = 32, N = 8192, a 30 % cluster at spread 1e-3, alpha 1e-6).  Each has make_illcond.problem()'s
candidate groups followed by uniform rows up to make_illcond_big.CANDIDATES = 4296 (34 tiles of 128).  On b_m15_d17
(np = 1024, d = 17) and b_m25_c3 (np = 4096) two constraint GPs join the target (constraint_cases()): an RBF GP at
alpha = 1e-8 (cond(K) about 1e11) under a two-sided bound that puts most candidates in its lower tail (the reflected
log1mexp pair of DESIGN.md 4.12), and a Matern 1.5 ARD + WhiteKernel GP under a one-sided bound (-inf, ub) that
straddles its data.

Every GP is fitted in double-double arithmetic (oracle/dd.py, about 106 bits): mu and sigma^2 at every candidate,
unrounded (mpmath values); on the 64 rows of make_nei_big.grad_rows() (training rows, their 1e-7 neighbours, the
incumbent's neighbourhood, uniform rows) d mu and d sigma^2 through dd.posterior_grad.  The acquisitions and their
input gradients follow from those at 50 digits, through the 50-digit definitions of tests/logei_oracle.py (log h, its
ratios, log Phi, the constraint factor) and tests/mes_oracle.py (the MES term), with y_max = max y + t s_y for
t in T_LEVELS, xi = make_illcond.XI, kappa = KAPPA and the y* sets of MES_SETS.  Keys of the fixture (the truth, not
negated; "g_<key>" its gradient on the grad rows, (64, d)):

  logei_t<t>, logpoi_t<t>, mes_k4, mes_k16                    every problem
  ucb, ei, poi                                                 b_m25_c5 (y_max = max y)
  ei_pof, poi_pof, mes_pof (K = 4), logei_c_t<t>, logpoi_c_t<t> (t = 0, 4)   the constrained problems:
                                                               product with prod_j p_j, or plus sum_j log p_j

and sd (the truth's sigma, rounded), y_max, ystar_k4 / ystar_k16, grad_rows, cond; on the constrained problems also
c<j>_sd (each constraint GP's sigma) and, on the grad rows, gp<j>_mu_g / _sd_g / _dmu_g / _dsd_g (mu, sigma and their
gradients of the target, j = 0, and of each constraint GP).  The referee is sklearn's fp64 mu
and sigma (already in illbig_*.npz for the four problems; stored here as sk_mu / sk_sd for b_m25_c5 and as
sk_c<j>_mu / sk_c<j>_sd for the constraint GPs); the tests evaluate its kinds through tests/logei_oracle.py and
tests/mes_oracle.py and its gradients through tests/grad_oracle.py.

The inputs are not stored again: load() rebuilds X, y and the candidates of the four problems from their illbig_*
fixtures (make_illcond_big.load()) and those of b_m25_c5 from its seeds (X and the uniform rows; y and the group rows
go through libm and are stored), and checks them against the SHA-256 digests kept here.  The constraint values go
through libm and are stored (c<j>_y).  No rows of L and no believer sequence: this is about predict, the acquisitions,
selection and gradients.

Regenerate with

    python -m oracle.make_acq_big                    # every problem
    python -m oracle.make_acq_big --only b_m15_d17   # some of them

About 15 minutes on 8 CPU cores for the whole table (measured 99 s for b_m15_d17 and 783 s for the other four, part of
that time sharing the cores with other work); b_m25_c5 takes 427 s of it (the N = 8192 factor and its 4296 forward
solves, about 2 GB of host memory).  Nothing here needs a GPU.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import sys
import time
import warnings

import mpmath as mp
import numpy as np

from oracle import dd
from oracle import make_illcond as MI
from oracle import make_illcond_big as MB
from oracle import make_nei_big as NB

sys.path.insert(0, os.path.join(MI.ROOT, "tests"))
import logei_oracle as LO  # noqa: E402
import mes_oracle as MO  # noqa: E402

XI, KAPPA = MI.XI, MI.KAPPA
T_LEVELS = (0, 1, 4)  # y_max = max y + t s_y
T_CONS = (0, 4)  # the levels of the constrained log forms
MES_SETS = {"k4": (1e-3, 0.5, 2.0, 8.0), "k16": tuple(np.geomspace(1e-3, 8.0, 16))}  # y* = max y + v s_y
C5 = dict(kern="m25", d=32, n=8192, ls=1.0, cluster=(0.3, 1e-3), alpha=1e-6, seed=25)
PROBLEMS = ("b_m05_ard", "b_m15_d17", "b_m25_c3", "b_m25_c5", "b_rbf_long")
CONSTRAINED = ("b_m15_d17", "b_m25_c3")
SMALL = "b_m15_d17"


def case(name):
    return C5 if name == "b_m25_c5" else MB.CASES[name]


def constraint_cases(d):
    """The two constraint GPs (make_illcond case dicts): RBF, ConstantKernel 2, l = 2, alpha 1e-8; Matern 1.5 ARD with
    length scales 1/2, 1, 2 in turn and WhiteKernel 1e-4."""
    return (dict(kern="rbf", d=d, ls=2.0, const=2.0, alpha=1e-8),
            dict(kern="m15", d=d, ls=[(0.5, 1.0, 2.0)[j % 3] for j in range(d)], white=1e-4, alpha=1e-6))


def constraint_values(X):
    """Smooth functions of the inputs, one per constraint GP."""
    c1 = np.cos(3.0 * X[:, 0]) + 0.5 * np.sin(2.0 * X[:, 1] + X[:, 2])
    c2 = X[:, 0] - X[:, 1] + 0.3 * np.sin(5.0 * X[:, 2])
    return c1, c2


def constraint_bounds(cy):
    """(lb, ub) per constraint: the first two-sided above its 90th percentile (most candidates in the lower tail,
    the reflected pair), the second (-inf, median)."""
    c1, c2 = cy
    lb = float(np.quantile(c1, 0.9))
    return ((lb, lb + 0.25 * float(np.std(c1))), (-np.inf, float(np.median(c2))))


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype="<f8").tobytes()).hexdigest()


def c5_inputs():
    """X, y, candidates and groups of b_m25_c5: make_illcond.problem()'s, then uniform rows up to 4296."""
    _, y, head, group = MI.problem(C5)
    X, extra = MB.uniform_inputs(C5)
    group = np.concatenate([group, np.full(len(extra), MI.G_UNIFORM, dtype=np.int8)])
    return X, y, np.vstack([head, extra]), group


def inputs(name):
    """X, y, the candidates and their groups."""
    if name == "b_m25_c5":
        return c5_inputs()
    r = MB.load(name)
    return r["X"], r["y"], r["xt"], r["group"]


# ---------------------------------------------------------------------------------------------------------------
# the double-double posterior and the 50-digit acquisitions
# ---------------------------------------------------------------------------------------------------------------
class Posterior:
    """The double-double fit of one GP: mu, var (mpmath lists, data units) at every candidate; dmu, dvar (mpmath
    (len(gi), d)) on the rows gi."""

    def __init__(self, c, X, y, xt, gi):
        mp.mp.dps = 50
        fit = self.fit = dd.Fit(c, X, y)
        xs = dd.scaled(c, xt)
        Ks = fit.cross(xs)
        self.mu = fit.mean(Ks)
        self.var = fit.variance(Ks, [fit.n])[0]
        Kg = (np.ascontiguousarray(Ks[0][gi]), np.ascontiguousarray(Ks[1][gi]))
        del Ks
        _, G = dd.posterior_grad(fit, xs[gi], Kg, (fit.alpha_[0][None, :], fit.alpha_[1][None, :]))
        ys, d = fit.y_std, G[0].shape[2]
        self.dmu = [[ys * dd.to_mp(G[0][k, 0, j], G[1][k, 0, j]) for j in range(d)] for k in range(len(gi))]
        self.dvar = [[-2 * ys * ys * dd.to_mp(G[0][k, 1, j], G[1][k, 1, j]) for j in range(d)] for k in range(len(gi))]

    def condition(self):
        ev = np.linalg.eigvalsh(self.fit.K[0] + self.fit.K[1])
        return float(ev[-1] / ev[0])


def base_term(kind, m, sd, p):
    """(value, cm, cs) of a base acquisition at 50 digits: d value = cm d mu + cs d sd.  p: y_max (EI, PoI and their
    logs), the y* list (MES)."""
    mp.mp.dps = 50
    if kind == "ucb":
        return m + mp.mpf(KAPPA) * sd, mp.mpf(1), mp.mpf(KAPPA)
    if kind == "mes":
        K = len(p)
        v = cm = cs = mp.mpf(0)
        for ys in p:
            g = (mp.mpf(ys) - m) / sd
            t, dt = MO.mp_mes_term(g)
            v, cm, cs = v + t, cm - dt, cs - dt * g
        return v / K, cm / (K * sd), cs / (K * sd)
    a = m - mp.mpf(p) - mp.mpf(XI)
    z = a / sd
    if kind == "ei":
        P, q = mp.ncdf(z), mp.npdf(z)
        return a * P + sd * q, P, q
    if kind == "poi":
        q = mp.npdf(z)
        return mp.ncdf(z), q / sd, -z * q / sd
    if kind == "logei":
        v = LO.mp_log_h(z, exact=True) + mp.log(sd)
        r, q = LO.mp_log_h_ratios(z, exact=True)
        mp.mp.dps = 50
        return v, r / sd, q / sd
    if kind == "logpoi":
        v = LO.mp_log_ndtr(z, exact=True)
        mp.mp.dps = 50
        lam = mp.npdf(z) / mp.ncdf(z)
        return v, lam / sd, -z * lam / sd
    raise ValueError(kind)


def cons_term(lb, ub, m, sd):
    """(log p, cm, cs) of one constraint factor p = Phi((ub - mu)/sd) - Phi((lb - mu)/sd): d log p = cm d mu + cs d sd."""
    l = -np.inf if lb == -np.inf else (mp.mpf(lb) - m) / sd
    u = np.inf if ub == np.inf else (mp.mpf(ub) - m) / sd
    lp, fl, fu = LO.mp_cfactor(l, u, exact=True)
    mp.mp.dps = 50
    cs = -((0 if lb == -np.inf else fl * l) + (0 if ub == np.inf else fu * u)) / sd
    return lp, -(fl + fu) / sd, cs


def kinds(name):
    """{key: (base kind, parameter, form, level)}: form None (unconstrained), "prod" or "log"."""
    out = {}
    for t in T_LEVELS:
        out[f"logei_t{t}"] = ("logei", t, None)
        out[f"logpoi_t{t}"] = ("logpoi", t, None)
    for k in MES_SETS:
        out[f"mes_{k}"] = ("mes", k, None)
    if name == "b_m25_c5":
        for k in ("ucb", "ei", "poi"):
            out[k] = (k, 0, None)
    if name in CONSTRAINED:
        out.update(ei_pof=("ei", 0, "prod"), poi_pof=("poi", 0, "prod"), mes_pof=("mes", "k4", "prod"))
        for t in T_CONS:
            out[f"logei_c_t{t}"] = ("logei", t, "log")
            out[f"logpoi_c_t{t}"] = ("logpoi", t, "log")
    return out


def params(y):
    """y_max per level and the y* sets, in fp64 as the device receives them."""
    ym, sy = float(np.max(y)), float(np.std(y))
    y_max = {t: ym + t * sy for t in T_LEVELS}
    ystar = {k: ym + np.asarray(v) * sy for k, v in MES_SETS.items()}
    return y_max, ystar


def evaluate(spec, post, cons, bounds, y_max, ystar, t, k=None):
    """The value of one kind at candidate t (mpmath), and with k (the row's index among the grad rows) its gradient
    (mpmath list)."""
    kind, p, form = spec
    par = ystar[p] if kind == "mes" else y_max[p]
    grad = k is not None
    m, sd = post.mu[t], mp.sqrt(post.var[t])
    v, cm, cs = base_term(kind, m, sd, par)
    if grad:
        dsd = [dv / (2 * sd) for dv in post.dvar[k]]
        g = [cm * a + cs * b for a, b in zip(post.dmu[k], dsd)]
    if form is not None:
        lsum, gsum = mp.mpf(0), [mp.mpf(0)] * len(post.dmu[0]) if grad else None
        for cp, (lb, ub) in zip(cons, bounds):
            mc, sc = cp.mu[t], mp.sqrt(cp.var[t])
            lp, ccm, ccs = cons_term(lb, ub, mc, sc)
            lsum += lp
            if grad:
                gsum = [s + ccm * a + ccs * b / (2 * sc) for s, a, b in zip(gsum, cp.dmu[k], cp.dvar[k])]
        if form == "log":
            v = v + lsum
            if grad:
                g = [a + b for a, b in zip(g, gsum)]
        else:
            P = mp.exp(lsum)
            if grad:
                g = [P * (a + v * b) for a, b in zip(g, gsum)]
            v = v * P
    return (v, g) if grad else v


def truth(name, X, y, xt, gi):
    """Every truth array of a problem (the fixture's keys but the referee's and the inputs')."""
    c = case(name)
    post = Posterior(c, X, y, xt, gi)
    out = dict(sd=np.array([float(mp.sqrt(v)) for v in post.var]), grad_rows=gi, cond=post.condition())
    cons, bounds = (), ()
    if name in CONSTRAINED:
        cy = constraint_values(X)
        bounds = constraint_bounds(cy)
        cons = tuple(Posterior(cc, X, v, xt, gi) for cc, v in zip(constraint_cases(X.shape[1]), cy))
        for j, (v, (lb, ub), cp) in enumerate(zip(cy, bounds, cons)):
            out[f"c{j}_y"] = v
            out[f"c{j}_bounds"] = np.array([lb, ub])
            out[f"c{j}_cond"] = cp.condition()
            out[f"c{j}_sd"] = np.array([float(mp.sqrt(u)) for u in cp.var])
        # each GP's posterior on the grad rows (gp0 the target), so that an error of a constrained form can be
        # traced to the GP and the quantity that carries it
        for j, p in enumerate((post,) + cons):
            sd = [mp.sqrt(p.var[t]) for t in gi]
            out[f"gp{j}_mu_g"] = np.array([float(p.mu[t]) for t in gi])
            out[f"gp{j}_sd_g"] = np.array([float(v) for v in sd])
            out[f"gp{j}_dmu_g"] = np.array([[float(u) for u in row] for row in p.dmu])
            out[f"gp{j}_dsd_g"] = np.array([[float(u / (2 * v)) for u in row] for row, v in zip(p.dvar, sd)])
    y_max, ystar = params(y)
    out["y_max"] = np.array([y_max[t] for t in T_LEVELS])
    out.update({f"ystar_{k}": v for k, v in ystar.items()})
    for key, spec in kinds(name).items():
        out[key] = np.array([float(evaluate(spec, post, cons, bounds, y_max, ystar, t)) for t in range(len(xt))])
        out[f"g_{key}"] = np.array([[float(u) for u in evaluate(spec, post, cons, bounds, y_max, ystar, t, k)[1]]
                                    for k, t in enumerate(gi)])
    return out


# ---------------------------------------------------------------------------------------------------------------
# the fp64 referee: sklearn's mu and sigma
# ---------------------------------------------------------------------------------------------------------------
def sk_predict(c, X, y, xt):
    from sklearn.gaussian_process import GaussianProcessRegressor

    sk = GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True, optimizer=None).fit(X, y)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return sk.predict(xt, return_std=True)


def referee(name, X, y, xt):
    out = {}
    if name == "b_m25_c5":
        out["sk_mu"], out["sk_sd"] = sk_predict(C5, X, y, xt)
    if name in CONSTRAINED:
        for j, (cc, v) in enumerate(zip(constraint_cases(X.shape[1]), constraint_values(X))):
            out[f"sk_c{j}_mu"], out[f"sk_c{j}_sd"] = sk_predict(cc, X, v, xt)
    return out


# ---------------------------------------------------------------------------------------------------------------
# fixtures
# ---------------------------------------------------------------------------------------------------------------
def make_problem(name, inputs_=None):
    """Every array of the fixture of one problem (the inputs' digests, and for b_m25_c5 the rows that go through
    libm)."""
    X, y, xt, group = inputs_ if inputs_ is not None else inputs(name)
    gi = NB.grad_rows(group)
    res = truth(name, X, y, xt, gi)
    res.update(referee(name, X, y, xt))
    res.update(X_sha256=np.array(_digest(X)), y_sha256=np.array(_digest(y)), xt_sha256=np.array(_digest(xt)))
    if name == "b_m25_c5":
        res.update(y=y, xt_head=xt[:len(MI.problem(C5)[2])], group=group)
    return res


def fixture_path(name):
    return os.path.join(MI.GOLDEN, f"acqbig_{name}.npz")


def load(name, path=None):
    """The fixture of a problem with its inputs (X, y, xt, group), checked against the digests it keeps; for the
    four illbig problems also their referee's sk_mu / sk_sd."""
    with np.load(path or fixture_path(name)) as z:
        r = {k: z[k] for k in z.files}
    if name == "b_m25_c5":
        X, extra = MB.uniform_inputs(C5)
        y, xt, group = r["y"], np.vstack([r["xt_head"], extra]), r["group"]
    else:
        b = MB.load(name)
        X, y, xt, group = b["X"], b["y"], b["xt"], b["group"]
        r.update(sk_mu=b["sk_mu"], sk_sd=b["sk_sd"])
    for k, v in (("X", X), ("y", y), ("xt", xt)):
        if _digest(v) != str(r[f"{k}_sha256"]):
            raise ValueError(f"{name}: the inputs {k} differ from those the fixture was computed on")
    r.update(X=X, y=y, xt=xt, group=group)
    return r


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--only", nargs="*", default=None, help="problem names (default: all)")
    ap.add_argument("--out", default=MI.GOLDEN)
    a = ap.parse_args(argv)
    t00 = time.perf_counter()
    for name in a.only or PROBLEMS:
        t0 = time.perf_counter()
        res = make_problem(name)
        np.savez_compressed(os.path.join(a.out, f"acqbig_{name}.npz"), **res)
        print(f"{name}: cond(K)={float(res['cond']):.2e} ({time.perf_counter() - t0:.0f} s)", flush=True)
    print(f"total {time.perf_counter() - t00:.0f} s", flush=True)


if __name__ == "__main__":
    main()

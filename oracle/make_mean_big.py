"""Double-double reference of the posterior-mean merit B200BO_ACQ_MEAN (include/b200bo.h, DESIGN.md 4.17), its input
gradient and its selection at production sizes, on ill-conditioned target and constraint GPs.

Problems (PROBLEMS): the target GP and candidates of an existing fixture, and the constraint GPs named there:

  b_m15_d17    illbig's target (np = 1024, d = 17: predict_mean_kernel<DREG=false>), acqbig's two constraint GPs
               (RBF at alpha = 1e-8, cond(K) 1.7e11; Matern 1.5 ARD + WhiteKernel): three GPs in one launch
  b_m25_c3     illbig's target at the C3 shape (N = 4096, d = 16: eight 512-row k-chunks on the small path), the same
               two constraint GPs
  b_rbf_long   illbig's target (RBF at alpha = 1e-8, cond(K) 1.8e11: A1 = sum |alpha_| about 1e10, so T about 3.6e9),
               cneibig's noisy Matern 2.5 constraint GP
  b_m25_c5     acqbig's C5 inputs (N = 8192, d = 32, sixteen k-chunks), no constraint
  o_offset_d2  prunemx's target and candidates (y at a 1e6 offset, N = 901, np = 1024) and one new constraint GP on the
               same X whose values sit at a 1e6 offset too, so that lb - mu and mu - ub cancel two numbers near 1e6

The inputs are not stored: they are rebuilt from the generators of those fixtures (load() checks them against the
SHA-256 digests kept here).  Constraint values: acqbig's go through libm and are stored there; cneibig's and
o_offset_d2's are IEEE polynomials of X.

Every GP is fitted in double-double arithmetic (oracle/dd.py): mu_j at every candidate (data units, (hi, lo) pairs:
hi is the value rounded to fp64), A1 = sum |alpha_| of the target and T = 2 (|y_mean| + y_std c A1) + 1 at 50 digits,
and on the 64 gradient rows (make_nei_big.grad_rows(); o_offset_d2: its first 64 base rows) d mu_j through
dd.posterior_grad, the computation of make_acq_big.Posterior (so on the shared problems the same bits as acqbig's
gp<j>_dmu_g).  On b_m15_d17 and o_offset_d2 also mu_j at the training rows (recommend(in_sample=True)).

Bound runs (RUNS), on the problems with constraint GPs:

  two   every constraint two-sided, 20 - 60 % of the candidates feasible
  one   (-inf, ub) on the even constraints, (lb, +inf) on the odd ones
  none  constraint 0 confined to a gap of its means: no candidate is feasible and the ranking is by viol alone
  inf   every bound +-inf: the unconstrained merit

Each finite bound sits at the midpoint (in "none": at a third and two thirds) of a gap of at least GAP y_std_j between
consecutive truth means of that GP over the candidates (and the training rows where those are stored), so every mean
is at least GAP / 3 y_std_j from every bound and the device's feasibility must equal the truth's exactly.  Per run the
merit (mu_0 where viol = 0, else -T (1 + viol)) at 50 digits, rounded; the feasibility mask; the truth's top 64 (by
descending merit, stable) and the 63 gaps between consecutive entries; d merit on the gradient rows.  The referee is
sklearn's fp64 mu_j (sk_mu<j>, sk_muX<j>).

Regenerate with

    python oracle/make_mean_big.py                      # every problem (or python -m oracle.make_mean_big)
    python oracle/make_mean_big.py --only o_offset_d2   # some of them

The output is byte-identical from run to run.  Measured on 8 CPU cores, one process over the whole table: 6 min 6 s
wall (361 s: b_m25_c5 202 s, most of it the N = 8192 double-double factor; b_m25_c3 113 s; b_m15_d17 30 s; b_rbf_long
15 s; o_offset_d2 2 s).  Nothing here needs a GPU.
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

if __package__ in (None, ""):  # run as a script: python oracle/make_mean_big.py
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import dd  # noqa: E402
from oracle import make_acq_big as AB  # noqa: E402
from oracle import make_cnei_big as CB  # noqa: E402
from oracle import make_illcond as MI  # noqa: E402
from oracle import make_illcond_big as MB  # noqa: E402
from oracle import make_nei_big as NB  # noqa: E402
from oracle import make_prune_matrix as PM  # noqa: E402

PROBLEMS = ("b_m15_d17", "b_m25_c3", "b_rbf_long", "b_m25_c5", "o_offset_d2")
IN_SAMPLE = ("b_m15_d17", "o_offset_d2")  # mu at the training rows too (recommend)
SMALL = "o_offset_d2"
RUNS = ("two", "one", "none", "inf")
GAP = 1e-5  # every finite bound in a gap of at least GAP y_std_j between consecutive truth means
FEASIBLE = 0.4  # the fraction of candidates run "two" aims to keep
TOPK = 64
OFFSET_CON = dict(kern="m25", d=2, ls=0.25, alpha=1e-6)


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype="<f8").tobytes()).hexdigest()


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def offset_constraint(X):
    """o_offset_d2's constraint values: 1e6 plus 1e-3 times a polynomial of X (exact IEEE operations)."""
    return 1e6 + 1e-3 * (X[:, 0] - 0.5 * X[:, 1] + 0.75 * X[:, 0] * X[:, 1])


def inputs(name):
    """X, the candidates xt, the gradient rows gi and per GP (case dict, y), the target first."""
    if name == "o_offset_d2":
        X, y, xt, src, _, _ = PM.inputs(name)
        return X, xt, np.flatnonzero(src >= 0)[:TOPK], [(PM.case(name), y), (OFFSET_CON, offset_constraint(X))]
    if name == "b_m25_c5":
        r = AB.load(name)
        return r["X"], r["xt"], NB.grad_rows(r["group"]), [(AB.C5, r["y"])]
    r = MB.load(name)
    X, xt, gi = r["X"], r["xt"], NB.grad_rows(r["group"])
    gps = [(MB.CASES[name], r["y"])]
    if name == "b_rbf_long":
        gps.append((CB.gp_specs(name, X.shape[1])[1][0], CB.constraint_y(name, X)[0]))
    else:
        gps += list(zip(AB.constraint_cases(X.shape[1]), AB.constraint_values(X)))
    return X, xt, gi, gps


# ---------------------------------------------------------------------------------------------------------------
# the double-double posterior mean
# ---------------------------------------------------------------------------------------------------------------
class Mean:
    """One GP's double-double mean: mu (mpmath list at the candidates), muX (at the training rows, or None), dmu
    (mpmath (64, d) on the gradient rows), A1 = sum |alpha_| and T (mpmath)."""

    def __init__(self, c, X, y, xt, gi, at_x):
        mp.mp.dps = 50
        fit = dd.Fit(c, X, y)
        xs = dd.scaled(c, xt)
        Ks = fit.cross(xs)
        self.mu = fit.mean(Ks)
        Kg = (np.ascontiguousarray(Ks[0][gi]), np.ascontiguousarray(Ks[1][gi]))
        del Ks
        _, G = dd.posterior_grad(fit, xs[gi], Kg, (fit.alpha_[0][None, :], fit.alpha_[1][None, :]))
        ys, d = fit.y_std, G[0].shape[2]
        self.dmu = [[ys * dd.to_mp(G[0][k, 0, j], G[1][k, 0, j]) for j in range(d)] for k in range(len(gi))]
        self.muX = fit.mean(fit.cross(fit.Xs)) if at_x else None
        self.A1 = mp.fsum(abs(dd.to_mp(h, l)) for h, l in zip(*fit.alpha_))
        self.y_mean, self.y_std = fit.y_mean, fit.y_std
        self.T = 2 * (abs(fit.y_mean) + fit.y_std * mp.mpf(fit.c) * self.A1) + 1


# ---------------------------------------------------------------------------------------------------------------
# bounds
# ---------------------------------------------------------------------------------------------------------------
def _gap_at(v, b, width):
    """(lo, hi) of the gap of the sorted values v nearest to b that is at least `width` wide."""
    k = int(np.searchsorted(v, b))
    for step in range(len(v)):
        for q in (k + step, k - step):
            if 0 < q < len(v) and v[q] - v[q - 1] >= width:
                return float(v[q - 1]), float(v[q])
    raise AssertionError("no gap wide enough for a bound")


def _mid(v, b, width):
    lo, hi = _gap_at(v, b, width)
    return 0.5 * (lo + hi)


def choose_bounds(gps):
    """{run: (lb, ub)} over the constraint GPs gps[1:] (module docstring)."""
    J = len(gps) - 1
    vals = []
    for g in gps[1:]:
        v = [float(u) for u in g.mu] + ([float(u) for u in g.muX] if g.muX is not None else [])
        vals.append(np.unique(np.array(v)))
    width = [GAP * float(g.y_std) for g in gps[1:]]
    q = FEASIBLE ** (1.0 / J)
    cand = [np.array([float(u) for u in g.mu]) for g in gps[1:]]
    out = {"inf": (np.full(J, -np.inf), np.full(J, np.inf))}
    out["two"] = (np.array([_mid(vals[j], np.quantile(cand[j], (1 - q) / 2), width[j]) for j in range(J)]),
                  np.array([_mid(vals[j], np.quantile(cand[j], 1 - (1 - q) / 2), width[j]) for j in range(J)]))
    lb, ub = np.full(J, -np.inf), np.full(J, np.inf)
    for j in range(J):
        if j % 2 == 0:
            ub[j] = _mid(vals[j], np.quantile(cand[j], 0.6), width[j])
        else:
            lb[j] = _mid(vals[j], np.quantile(cand[j], 0.4), width[j])
    out["one"] = (lb, ub)
    lo, hi = _gap_at(vals[0], np.quantile(cand[0], 0.5), 3 * width[0])
    lb, ub = np.full(J, -np.inf), np.full(J, np.inf)
    lb[0], ub[0] = lo + (hi - lo) / 3, lo + 2 * (hi - lo) / 3
    out["none"] = (lb, ub)
    return {r: out[r] for r in RUNS}


# ---------------------------------------------------------------------------------------------------------------
# the merit at 50 digits
# ---------------------------------------------------------------------------------------------------------------
def merit(mus, T, lb, ub):
    """(merit (mpmath list), viol (mpmath list), signs [row][j]) from the means mus[g] (the target first)."""
    mp.mp.dps = 50
    out, viol, signs = [], [], []
    for t in range(len(mus[0])):
        v, s = mp.mpf(0), []
        for j, (lo, hi) in enumerate(zip(lb, ub)):
            m = mus[j + 1][t]
            if lo != -np.inf and m < lo:
                v += mp.mpf(lo) - m
                s.append(-1)
            elif hi != np.inf and m > hi:
                v += m - mp.mpf(hi)
                s.append(1)
            else:
                s.append(0)
        viol.append(v)
        signs.append(s)
        out.append(mus[0][t] if v == 0 else -T * (1 + v))
    return out, viol, signs


def merit_grad(gps, T, signs, feas):
    """d merit on the gradient rows (mpmath [k][j]): d mu_0 where feasible, else -T sum_j s_j d mu_j."""
    d = len(gps[0].dmu[0])
    out = []
    for k in range(len(gps[0].dmu)):
        if feas[k]:
            out.append(list(gps[0].dmu[k]))
        else:
            out.append([-T * mp.fsum(signs[k][j] * gps[j + 1].dmu[k][q] for j in range(len(gps) - 1))
                        for q in range(d)])
    return out


def truth(name, X, xt, gi, spec):
    gps = [Mean(c, X, y, xt, gi, name in IN_SAMPLE) for c, y in spec]
    out = dict(grad_rows=gi, A1=float(gps[0].A1), T=float(gps[0].T))
    for g, m in enumerate(gps):
        for key, v in (("mu", m.mu), ("muX", m.muX)):
            if v is None:
                continue
            pr = [dd.from_mp(u) for u in v]
            out[f"{key}{g}_hi"] = np.array([a for a, _ in pr])
            out[f"{key}{g}_lo"] = np.array([b for _, b in pr])
        out[f"dmu{g}"] = np.array([[float(u) for u in row] for row in m.dmu])
        out[f"y_mean{g}"], out[f"y_std{g}"] = float(m.y_mean), float(m.y_std)
    if len(gps) == 1:
        return out
    T = gps[0].T
    for run, (lb, ub) in choose_bounds(gps).items():
        val, viol, signs = merit([g.mu for g in gps], T, lb, ub)
        feas = np.array([v == 0 for v in viol])
        assert {"two": 0.2 <= feas.mean() <= 0.6, "none": not feas.any(), "inf": feas.all()}.get(run, True), (run, feas.mean())
        rounded = np.array([float(v) for v in val])
        order = sorted(range(len(val)), key=lambda t: -val[t])[:TOPK]  # stable: ties to the lower index
        out[f"{run}_lb"], out[f"{run}_ub"] = lb, ub
        out[f"{run}_merit"] = rounded
        out[f"{run}_feas"] = feas
        out[f"{run}_top"] = np.array(order, dtype=np.int64)
        out[f"{run}_gap"] = np.array([float(val[a] - val[b]) for a, b in zip(order, order[1:])])
        out[f"{run}_dmerit"] = np.array([[float(u) for u in row]
                                         for row in merit_grad(gps, T, [signs[t] for t in gi], feas[gi])])
        margin = np.inf
        for j, g in enumerate(gps[1:]):
            v = np.array([float(u) for u in g.mu] + ([float(u) for u in g.muX] if g.muX is not None else []))
            for b in (lb[j], ub[j]):
                if np.isfinite(b):
                    margin = min(margin, float(np.min(np.abs(v - b))) / float(g.y_std))
        out[f"{run}_margin"] = margin
        if name in IN_SAMPLE:
            vx, violx, _ = merit([g.muX for g in gps], T, lb, ub)
            out[f"{run}_meritX"] = np.array([float(v) for v in vx])
            out[f"{run}_feasX"] = np.array([v == 0 for v in violx])
    return out


# ---------------------------------------------------------------------------------------------------------------
# the fp64 referee: sklearn's mu
# ---------------------------------------------------------------------------------------------------------------
def referee(name, X, xt, spec):
    from sklearn.gaussian_process import GaussianProcessRegressor

    out = {}
    for g, (c, y) in enumerate(spec):
        sk = GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True,
                                      optimizer=None).fit(X, y)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out[f"sk_mu{g}"] = sk.predict(xt)
            if name in IN_SAMPLE:
                out[f"sk_muX{g}"] = sk.predict(X)
    return out


# ---------------------------------------------------------------------------------------------------------------
# fixtures
# ---------------------------------------------------------------------------------------------------------------
def make_problem(name, with_referee=True):
    X, xt, gi, spec = inputs(name)
    res = truth(name, X, xt, gi, spec)
    if with_referee:
        res.update(referee(name, X, xt, spec))
    res.update(X_sha256=np.array(_digest(X)), xt_sha256=np.array(_digest(xt)),
               **{f"y{g}_sha256": np.array(_digest(y)) for g, (_, y) in enumerate(spec)})
    return res


def fixture_path(name):
    return os.path.join(MI.GOLDEN, f"meanbig_{name}.npz")


def load(name, path=None):
    """The fixture of a problem with its inputs (X, xt, gi, spec: per GP (case, y)), checked against the digests."""
    with np.load(path or fixture_path(name)) as z:
        r = {k: z[k] for k in z.files}
    X, xt, gi, spec = inputs(name)
    checks = [("X", X), ("xt", xt)] + [(f"y{g}", y) for g, (_, y) in enumerate(spec)]
    for k, v in checks:
        if _digest(v) != str(r[f"{k}_sha256"]):
            raise ValueError(f"{name}: the inputs {k} differ from those the fixture was computed on")
    if not np.array_equal(gi, r["grad_rows"]):
        raise ValueError(f"{name}: the gradient rows differ from the fixture's")
    r.update(X=X, xt=xt, spec=spec)
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
        np.savez_compressed(os.path.join(a.out, f"meanbig_{name}.npz"), **res)
        feas = {r: float(np.mean(res[f"{r}_feas"])) for r in RUNS if f"{r}_feas" in res}
        print(f"{name}: A1={float(res['A1']):.3e} T={float(res['T']):.3e} feasible {feas} "
              f"({time.perf_counter() - t0:.0f} s)", flush=True)
    print(f"total {time.perf_counter() - t00:.0f} s", flush=True)


if __name__ == "__main__":
    main()

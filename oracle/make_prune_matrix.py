"""Double-double reference of every prunable acquisition (UCB, EI, PoI, LogEI, LogPoI; DESIGN.md 4.9, 4.12) over a
grid of acquisition parameters, on candidate sets built to stress selection-only pruning.

Problems:
  * three of oracle/make_illcond_big.py's (b_m15_d17: np = 1024, d = 17; b_rbf_long: cond(K) 1e11, N = 2000;
    b_m25_c3: the C3 shape), their inputs rebuilt and checked against the illbig_* digests (make_illcond_big.load());
    the base candidates are the fixture's first SHARED rows, whose mu and sigma^2 must equal the stored truths bit for
    bit (tests/test_prune_matrix_cpu.py);
  * three of this module's (OWN): o_offset_d2, a target offset of 1e6 with y_std 5e-4 at d = 2 and N = 901
    (ragged against 64 and 128; np = 1024, the smallest launch with refine stages: b = 1, one level to 2);
    o_clo_d5, ConstantKernel 2^-13 (1.2e-4) x Matern 1.5 + WhiteKernel 1e-6 at d = 5; o_chi_d32, ConstantKernel 2^13
    (8192) x Matern 2.5 + WhiteKernel 1e-2 at d = 32.  Their base candidates are make_illcond.problem()'s groups
    (cluster, training copies, 1e-7 / 1e-9 neighbours, the incumbent's neighbourhood) and uniform rows up to SHARED.

The candidates (xt, stored) are the base rows with EXTRA rows spread between them: exact copies of training rows, rows
1e-9 from them, rows 1e3 away (every k* underflows to 0, sigma^2 = prior) and exact copies of earlier candidates, one
extra after every sixth base row; "src" gives each row's base index (-1 for an extra) and "dup_of" the candidate an
extra duplicates (-1 otherwise).  Eight copies of xt make 35 tiles of 128, enough for the refine stages (at least 32).
"bad_rows" holds rows with a NaN or +-inf coordinate, which every selection call refuses.

Truth: mu and sigma^2 in double-double (oracle/dd.py), stored as (hi, lo) pairs in data units; from them every kind at
50 digits:

  ucb      (len(KAPPAS), M)   kappa in KAPPAS
  ei, poi, logei, logpoi   (9, M)   row 3 i + j: y_max rule i (below every mu: min y - 40 s_y max(1, prior^1/2),
                                    where PoI is 1.0 at every candidate; max y; max y + 4 s_y), xi rule j (0, 0.01,
                                    10 s_y); s_y = std(y)

(the acquisition itself, not negated), with "kappa", "y_max" and "xi" the parameters in fp64 as the device receives
them, "top_<kind>" the 64 candidates of smallest closure value -acq (stable order: ties to the lowest index) and
"gap_<kind>" the 63 differences between consecutive truth values of that order.  X is rebuilt from seeds and checked
against "X_sha256"; y is stored where it goes through libm (OWN problems).

Regenerate with

    python -m oracle.make_prune_matrix                   # every problem
    python -m oracle.make_prune_matrix --only o_offset_d2

About 2 minutes on 8 CPU cores for the whole table (measured 115 s), half of it the N = 4096 factor of b_m25_c3.  Nothing here needs
a GPU.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import sys
import time

import mpmath as mp
import numpy as np

from oracle import dd
from oracle import make_illcond as MI
from oracle import make_illcond_big as MB

sys.path.insert(0, os.path.join(MI.ROOT, "tests"))
import logei_oracle as LO  # noqa: E402

SHARED = 512  # base candidates per problem
EXTRA_EVERY = 6
KAPPAS = (-1.0, 0.0, 2.576, 100.0)
KINDS = ("ucb", "ei", "poi", "logei", "logpoi")
TOPK = 64  # B200BO_MAX_TOPK
SHARED_PROBLEMS = ("b_m15_d17", "b_rbf_long", "b_m25_c3")
OWN = {
    "o_offset_d2": dict(kern="m25", d=2, n=901, ls=0.25, cluster=(0.3, 1e-3), alpha=1e-6, seed=41,
                        offset=1e6, scale=1e-3),
    "o_clo_d5": dict(kern="m15", d=5, n=1100, ls=0.5, const=2.0 ** -13, white=1e-6, cluster=(0.3, 1e-3),
                     alpha=1e-6, seed=42),
    "o_chi_d32": dict(kern="m25", d=32, n=1200, ls=2.0, const=2.0 ** 13, white=1e-2, cluster=None, alpha=1e-6,
                      seed=43),
}
PROBLEMS = SHARED_PROBLEMS + tuple(OWN)


def case(name):
    return OWN[name] if name in OWN else MB.CASES[name]


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype="<f8").tobytes()).hexdigest()


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def base_inputs(name):
    """X, y and the base candidates of a problem."""
    if name in SHARED_PROBLEMS:
        r = MB.load(name)
        return r["X"], r["y"], r["xt"][:SHARED]
    c = OWN[name]
    X, y, head, _ = MI.problem(c)
    if "offset" in c:
        y = c["offset"] + c["scale"] * y
    rs = np.random.RandomState(3000 + c["seed"])
    return X, y, np.vstack([head, rs.uniform(size=(SHARED - len(head), c["d"]))])


def candidates(name, X, base):
    """xt, src, dup_of and the non-finite rows: the base rows with the extras spread between them."""
    c = case(name)
    rs = np.random.RandomState(4000 + c["seed"])
    n, d = X.shape
    ne = len(base) // EXTRA_EVERY
    tr = rs.choice(n, 24, replace=False)
    copies = X[tr]
    near = X[tr] + 1e-9 * rs.choice([-1.0, 1.0], size=(24, d))
    far = 1e3 + rs.uniform(size=(12, d))
    kinds = np.concatenate([np.zeros(24, int), np.ones(24, int), np.full(12, 2), np.full(ne - 60, 3)])
    kinds = kinds[rs.permutation(ne)]
    rows, src, dup = [], [], []
    it = {0: iter(copies), 1: iter(near), 2: iter(far)}
    for i, b in enumerate(base):
        rows.append(b)
        src.append(i)
        dup.append(-1)
        if (i + 1) % EXTRA_EVERY == 0 and (i + 1) // EXTRA_EVERY <= ne:
            k = kinds[(i + 1) // EXTRA_EVERY - 1]
            if k == 3:  # an exact copy of an earlier candidate
                j = int(rs.randint(len(rows)))
                rows.append(rows[j].copy())
                dup.append(j if dup[j] < 0 else dup[j])
            else:
                rows.append(next(it[k]))
                dup.append(-1)
            src.append(-1)
    bad = base[:4].copy()
    bad[0, 0], bad[1, d - 1], bad[2, d // 2], bad[3, 0] = np.nan, np.inf, -np.inf, np.nan
    return np.array(rows), np.array(src, dtype=np.int64), np.array(dup, dtype=np.int64), bad


def inputs(name):
    X, y, base = base_inputs(name)
    xt, src, dup, bad = candidates(name, X, base)
    return X, y, xt, src, dup, bad


# ---------------------------------------------------------------------------------------------------------------
# the truth
# ---------------------------------------------------------------------------------------------------------------
def params(y, prior):
    """kappa, (y_max, xi) per row of the EI-type tables, in fp64."""
    ym, sy = float(np.max(y)), float(np.std(y))
    y_max = (float(np.min(y)) - 40.0 * sy * max(1.0, float(np.sqrt(prior))), ym, ym + 4.0 * sy)
    xis = (0.0, 0.01, 10.0 * sy)
    return np.array(KAPPAS), np.array([v for v in y_max for _ in xis]), np.array([x for _ in y_max for x in xis])


def value(kind, m, sd, p):
    """The acquisition at 50 digits; p = kappa (UCB) or (y_max, xi)."""
    mp.mp.dps = 50
    if kind == "ucb":
        return m + mp.mpf(p) * sd
    a = m - mp.mpf(p[0]) - mp.mpf(p[1])
    z = a / sd
    if kind == "ei":
        return a * mp.ncdf(z) + sd * mp.npdf(z)
    if kind == "poi":
        return mp.ncdf(z)
    if kind == "logei":
        v = LO.mp_log_h(z, exact=True) + mp.log(sd)
    else:
        v = LO.mp_log_ndtr(z, exact=True)
    mp.mp.dps = 50
    return v


def truth(name, X, y, xt):
    c = case(name)
    mp.mp.dps = 50
    fit = dd.Fit(c, X, y)
    Ks = fit.cross(dd.scaled(c, xt))
    mu = fit.mean(Ks)
    var = fit.variance(Ks, [fit.n])[0]
    del Ks
    out = {}
    for key, v in (("mu", mu), ("var", var)):
        pr = [dd.from_mp(u) for u in v]
        out[f"{key}_hi"] = np.array([a for a, _ in pr])
        out[f"{key}_lo"] = np.array([b for _, b in pr])
    sd = [mp.sqrt(v) for v in var]
    kappa, y_max, xi = params(y, float(fit.prior))
    out.update(kappa=kappa, y_max=y_max, xi=xi)
    for kind in KINDS:
        ps = list(kappa) if kind == "ucb" else list(zip(y_max, xi))
        t = np.array([[float(value(kind, m, s, p)) for m, s in zip(mu, sd)] for p in ps])
        out[kind] = t
        order = np.argsort(-t, axis=1, kind="stable")[:, :TOPK]
        out[f"top_{kind}"] = order
        out[f"gap_{kind}"] = np.diff(-np.take_along_axis(t, order, axis=1), axis=1)
    ev = np.linalg.eigvalsh(fit.K[0] + fit.K[1])
    out["cond"] = float(ev[-1] / ev[0])
    out["prior"] = float(fit.prior)
    return out


def make_problem(name):
    X, y, xt, src, dup, bad = inputs(name)
    res = truth(name, X, y, xt)
    res.update(xt=xt, src=src, dup_of=dup, bad_rows=bad, X_sha256=np.array(_digest(X)))
    if name in OWN:
        res["y"] = y
    return res


# ---------------------------------------------------------------------------------------------------------------
# fixtures
# ---------------------------------------------------------------------------------------------------------------
def fixture_path(name):
    return os.path.join(MI.GOLDEN, f"prunemx_{name}.npz")


def load(name, path=None):
    """The fixture of a problem with X and y, X checked against its digest (and, for the shared problems, against
    the illbig_* fixture's)."""
    with np.load(path or fixture_path(name)) as z:
        r = {k: z[k] for k in z.files}
    if name in OWN:
        X = MI.problem(OWN[name])[0]
    else:
        b = MB.load(name)
        X, r["y"] = b["X"], b["y"]
    if _digest(X) != str(r["X_sha256"]):
        raise ValueError(f"{name}: the inputs X differ from those the fixture was computed on")
    r["X"] = X
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
        np.savez_compressed(os.path.join(a.out, f"prunemx_{name}.npz"), **res)
        print(f"{name}: M={len(res['xt'])} cond(K)={float(res['cond']):.2e} ({time.perf_counter() - t0:.0f} s)",
              flush=True)
    print(f"total {time.perf_counter() - t00:.0f} s", flush=True)


if __name__ == "__main__":
    main()

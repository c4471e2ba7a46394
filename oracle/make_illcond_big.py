"""Double-double reference of the GP fit, posterior, selection and Kriging-believer conditioning at production sizes
on ill-conditioned training sets.

The 50-digit fixtures of oracle/make_illcond.py stop at N = 200 (two 128-row blocks).  These cases reach the shapes
the device runs at (N = 1000 .. 4096, d up to 17) with cond(K) from 1e7 to 1e11, and evaluate the same operations in
double-double arithmetic (oracle/dd.py, about 106 bits):

  K and L = chol(K); alpha_ = K^-1 y_n; at every candidate mu, sigma^2 = prior - |L^-1 k*|^2, UCB / EI / PoI; the LML
  and its gradient in sklearn's theta order; and one believer sequence (64 pending rows at geomspace(1e-2, 1e-6)
  from the incumbent, as make_illcond_ext's "incumbent" sequence) with its pivots, believer targets and sigma^2 at
  every candidate after 1, 8 and 64 rows.

The candidates are make_illcond.problem()'s groups followed by uniform rows up to CANDIDATES = 4296, so a selection
call over them has 34 tiles of 128 and the refine stages of pruning (DESIGN.md 4.9: N > 896 and at least 32 tiles)
run.  Each fixture, tests/golden/illbig_<case>.npz, stores the truth rounded to fp64 (diag(L) and the rows of L in
l_rows() rather than the whole factor) and sklearn's fp64 results on the same rows as the referee, and the inputs in a
compact form (stored() / load()):

  * X and the uniform candidate rows are plain MT19937 draws scaled and shifted in IEEE arithmetic, so load() rebuilds
    them bit-exactly from the case's seeds; the fixture keeps their SHA-256 digests, and load() refuses a rebuild
    that differs from the rows the truth was computed on.
  * y, the candidate rows of make_illcond.problem()'s groups and the pending rows go through libm (exp, sin, pow), so
    they are stored.
  * sklearn's UCB / EI / PoI are gp_oracle.base_acq of its stored mu and sigma; load() recomputes them.

Regenerate with

    python -m oracle.make_illcond_big                   # every case of CASES
    python -m oracle.make_illcond_big --only b_m15_d17  # some of them

About five minutes on 8 CPU cores for the whole table, most of it b_m25_c3; nothing here needs a GPU.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import time
import warnings

import mpmath as mp
import numpy as np

from oracle import dd
from oracle import make_illcond as MI
from oracle import make_illcond_ext as XE
from oracle.make_illcond import KAPPA, XI

CANDIDATES = 4296  # 34 tiles of 128 candidates
N_PEND = 64
PREFIXES = (1, 8, N_PEND)
# kern / ls / const / white / cluster / alpha as in make_illcond.CASES
CASES = {
    # the C3 shape: np = N (no padding), so the first pending row re-pitches every N^2 buffer
    "b_m25_c3": dict(kern="m25", d=16, n=4096, ls=1.0, cluster=(0.3, 1e-3), alpha=1e-6, seed=21),
    # just past the refine gate (np = 1024: eight row blocks); d = 17: phase A without candidate registers
    "b_m15_d17": dict(kern="m15", d=17, n=1000, ls=2.0, cluster=(0.5, 1e-3), alpha=1e-6, seed=22),
    # long length scale on the unit box at alpha = 1e-8: cond(K) 1e11; N ragged against 64 and 128
    "b_rbf_long": dict(kern="rbf", d=6, n=2000, ls=2.0, cluster=None, alpha=1e-8, seed=23),
    # ConstantKernel x Matern 1/2 ARD + WhiteKernel: a noise term and five length-scale gradients
    "b_m05_ard": dict(kern="m05", d=5, n=1500, ls=[0.5, 1.0, 2.0, 1.0, 0.5], const=4.0, white=1e-5,
                      cluster=(0.3, 1e-3), alpha=1e-6, seed=24),
}
SMALL_CASE = "b_m15_d17"


def l_rows(n):
    """Rows of L stored in full: both sides of the 64- and 128-row block edges at the start and in the middle of the
    factor, and the last row."""
    rows = {63, 64, 127, 128, n // 2 - 1, n // 2, n - 129, n - 1}
    return np.array(sorted(r for r in rows if 0 <= r < n), dtype=np.int64)


def uniform_inputs(case):
    """X and the uniform candidate rows after make_illcond.problem()'s groups: exact functions of the case's seeds."""
    X, _, head, _ = MI.problem(case)
    rs = np.random.RandomState(2000 + case["seed"])
    return X, rs.uniform(size=(CANDIDATES - len(head), case["d"]))


def problem(case):
    """make_illcond.problem()'s rows, then uniform candidates (group 'uniform') up to CANDIDATES, and the pending
    sequence."""
    _, y, xt, group = MI.problem(case)
    X, extra = uniform_inputs(case)
    xt = np.vstack([xt, extra])
    group = np.concatenate([group, np.full(len(extra), MI.G_UNIFORM, dtype=np.int8)])
    rs = np.random.RandomState(1000 + case["seed"])
    dirs = rs.randn(N_PEND, case["d"])
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    P = X[int(np.argmax(y))] + np.geomspace(1e-2, 1e-6, N_PEND)[:, None] * dirs
    return X, y, xt, group, P


def exact(case, X, y, xt, P):
    """The double-double results of a case, rounded to fp64."""
    mp.mp.dps = 50
    n = len(X)
    fit = dd.Fit(case, X, y, extra=N_PEND)
    Ps = dd.scaled(case, P)
    piv, Kp = fit.extend(Ps)
    Ks = fit.cross(dd.scaled(case, xt), np.vstack([fit.Xs, Ps]))
    mu = fit.mean(Ks)
    var = fit.variance(Ks, [n] + [n + p for p in PREFIXES])
    y_max = float(np.max(y))
    res = dict(mu=np.array([float(v) for v in mu]), var=np.array([float(v) for v in var[0]]))
    res.update(dd.acquisitions(mu, var[0], y_max, KAPPA, XI))
    for p, v in zip(PREFIXES, var[1:]):
        res[f"inc_p{p}_var"] = np.array([float(u) for u in v])
    res["inc_pivot"] = piv[0] + piv[1]
    res["inc_target"] = np.array([float(v) for v in fit.mean(Kp)])
    res["alpha_"] = fit.alpha_[0] + fit.alpha_[1]
    L = dd.l_dense(fit)
    res["L_diag"] = np.diag(L).copy()
    res["L_rows_idx"] = l_rows(n)
    res["L_rows"] = L[res["L_rows_idx"]]
    res["prior"] = float(fit.prior)
    res["y_std"] = float(fit.y_std)
    res["lml"] = float(fit.lml())
    res["lml_grad"] = fit.lml_grad()
    ev = np.linalg.eigvalsh(fit.K[0] + fit.K[1])
    res["cond"] = float(ev[-1] / ev[0])
    return res


def sklearn_results(case, X, y, xt, P):
    """sklearn's fp64 results on the same rows: make_illcond.sklearn_results, diag(L) and the stored rows of L, and
    the believer sequence through make_illcond_ext.sk_conditioned."""
    from sklearn.gaussian_process import GaussianProcessRegressor

    res = MI.sklearn_results(case, X, y, xt)
    sk = GaussianProcessRegressor(kernel=MI.sk_kernel(case), alpha=case["alpha"], normalize_y=True,
                                  optimizer=None).fit(X, y)
    res["sk_L_diag"] = np.diag(sk.L_).copy()
    res["sk_L_rows"] = sk.L_[l_rows(len(X))]
    for p in PREFIXES:
        aug, ym, ys, bel = XE.sk_conditioned(case, X, y, P[:p])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            res[f"sk_inc_p{p}_mu"], res[f"sk_inc_p{p}_sd"] = XE._sk_predict(aug, ym, ys, xt)
        if p == N_PEND:
            res["sk_inc_target"] = bel * ys + ym
            res["sk_inc_pivot"] = np.diag(aug.L_)[len(X):].copy()
    return res


def make_case(name, inputs=None):
    """Every array of the fixture of one case; `inputs` = (X, y, xt, group, P) instead of problem()'s."""
    case = CASES[name]
    X, y, xt, group, P = inputs if inputs is not None else problem(case)
    res = exact(case, X, y, xt, P)
    res.update(sklearn_results(case, X, y, xt, P))
    res.update(X=X, y=y, xt=xt, group=group, P=P)
    return res


def fixture_path(name):
    return os.path.join(MI.GOLDEN, f"illbig_{name}.npz")


SK_ACQ = {"ucb": "ACQ_UCB", "ei": "ACQ_EI", "poi": "ACQ_POI"}


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype="<f8").tobytes()).hexdigest()


def stored(res, case):
    """The arrays of make_case() as the fixture keeps them (module docstring)."""
    X, extra = uniform_inputs(case)
    head = len(res["xt"]) - len(extra)
    assert np.array_equal(res["X"], X) and np.array_equal(res["xt"][head:], extra)
    out = {k: v for k, v in res.items() if k not in ("X", "xt") and not k.startswith("sk_acq_")}
    out.update(xt_head=res["xt"][:head], X_sha256=np.array(_digest(X)), xt_tail_sha256=np.array(_digest(extra)))
    return out


def load(name, path=None):
    """Every array of make_case() from the fixture of a case: X and the uniform candidates rebuilt and checked against
    their digests, sklearn's acquisitions recomputed from its mu and sigma."""
    from oracle import gp_oracle as O

    case = CASES[name]
    with np.load(path or fixture_path(name)) as z:
        r = {k: z[k] for k in z.files}
    X, extra = uniform_inputs(case)
    if _digest(X) != str(r.pop("X_sha256")) or _digest(extra) != str(r.pop("xt_tail_sha256")):
        raise ValueError(f"{name}: the inputs rebuilt from the seeds differ from the fixture's")
    r["X"], r["xt"] = X, np.vstack([r.pop("xt_head"), extra])
    with np.errstate(all="ignore"):
        for kind, code in SK_ACQ.items():
            r[f"sk_acq_{kind}"] = O.base_acq(getattr(O, code), r["sk_mu"], r["sk_sd"], kappa=KAPPA, xi=XI,
                                             y_max=float(np.max(r["y"])))
    return r


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--only", nargs="*", default=None, help="case names (default: all)")
    ap.add_argument("--out", default=MI.GOLDEN)
    a = ap.parse_args(argv)
    for name in a.only or sorted(CASES):
        t0 = time.perf_counter()
        res = make_case(name)
        np.savez_compressed(os.path.join(a.out, f"illbig_{name}.npz"), **stored(res, CASES[name]))
        print(f"{name}: n={len(res['X'])} cond(K)={res['cond']:.2e} min var/prior="
              f"{np.min(res['var']) / (res['prior'] * res['y_std'] ** 2):.1e} ({time.perf_counter() - t0:.0f} s)",
              flush=True)


if __name__ == "__main__":
    main()

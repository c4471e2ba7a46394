"""Double-double reference of the posterior sample paths (DESIGN.md 4.7) at production sizes on ill-conditioned
training sets.

Problems: the four of oracle/make_illcond_big.py (N = 1000 .. 4096, cond(K) 6e6 .. 2e11) and b_m25_c5, bench.py's C5
shape (Matern 2.5, d = 32, N = 8192), with their 4296 candidates (make_illcond.problem()'s groups, then uniform rows).
On each, four draw sets from paths.draw_path_inputs, each from RandomState(seed(problem, set)):

  q16       q = 16, L = 4096   the QT = 16 instantiation of csrc/paths.cuh
  q4        q = 4,  L = 4096   QT = 4
  q1        q = 1,  L = 4096   QT = 1, what ThompsonSampling.suggest draws
  q5_L1000  q = 5,  L = 1000   QT = 16 with q < QT; L ragged against the 64-row stage and the 256-item gradient chunk

The truth is dd.Paths on dd.Fit: the features at the training rows, V = K^-1 (y_n - Phi w - eps) through the
double-double factor, then the values and the input gradients (the features through dd_cos_sin, the update term
through dd.cross_cov_grad).  Keys of tests/golden/pathbig_<problem>.npz, per set s:

  val_<s>        the values rounded to fp64: on every candidate for q16, on the rows `subset` (every row that is not
                 uniform, then uniform rows up to 1024) for the others
  gval_<s>, grad_<s>   value and gradient on the 64 rows `grad_rows` (make_nei_big.grad_rows()), path row mod q
  vabs_<s>, bound_<s>  per path sum_i |V_pi| and B_p = |y_mean| + s_y (sqrt(2c/L) sum_l |w_lp| + c sum_i |V_pi|)
  ident_<s>      max over the training-row candidates and paths of |f(X_i) - (y_mean + s_y (y_n,i - eps_i -
                 (white + alpha) V_i))| / (|f| + s_y), both sides unrounded: the feature and update terms agree
  phase_<s>      the largest |omega . xs + b| over the training rows and the candidates (fp64)
  train_eval_<s> per training-row candidate, the error of an fp64 sequential evaluation of c k*^T V with the true V
                 (train_eval()): the part of a path's error at a training row that no V solve can remove
  ref_err_<s>, ref_gerr_<s>   the referee's error against the truth per row (the largest over the paths on val_<s>'s
                 rows; on the grad rows the gradient metric of DESIGN.md 4.10)

The referee is tests/thompson_oracle.make_paths for the values and tests/grad_oracle.path_value_grad for the
gradients: fp64 with Cholesky solves on the same draws.  Only its errors are stored.  The inputs are not: they are
rebuilt (make_acq_big.inputs()) and checked against the SHA-256 digests kept here.

Regenerate with

    python oracle/make_paths_big.py                    # every problem (or python -m oracle.make_paths_big)
    python oracle/make_paths_big.py --only b_m15_d17   # some of them

Nothing here needs a GPU; the time per problem is printed (the module's total is recorded in DESIGN.md section 2).
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import mpmath as mp
import numpy as np

if __package__ in (None, ""):  # run as a script: the repository root, not oracle/, is the import root
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import dd  # noqa: E402
from oracle import make_acq_big as AB  # noqa: E402
from oracle import make_illcond as MI  # noqa: E402
from oracle import make_nei_big as NB  # noqa: E402

sys.path.insert(0, os.path.join(MI.ROOT, "tests"))
import grad_oracle as GO  # noqa: E402
import thompson_oracle as TO  # noqa: E402

PROBLEMS = AB.PROBLEMS
SMALL = "b_m15_d17"
SETS = {"q16": (16, 4096), "q4": (4, 4096), "q1": (1, 4096), "q5_L1000": (5, 1000)}
SUBSET = 1024
NU = {"m05": 0.5, "m15": 1.5, "m25": 2.5, "rbf": np.inf}


def seed(name, s):
    """The RandomState seed of draw set s on a problem."""
    return 5000 + 10 * AB.case(name)["seed"] + list(SETS).index(s)


def draws(name, s, n):
    """(omega, b, w, eps) of draw set s: what sample_paths(q, L, random_state=seed(name, s)) draws on the problem."""
    from bayesianoptimization_b200.paths import draw_path_inputs

    c = AB.case(name)
    q, L = SETS[s]
    return draw_path_inputs(np.random.RandomState(seed(name, s)), q, L, c["d"], NU[c["kern"]], n,
                            c["alpha"] + (c.get("white") or 0.0))


def subset(group):
    """Every candidate that is not uniform, then the first uniform ones up to SUBSET rows."""
    head = np.flatnonzero(group != MI.G_UNIFORM)
    uni = np.flatnonzero(group == MI.G_UNIFORM)[:SUBSET - len(head)]
    return np.sort(np.concatenate([head, uni]))


def rows_of(s, group):
    return np.arange(len(group)) if s == "q16" else subset(group)


def grad_metric(grad, want, val, ls):
    """DESIGN.md 4.10's gradient metric per row: max_j |d g_j| / (max_j |g_j| + |value| / l_min + 1e-6)."""
    scale = np.max(np.abs(want), axis=1) + np.abs(val) / np.min(ls) + 1e-6
    return np.max(np.abs(grad - want), axis=1) / scale


def value_metric(v, want, s_y):
    return np.abs(v - want) / (np.abs(want) + s_y)


def _max_phase(Xs, omega, b, chunk=512):
    out = 0.0
    for i in range(0, len(Xs), chunk):
        out = max(out, float(np.max(np.abs(Xs[i:i + chunk] @ omega.T + b))))
    return out


def train_eval(P, Ks, train, f, fit):
    """Per training-row candidate, the largest over the paths of the value metric of an fp64 evaluation of the
    truth's own path: c k*^T V summed in index order in fp64 from the fp64 roundings of c k* and of the true V, the
    rest exact.  This is the error a path evaluator leaves with no error in V at all: a sequential sum of N terms
    c k_i V_i, whose |V_i| grow toward 1/alpha while their sum stays O(1)."""
    kh = np.ascontiguousarray(Ks[0][train])
    Vh = P.V[0]
    acc = np.zeros((len(train), Vh.shape[0]))
    for i in range(Vh.shape[1]):
        acc = acc + kh[:, i:i + 1] * Vh[None, :, i]
    Uh, Ul = dd._rows_dot(kh, np.ascontiguousarray(Ks[1][train]), P.V[0], P.V[1])
    return np.array([float(max(abs(dd.to_mp(Uh[t, p], Ul[t, p]) - mp.mpf(float(acc[t, p]))) * fit.y_std
                               / (abs(f[t][p]) + fit.y_std) for p in range(acc.shape[1])))
                     for t in range(len(train))])


def truth(name, X, y, xt, group):
    c = AB.case(name)
    fit = dd.Fit(c, X, y)
    xs = dd.scaled(c, xt)
    Ks = fit.cross(xs)
    gi = NB.grad_rows(group)
    train = np.flatnonzero(group == MI.G_TRAIN)
    xi = np.array([int(np.flatnonzero(np.all(X == xt[t], axis=1))[0]) for t in train])
    out = dict(grad_rows=gi, subset=subset(group), y_std=float(fit.y_std), y_mean=float(fit.y_mean))
    for s, (q, L) in SETS.items():
        omega, b, w, eps = draws(name, s, len(X))
        P = dd.Paths(fit, omega, b, w, eps)
        rows = rows_of(s, group)
        Kr = (np.ascontiguousarray(Ks[0][rows]), np.ascontiguousarray(Ks[1][rows]))
        vals = P.values(xs[rows], Kr)
        out[f"val_{s}"] = np.array([[float(v) for v in row] for row in vals])
        pos = {int(t): k for k, t in enumerate(rows)}
        ident = mp.mpf(0)
        for t, i in zip(train, xi):
            for p in range(q):
                f = vals[pos[int(t)]][p]
                ident = max(ident, abs(f - P.train_identity(i, p)) / (abs(f) + fit.y_std))
        out[f"ident_{s}"] = np.array(float(ident))
        out[f"train_eval_{s}"] = train_eval(P, Ks, train, [vals[pos[int(t)]] for t in train], fit)
        gv = P.values(xs[gi], (np.ascontiguousarray(Ks[0][gi]), np.ascontiguousarray(Ks[1][gi])))
        gg = P.grads(xs[gi])
        out[f"gval_{s}"] = np.array([float(gv[k][t % q]) for k, t in enumerate(gi)])
        out[f"grad_{s}"] = np.array([[float(a) for a in gg[k][t % q]] for k, t in enumerate(gi)])
        out[f"vabs_{s}"] = np.array([float(v) for v in P.v_abs_sums()])
        out[f"bound_{s}"] = np.array([float(v) for v in P.bounds()])
        out[f"phase_{s}"] = np.array(max(_max_phase(fit.Xs, omega, b), _max_phase(xs, omega, b)))
    return out


def referee(name, X, y, xt, group, res):
    """The fp64 referee's errors against the truth."""
    c = AB.case(name)
    nu, ls = NU[c["kern"]], dd.ls_vec(c)
    const, white = float(c.get("const") or 1.0), float(c.get("white") or 0.0)
    kind = TO.KIND_RBF if nu == np.inf else TO.KIND_MATERN
    og = GO.GradGP(X, y, nu, ls, const, white, c["alpha"])
    gi = res["grad_rows"]
    out = {}
    for s, (q, L) in SETS.items():
        dr = draws(name, s, len(X))
        rows = rows_of(s, group)
        f = TO.make_paths(X, y, dr, kind=kind, nu=nu, length_scale=ls if np.iterable(c["ls"]) else float(c["ls"]),
                          const=const, alpha=c["alpha"], noise_level=white)
        v = np.vstack([f(xt[rows[i:i + 256]]) for i in range(0, len(rows), 256)])
        out[f"ref_err_{s}"] = np.max(value_metric(v, res[f"val_{s}"], res["y_std"]), axis=1)
        omega, b, w, eps = dr
        feat = np.sqrt(2.0 * const / L) * np.cos(og.Xs @ omega.T + b)
        from scipy.linalg import cho_solve

        V = cho_solve((og.L, True), og.y_norm[:, None] - feat @ w - eps)
        gv, gg = np.empty(len(gi)), np.empty((len(gi), X.shape[1]))
        for k, t in enumerate(gi):
            a, g = GO.path_value_grad(og, omega, b, w[:, t % q], V[:, t % q], xt[t:t + 1])
            gv[k], gg[k] = a[0], g[0]
        out[f"ref_gerr_{s}"] = grad_metric(gg, res[f"grad_{s}"], res[f"gval_{s}"], ls)
    return out


def make_problem(name, inputs=None):
    X, y, xt, group = inputs if inputs is not None else AB.inputs(name)
    res = truth(name, X, y, xt, group)
    res.update(referee(name, X, y, xt, group, res))
    res.update(X_sha256=np.array(AB._digest(X)), y_sha256=np.array(AB._digest(y)),
               xt_sha256=np.array(AB._digest(xt)), group=group,
               seeds=np.array([seed(name, s) for s in SETS]))
    return res


def fixture_path(name):
    return os.path.join(MI.GOLDEN, f"pathbig_{name}.npz")


def load(name, path=None):
    """The fixture of a problem with its inputs (X, y, xt), rebuilt and checked against the digests it keeps."""
    with np.load(path or fixture_path(name)) as z:
        r = {k: z[k] for k in z.files}
    X, y, xt, group = AB.inputs(name)
    for k, v in (("X", X), ("y", y), ("xt", xt)):
        if AB._digest(v) != str(r[f"{k}_sha256"]):
            raise ValueError(f"{name}: the inputs {k} differ from those the fixture was computed on")
    if not np.array_equal(group, r["group"]):
        raise ValueError(f"{name}: the candidate groups differ from the fixture's")
    r.update(X=X, y=y, xt=xt)
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
        np.savez_compressed(os.path.join(a.out, f"pathbig_{name}.npz"), **res)
        print(f"{name}: ident " + " ".join(f"{s} {float(res[f'ident_{s}']):.1e}" for s in SETS)
              + f" ({time.perf_counter() - t0:.0f} s)", flush=True)
    print(f"total {time.perf_counter() - t00:.0f} s", flush=True)


if __name__ == "__main__":
    main()

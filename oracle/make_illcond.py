"""Extended-precision reference of the GP posterior on ill-conditioned, clustered training sets.

Late in a Bayesian-optimisation run the registered points cluster around the incumbent and the fitted length scales
are long against their spacing, so cond(K) climbs towards the 1/alpha limit.  Both fp64 computations of the posterior
(sklearn's triangular solve and the device's product with the explicit inverse L^-1) then carry errors of order
cond(K) eps, and neither can referee the other.  This module builds such training sets from seeds and evaluates the
same operations at 50 significant digits with mpmath:

  K and L = chol(K); alpha_ = K^-1 y_n; at every candidate mu, the posterior variance prior - k*^T K^-1 k* (through
  V = L^-1 k*^T), UCB / EI / PoI; the log-marginal likelihood and its gradient in theta (sklearn's order).

The inputs are fp64 and enter exactly (length scales and ConstantKernel values are powers of two, so the scaled
inputs X / l are the same numbers in fp64 and in extended precision).  Results are rounded to fp64 and stored, with
the inputs and sklearn's fp64 results on the same rows, in tests/golden/illcond_<case>.npz.  Regenerate with

    python -m oracle.make_illcond                   # every case of CASES
    python -m oracle.make_illcond --only t_m25_d2   # some of them

(a few minutes of CPU for the whole table; nothing here needs a GPU).
"""
from __future__ import annotations

import argparse
import os
import warnings

import mpmath as mp
import numpy as np

DPS = 50
KAPPA, XI = 2.576, 0.01
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

# Candidate groups (the `group` array of a fixture)
G_CLUSTER, G_TRAIN, G_DUP7, G_DUP9, G_INC, G_UNIFORM = range(6)
GROUP_NAMES = ("cluster", "train", "dup1e-7", "dup1e-9", "incumbent", "uniform")

# ---------------------------------------------------------------------------------------------------------------
# Cases.  kern: m05 / m15 / m25 / rbf (covariance codes 0-3 of the device kernels); ls: a power of two (iso) or a
# list of them (ARD); const / white: ConstantKernel / WhiteKernel values (None: absent); cluster: (fraction of n,
# spread) of the points drawn around one centre, or None; alpha: the GPR's diagonal jitter.  N is never a multiple
# of 64 except where the append path needs the 128-row capacity, so the padding and the 64-row blocks of the
# look-ahead Cholesky and of the recursive-doubling inverse are crossed.
# ---------------------------------------------------------------------------------------------------------------
CASES = {
    # clustered late-run sets, d = 2, 3, 6, 17 (d = 17: phase A without candidate registers)
    "c_m25_d2": dict(kern="m25", d=2, n=150, ls=0.5, cluster=(0.4, 1e-2), alpha=1e-6, seed=1),
    "c_m25_d3": dict(kern="m25", d=3, n=121, ls=1.0, cluster=(0.3, 1e-3), alpha=1e-6, seed=2),
    "c_rbf_d6": dict(kern="rbf", d=6, n=200, ls=1.0, cluster=(0.25, 1e-4), alpha=1e-6, seed=3),
    "c_m15_d17": dict(kern="m15", d=17, n=130, ls=2.0, cluster=(0.5, 1e-3), alpha=1e-6, seed=4),
    "c_m05_ard": dict(kern="m05", d=3, n=140, ls=[0.5, 1.0, 2.0], const=4.0, white=1e-5, cluster=(0.3, 1e-3),
                      alpha=1e-6, seed=5),
    # long length scales on the unit box: cond(K) 1e8 .. 1e11, and alpha = 1e-8 / 1e-10
    "l_rbf_d3": dict(kern="rbf", d=3, n=190, ls=2.0, const=64.0, cluster=None, alpha=1e-6, seed=6),
    "l_m25_d4": dict(kern="m25", d=4, n=200, ls=4.0, const=8.0, cluster=None, alpha=1e-6, seed=7),
    "l_m15_a8": dict(kern="m15", d=2, n=97, ls=1.0, cluster=(0.2, 1e-2), alpha=1e-8, seed=8),
    "l_rbf_a10": dict(kern="rbf", d=2, n=90, ls=1.0, cluster=None, alpha=1e-10, seed=9),
    "l_m25_ard_d5": dict(kern="m25", d=5, n=170, ls=[1.0, 2.0, 1.0, 0.5, 2.0], const=2.0, white=1e-6,
                         cluster=(0.3, 1e-4), alpha=1e-6, seed=10),
    # the small case the CPU round-trip test regenerates
    "t_m25_d2": dict(kern="m25", d=2, n=70, ls=1.0, cluster=(0.3, 1e-3), alpha=1e-6, seed=11),
    # grown point by point from 60 to the 128-row capacity by the append path
    "a_m25_d3": dict(kern="m25", d=3, n=128, ls=1.0, cluster=(0.4, 1e-3), alpha=1e-6, seed=12),
}
SMALL_CASE = "t_m25_d2"


def _ls_vec(case):
    ls = case["ls"]
    return np.asarray(ls, dtype=float) if np.iterable(ls) else np.full(case["d"], float(ls))


def sk_kernel(case):
    """The sklearn kernel of a case (all hyper-parameters free, so theta has every one of them)."""
    from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, WhiteKernel

    ls = case["ls"]
    ls = list(map(float, ls)) if np.iterable(ls) else float(ls)
    nu = {"m05": 0.5, "m15": 1.5, "m25": 2.5}
    k = RBF(ls, length_scale_bounds=(1e-5, 1e5)) if case["kern"] == "rbf" else \
        Matern(ls, length_scale_bounds=(1e-5, 1e5), nu=nu[case["kern"]])
    if case.get("const") is not None:
        k = ConstantKernel(case["const"], constant_value_bounds=(1e-5, 1e5)) * k
    if case.get("white") is not None:
        k = k + WhiteKernel(case["white"], noise_level_bounds=(1e-12, 1e1))
    return k


def problem(case):
    """Training inputs and targets, and the candidate rows with their group labels.

    X: uniform rows in [0, 1]^d plus a cluster of `fraction * n` rows within `spread` (per coordinate) of a centre,
    shuffled so the cluster spreads over every row block.  y: a smooth bump at the centre (noise-free objective), so
    the incumbent lies in the cluster.  Candidates: 32 rows inside the cluster, 16 training rows (half of them from
    the cluster), each of those moved by 1e-7 and by 1e-9, 16 rows at 1e-2 .. 1e-8 from the incumbent, 64 uniform."""
    rs = np.random.RandomState(case["seed"])
    n, d = case["n"], case["d"]
    centre = rs.uniform(0.3, 0.7, size=d)
    nc = int(round(case["cluster"][0] * n)) if case.get("cluster") else 0
    spread = case["cluster"][1] if case.get("cluster") else 1e-2
    X = np.vstack([rs.uniform(size=(n - nc, d)), centre + spread * rs.uniform(-1, 1, size=(nc, d))])
    X = X[rs.permutation(n)]
    dc = np.sum((X - centre) ** 2, axis=1)
    y = np.exp(-8.0 * dc) + 0.3 * np.sin(3.0 * X.sum(1) / np.sqrt(d)) + 0.1 * X[:, 0] ** 2
    inc = int(np.argmax(y))
    near = np.argsort(dc, kind="stable")
    tr = np.concatenate([near[:8], rs.choice(near[8:], 8, replace=False)])
    steps = np.geomspace(1e-2, 1e-8, 16)
    dirs = rs.randn(16, d)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    groups = [
        (G_CLUSTER, centre + spread * rs.uniform(-1, 1, size=(32, d))),
        (G_TRAIN, X[tr]),
        (G_DUP7, X[tr] + 1e-7 * rs.choice([-1.0, 1.0], size=(16, d))),
        (G_DUP9, X[tr] + 1e-9 * rs.choice([-1.0, 1.0], size=(16, d))),
        (G_INC, X[inc] + steps[:, None] * dirs),
        (G_UNIFORM, rs.uniform(size=(64, d))),
    ]
    xt = np.vstack([g for _, g in groups])
    group = np.concatenate([np.full(len(g), c, dtype=np.int8) for c, g in groups])
    return X, y, xt, group


# ---------------------------------------------------------------------------------------------------------------
# extended-precision evaluation
# ---------------------------------------------------------------------------------------------------------------
def _cov(code, r2):
    """sklearn's covariance of the scaled squared distance r2 (SK kernels.py Matern.__call__ / RBF.__call__)."""
    if code == "rbf":
        return mp.exp(-r2 / 2)
    dist = mp.sqrt(r2)
    if code == "m05":
        return mp.exp(-dist)
    if code == "m15":
        k = dist * mp.sqrt(3)
        return (1 + k) * mp.exp(-k)
    k = dist * mp.sqrt(5)
    return (1 + k + k * k / 3) * mp.exp(-k)


def _grad_factor(code, r2, kv):
    """g with dk/dlog(l_t) = g * D_t, D_t = (dx_t / l_t)^2 (SK kernels.py, the eval_gradient branches)."""
    if code == "rbf":
        return kv
    if code == "m05":
        return kv / mp.sqrt(r2) if r2 != 0 else mp.mpf(0)
    if code == "m15":
        return 3 * mp.exp(-mp.sqrt(3 * r2))
    t = mp.sqrt(5 * r2)
    return mp.mpf(5) / 3 * (t + 1) * mp.exp(-t)


def _scaled(case, X):
    ls = _ls_vec(case)
    return [[mp.mpf(float(v)) / mp.mpf(float(l)) for v, l in zip(row, ls)] for row in X]


def _dsq(a, b):
    return [(u - v) ** 2 for u, v in zip(a, b)]


def kernel_matrix_mp(case, X):
    """K = const * k(X, X) + (white + alpha) I at DPS digits, as a list of rows."""
    mp.mp.dps = DPS
    Xs = _scaled(case, X)
    n = len(Xs)
    c = mp.mpf(case.get("const") or 1.0)
    diag = c + mp.mpf(case.get("white") or 0.0) + mp.mpf(case["alpha"])
    K = [[None] * n for _ in range(n)]
    for i in range(n):
        K[i][i] = diag
        for j in range(i):
            K[i][j] = K[j][i] = c * _cov(case["kern"], mp.fsum(_dsq(Xs[i], Xs[j])))
    return K


def _cholesky(K):
    n = len(K)
    L = [[mp.mpf(0)] * n for _ in range(n)]
    for j in range(n):
        s = K[j][j] - mp.fdot(L[j][:j], L[j][:j])
        if s <= 0:
            raise ValueError(f"K is not positive definite at row {j}")
        L[j][j] = mp.sqrt(s)
        for i in range(j + 1, n):
            L[i][j] = (K[i][j] - mp.fdot(L[i][:j], L[j][:j])) / L[j][j]
    return L


def _forward(L, b):
    v = []
    for i in range(len(b)):
        v.append((b[i] - mp.fdot(L[i][:i], v)) / L[i][i])
    return v


def _backward(L, z):
    n = len(z)
    x = [mp.mpf(0)] * n
    for i in range(n - 1, -1, -1):
        x[i] = (z[i] - mp.fdot([L[k][i] for k in range(i + 1, n)], x[i + 1:])) / L[i][i]
    return x


def _to64(rows):
    return np.array([[float(v) for v in r] for r in rows])


def _acq_mp(mu, sd, y_max):
    ucb = mu + KAPPA * sd
    a = mu - mp.mpf(y_max) - mp.mpf(XI)
    if sd == 0:
        return ucb, max(a, mp.mpf(0)), mp.mpf(1 if a > 0 else 0)
    z = a / sd
    return ucb, a * mp.ncdf(z) + sd * mp.npdf(z), mp.ncdf(z)


def exact(case, X, y, xt, with_grad=True):
    """The extended-precision results of a case, rounded to fp64."""
    mp.mp.dps = DPS
    n = len(X)
    K = kernel_matrix_mp(case, X)
    L = _cholesky(K)
    ym = [mp.mpf(float(v)) for v in y]
    mean = mp.fsum(ym) / n
    std = mp.sqrt(mp.fsum([(v - mean) ** 2 for v in ym]) / n)
    if std == 0:
        std = mp.mpf(1)
    yn = [(v - mean) / std for v in ym]
    alpha_ = _backward(L, _forward(L, yn))
    c = mp.mpf(case.get("const") or 1.0)
    prior = c + mp.mpf(case.get("white") or 0.0)
    Xs = _scaled(case, X)
    Xt = _scaled(case, xt)
    y_max = float(np.max(y))
    out = {k: [] for k in ("mu", "var", "sd", "acq_ucb", "acq_ei", "acq_poi")}
    for row in Xt:
        ks = [c * _cov(case["kern"], mp.fsum(_dsq(row, xr))) for xr in Xs]
        mu = mp.fdot(ks, alpha_) * std + mean
        V = _forward(L, ks)
        var = (prior - mp.fdot(V, V)) * std * std
        sd = mp.sqrt(var) if var > 0 else mp.mpf(0)
        u, e, p = _acq_mp(mu, sd, y_max)
        for k, v in zip(("mu", "var", "sd", "acq_ucb", "acq_ei", "acq_poi"), (mu, var, sd, u, e, p)):
            out[k].append(float(v))
    res = {k: np.array(v) for k, v in out.items()}
    Lf = _to64(L)
    res["L_packed"] = Lf[np.tril_indices(n)]
    res["alpha_"] = np.array([float(v) for v in alpha_])
    res["prior"] = float(prior)
    res["y_std"] = float(std)
    res["lml"] = float(-mp.fdot(yn, alpha_) / 2 - mp.fsum([mp.log(L[i][i]) for i in range(n)])
                       - n * mp.log(2 * mp.pi) / 2)
    # cond_2(K) from the fp64 rounding of K (the condition number only has to be right to a few digits)
    ev = np.linalg.eigvalsh(_to64(K))
    res["cond"] = float(ev[-1] / ev[0])
    if with_grad:
        res["lml_grad"] = _lml_grad(case, K, L, Xs, alpha_)
    return res


def _lml_grad(case, K, L, Xs, alpha_):
    """d lml / d theta = 1/2 sum_ij (alpha alpha^T - K^-1)_ij dK_ij / dtheta, theta = log of (const, length scales,
    white) in sklearn's order, every one of them free."""
    n = len(K)
    # K^-1 = W^T W with W = L^-1 (column by column through forward solves of the unit vectors)
    Wt = [_forward(L, [mp.mpf(1) if k == j else mp.mpf(0) for k in range(n)]) for j in range(n)]  # Wt[j] = W[:, j]
    Kinv = [[None] * n for _ in range(n)]
    for i in range(n):
        for j in range(i + 1):
            Kinv[i][j] = Kinv[j][i] = mp.fdot(Wt[i][max(i, j):], Wt[j][max(i, j):])
    ard = np.iterable(case["ls"])
    d = len(Xs[0])
    c = mp.mpf(case.get("const") or 1.0)
    nls = d if ard else 1
    g_c = mp.mpf(0)
    g_l = [mp.mpf(0)] * nls
    g_w = mp.mpf(0)
    for i in range(n):
        for j in range(i + 1):
            w = (alpha_[i] * alpha_[j] - Kinv[i][j]) * (1 if i == j else 2)
            D = _dsq(Xs[i], Xs[j])
            r2 = mp.fsum(D)
            kv = _cov(case["kern"], r2)
            g_c += w * c * kv
            gf = c * _grad_factor(case["kern"], r2, kv) * w
            if ard:
                for t in range(d):
                    g_l[t] += gf * D[t]
            else:
                g_l[0] += gf * r2
            if i == j:
                g_w += w
    grad = ([g_c] if case.get("const") is not None else []) + g_l
    if case.get("white") is not None:
        grad.append(g_w * mp.mpf(case["white"]))
    return np.array([float(g / 2) for g in grad])


def sklearn_results(case, X, y, xt):
    """sklearn's fp64 results on the same rows: mu, sd, the acquisitions, alpha_, LML and gradient."""
    from sklearn.gaussian_process import GaussianProcessRegressor

    from oracle import gp_oracle as O

    k = sk_kernel(case)
    sk = GaussianProcessRegressor(kernel=k, alpha=case["alpha"], normalize_y=True, optimizer=None).fit(X, y)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mu, sd = sk.predict(xt, return_std=True)
        acq = {kind: O.base_acq(code, mu, sd, kappa=KAPPA, xi=XI, y_max=float(np.max(y)))
               for kind, code in (("ucb", O.ACQ_UCB), ("ei", O.ACQ_EI), ("poi", O.ACQ_POI))}
    lml, grad = sk.log_marginal_likelihood(k.theta, eval_gradient=True)
    return dict(sk_mu=mu, sk_sd=sd, sk_acq_ucb=acq["ucb"], sk_acq_ei=acq["ei"], sk_acq_poi=acq["poi"],
                sk_alpha_=sk.alpha_, sk_lml=float(lml), sk_lml_grad=grad)


def make_case(name, inputs=None):
    """Every array of the fixture of one case; `inputs` = (X, y, xt, group) instead of problem()'s."""
    case = CASES[name]
    X, y, xt, group = inputs if inputs is not None else problem(case)
    res = exact(case, X, y, xt)
    res.update(sklearn_results(case, X, y, xt))
    res.update(X=X, y=y, xt=xt, group=group)
    return res


def fixture_path(name):
    return os.path.join(GOLDEN, f"illcond_{name}.npz")


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--only", nargs="*", default=None, help="case names (default: all)")
    ap.add_argument("--out", default=GOLDEN)
    a = ap.parse_args(argv)
    for name in a.only or sorted(CASES):
        res = make_case(name)
        np.savez_compressed(os.path.join(a.out, f"illcond_{name}.npz"), **res)
        print(f"{name}: n={len(res['X'])} cond(K)={res['cond']:.2e} min var/prior="
              f"{np.min(res['var']) / (res['prior'] * res['y_std'] ** 2):.1e}")


if __name__ == "__main__":
    main()

"""Extended-precision reference of the conditioned posterior, the sample paths and the input gradients on the
ill-conditioned training sets of oracle/make_illcond.py.

Three device features grow or differentiate the posterior of a fitted GP, and on clustered, long-length-scale sets
their fp64 restatements carry errors of order cond(K) eps like the posterior itself:

  a. Kriging-believer conditioning (DESIGN.md 4.11).  Three pending sequences per case: "incumbent" (64 rows at
     geomspace(1e-2, 1e-6) from the incumbent), "edge" (7 rows 1e-7 from the training rows nearest the incumbent,
     8 rows inside the cluster, then an exact repeat of pending row 2) and "believer" (16 greedy picks of EI over the
     case's candidates under the fp64 conditioned posterior).  The truth holds each row's believer target (the
     original mu), every new pivot L[n+r, n+r], and for the prefixes p = 1, 8 and all of each sequence mu, sigma^2,
     UCB, EI and PoI at the case's candidates.  The leading block of the Cholesky factor does not change when rows
     are appended, so the 50-digit factor of K is extended row by row and serves every prefix.
  b. Posterior sample paths (DESIGN.md 4.7): q = 4 paths with L = 512 features drawn from RandomState(case seed) by
     paths.draw_path_inputs; v = K^-1 (y_n - Phi w - eps), the path values and their input gradients.
  c. Input gradients (DESIGN.md 4.10): value and gradient of the closures -UCB, -EI, -PoI and -MES (y* = y_max +
     s_y {1e-3, 1e-2, 1e-1, 1}) on the original GP and on the GP conditioned on the first 8 "incumbent" rows, with
     d sigma^2 = -2 dk*^T K^-1 k* from the kernel derivatives (the Matern 1/2 term at r = 0 contributes 0).

Each fixture, tests/golden/illext_<case>.npz, stores the inputs, the truth rounded to fp64 and the fp64 referee's
results on the same rows: sklearn refitted on [X; P] with the normalised targets followed by the believer targets
(normalize_y=False, the original statistics re-applied) for (a), and tests/grad_oracle.py for (b) and (c).
Regenerate with

    python -m oracle.make_illcond_ext                   # every case of make_illcond.CASES
    python -m oracle.make_illcond_ext --only t_m25_d2   # some of them

(a few minutes of CPU; nothing here needs a GPU).
"""
from __future__ import annotations

import argparse
import os
import sys
import warnings
from concurrent.futures import ProcessPoolExecutor

import mpmath as mp
import numpy as np

from oracle import make_illcond as MI
from oracle.make_illcond import DPS, KAPPA, XI

SEQS = ("incumbent", "edge", "believer")
N_INC, N_EDGE, N_BEL = 64, 16, 16
EDGE_REPEAT = (15, 2)  # edge row 15 repeats edge row 2 exactly
N_PATHS, N_FEATURES = 4, 512
MES_OFFSETS = (1e-3, 1e-2, 1e-1, 1.0)  # y* = y_max + s_y * offset
N_COND_GRAD = 8  # the conditioned GP of (c): the first 8 "incumbent" rows
GPS = ("orig", "cond")
KINDS = ("ucb", "ei", "poi", "mes")
NU = {"m05": 0.5, "m15": 1.5, "m25": 2.5, "rbf": np.inf}


def prefixes(seq):
    return (1, 8, {"incumbent": N_INC, "edge": N_EDGE, "believer": N_BEL}[seq])


def fixture_path(name):
    return os.path.join(MI.GOLDEN, f"illext_{name}.npz")


def _tests_path():
    p = os.path.join(MI.ROOT, "tests")
    if p not in sys.path:
        sys.path.insert(0, p)


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def sk_conditioned(case, X, y, P):
    """sklearn's fp64 GP of a case conditioned on P: fitted on [X; P] with the normalised targets followed by the
    believer targets mu_norm(P) of the original fit, normalize_y=False.  Returns (gp, y_mean, y_std, mu_norm(P))."""
    from sklearn.gaussian_process import GaussianProcessRegressor

    sk = GaussianProcessRegressor(kernel=MI.sk_kernel(case), alpha=case["alpha"], normalize_y=True,
                                  optimizer=None).fit(X, y)
    ym, ys = float(np.ravel(sk._y_train_mean)[0]), float(np.ravel(sk._y_train_std)[0])
    bel = sk.kernel_(P, sk.X_train_) @ sk.alpha_ if len(P) else np.empty(0)
    aug = GaussianProcessRegressor(kernel=sk.kernel_, alpha=case["alpha"], normalize_y=False, optimizer=None)
    aug.fit(np.vstack([X, P]), np.concatenate([sk.y_train_, bel]))
    return aug, ym, ys, bel


def _sk_predict(aug, ym, ys, x):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mu, sd = aug.predict(x, return_std=True)
    return mu * ys + ym, sd * ys


def believer_picks(case, X, y, xt):
    """N_BEL greedy picks: each the argmax of EI over the candidates not picked yet, under the fp64 GP conditioned on
    the earlier picks (the random stage of a Kriging-believer batch)."""
    from oracle import gp_oracle as O

    y_max = float(np.max(y))
    free = np.ones(len(xt), dtype=bool)
    picks = []
    for _ in range(N_BEL):
        aug, ym, ys, _ = sk_conditioned(case, X, y, xt[picks])
        mu, sd = _sk_predict(aug, ym, ys, xt)
        with np.errstate(all="ignore"):
            ei = O.base_acq(O.ACQ_EI, mu, sd, kappa=KAPPA, xi=XI, y_max=y_max)
        ei = np.where(free & np.isfinite(ei), ei, -np.inf)
        j = int(np.argmax(ei))
        picks.append(j)
        free[j] = False
    return np.array(picks)


def pending_inputs(case, X, y, xt):
    """The three pending sequences of a case (module docstring)."""
    rs = np.random.RandomState(1000 + case["seed"])
    d = X.shape[1]
    inc = int(np.argmax(y))
    dirs = rs.randn(N_INC, d)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    p_inc = X[inc] + np.geomspace(1e-2, 1e-6, N_INC)[:, None] * dirs
    near = np.argsort(np.sum((X - X[inc]) ** 2, axis=1), kind="stable")[:7]
    spread = case["cluster"][1] if case.get("cluster") else 1e-2
    p_edge = np.vstack([X[near] + 1e-7 * rs.choice([-1.0, 1.0], size=(7, d)),
                        X[inc] + spread * rs.uniform(-1, 1, size=(8, d))])
    p_edge = np.vstack([p_edge, p_edge[EDGE_REPEAT[1]]])
    picks = believer_picks(case, X, y, xt)
    return dict(P_incumbent=p_inc, P_edge=p_edge, P_believer=xt[picks], believer_idx=picks)


def path_draws(case, n):
    from bayesianoptimization_b200.paths import draw_path_inputs

    return draw_path_inputs(np.random.RandomState(case["seed"]), N_PATHS, N_FEATURES, case["d"], NU[case["kern"]], n,
                            case["alpha"] + (case.get("white") or 0.0))


# ---------------------------------------------------------------------------------------------------------------
# extended precision
# ---------------------------------------------------------------------------------------------------------------
def _h(code, r):
    """h(r) = -(1/r) dk/dr of the unit covariance, h(0) := 0 for Matern 1/2 (the ABI's rule at a training input)."""
    if code == "rbf":
        return mp.exp(-r * r / 2)
    if code == "m05":
        return mp.exp(-r) / r if r != 0 else mp.mpf(0)
    if code == "m15":
        return 3 * mp.exp(-mp.sqrt(3) * r)
    t = mp.sqrt(5) * r
    return mp.mpf(5) / 3 * (1 + t) * mp.exp(-t)


def _mes_term(g):
    return g * mp.npdf(g) / (2 * mp.ncdf(g)) - mp.log(mp.ncdf(g))


def _closures(mu, sd, dmu, dsd, y_max, ystar):
    """{kind: (value, gradient)} of the closures -base at one row (data units)."""
    a = mu - mp.mpf(y_max) - mp.mpf(XI)
    z = a / sd
    out = {"ucb": (mu + KAPPA * sd, [m + KAPPA * s for m, s in zip(dmu, dsd)]),
           "ei": (a * mp.ncdf(z) + sd * mp.npdf(z), [mp.ncdf(z) * m + mp.npdf(z) * s for m, s in zip(dmu, dsd)]),
           "poi": (mp.ncdf(z), [mp.npdf(z) / sd * (m - z * s) for m, s in zip(dmu, dsd)])}
    val, cm, cs = mp.mpf(0), mp.mpf(0), mp.mpf(0)
    for ys in ystar:
        g = (mp.mpf(ys) - mu) / sd
        t = mp.diff(_mes_term, g)
        val += _mes_term(g)
        cm -= t / sd
        cs -= t * g / sd
    k = len(ystar)
    out["mes"] = (val / k, [(cm * m + cs * s) / k for m, s in zip(dmu, dsd)])
    return {kind: (-v, [-x for x in g]) for kind, (v, g) in out.items()}


def exact_ext(case, X, y, xt, seqs, draws):
    """The truth of (a), (b) and (c), rounded to fp64."""
    mp.mp.dps = DPS
    n, d = X.shape
    code = case["kern"]
    K = MI.kernel_matrix_mp(case, X)
    L = MI._cholesky(K)
    ym = [mp.mpf(float(v)) for v in y]
    mean = mp.fsum(ym) / n
    std = mp.sqrt(mp.fsum([(v - mean) ** 2 for v in ym]) / n)
    yn = [(v - mean) / std for v in ym]
    alpha_ = MI._backward(L, MI._forward(L, yn))
    c = mp.mpf(case.get("const") or 1.0)
    prior = c + mp.mpf(case.get("white") or 0.0)
    diag = prior + mp.mpf(case["alpha"])
    ls = [mp.mpf(float(v)) for v in MI._ls_vec(case)]
    Xs, Xt = MI._scaled(case, X), MI._scaled(case, xt)
    y_max = float(np.max(y))

    def cov(a, b):
        return c * MI._cov(code, mp.fsum(MI._dsq(a, b)))

    ks = [[cov(row, xr) for xr in Xs] for row in Xt]
    V0 = [MI._forward(L, k) for k in ks]
    mu = [mp.fdot(k, alpha_) * std + mean for k in ks]
    res = {}
    # (a) conditioning: the factor extended row by row, V extended per candidate
    Vinc = None
    for s in SEQS:
        Ps = MI._scaled(case, seqs[f"P_{s}"])
        Lx, rows, piv, bel = [r[:] for r in L], list(Xs), [], []
        for x in Ps:
            k = [cov(x, r) for r in rows]
            l = MI._forward(Lx, k)
            p2 = diag - mp.fdot(l, l)
            if p2 <= 0:
                raise ValueError(f"{s}: the extended K is not positive definite at row {len(rows)}")
            Lx.append(l + [mp.sqrt(p2)])
            rows.append(x)
            piv.append(mp.sqrt(p2))
            bel.append(mp.fdot(k[:n], alpha_) * std + mean)
        res[f"{s}_pivot"] = np.array([float(v) for v in piv])
        res[f"{s}_target"] = np.array([float(v) for v in bel])
        Vx = []
        for t, row in enumerate(Xt):
            V = V0[t][:]
            for r, x in enumerate(Ps):
                V.append((cov(row, x) - mp.fdot(Lx[n + r][:n + r], V)) / Lx[n + r][n + r])
            Vx.append(V)
        for p in prefixes(s):
            out = {k: [] for k in ("mu", "var", "acq_ucb", "acq_ei", "acq_poi")}
            for t in range(len(Xt)):
                var = (prior - mp.fdot(Vx[t][:n + p], Vx[t][:n + p])) * std * std
                u, e, q = MI._acq_mp(mu[t], mp.sqrt(var), y_max)
                for k, v in zip(out, (mu[t], var, u, e, q)):
                    out[k].append(float(v))
            for k, v in out.items():
                res[f"{s}_p{p}_{k}"] = np.array(v)
        if s == "incumbent":
            Vinc, Linc, rows_inc = Vx, Lx, rows
    # (c) input gradients on the original GP and on the one conditioned on the first N_COND_GRAD incumbent rows
    ystar = [y_max + float(std) * o for o in MES_OFFSETS]
    for gname in GPS:
        m = n if gname == "orig" else n + N_COND_GRAD
        Lg, rows_g = Linc[:m], rows_inc[:m]
        vals = {k: [] for k in KINDS}
        grads = {k: [] for k in KINDS}
        for t, row in enumerate(Xt):
            V = Vinc[t][:m]
            u = MI._backward(Lg, V)
            dk = []
            for xr in rows_g:
                diff = [a - b for a, b in zip(row, xr)]
                hr = c * _h(code, mp.sqrt(mp.fsum([q * q for q in diff])))
                dk.append([-hr * q / l for q, l in zip(diff, ls)])
            dmu = [std * mp.fdot(alpha_, [dk[i][j] for i in range(n)]) for j in range(d)]
            dvar = [-2 * std * std * mp.fdot(u, [dk[i][j] for i in range(m)]) for j in range(d)]
            sd = mp.sqrt((prior - mp.fdot(V, V)) * std * std)
            dsd = [v / (2 * sd) for v in dvar]
            for kind, (v, g) in _closures(mu[t], sd, dmu, dsd, y_max, ystar).items():
                vals[kind].append(float(v))
                grads[kind].append([float(q) for q in g])
        for kind in KINDS:
            res[f"gr_{gname}_{kind}_val"] = np.array(vals[kind])
            res[f"gr_{gname}_{kind}_grad"] = np.array(grads[kind])
    res["mes_ystar"] = np.array(ystar)
    # (b) sample paths
    omega, b, w, eps = draws
    om = [[mp.mpf(float(v)) for v in r] for r in omega]
    bm = [mp.mpf(float(v)) for v in b]
    fs = mp.sqrt(2 * c / N_FEATURES)

    def phases(xs):
        return [mp.fdot(o, xs) + bb for o, bb in zip(om, bm)]

    wm = [[mp.mpf(float(v)) for v in r] for r in w]
    rhs = [[mp.mpf(0)] * n for _ in range(N_PATHS)]
    for i, xs in enumerate(Xs):
        f = [fs * mp.cos(ph) for ph in phases(xs)]
        for q in range(N_PATHS):
            rhs[q][i] = yn[i] - mp.fdot(f, [wr[q] for wr in wm]) - mp.mpf(float(eps[i, q]))
    v = [MI._backward(L, MI._forward(L, r)) for r in rhs]
    pv, pg = [], []
    for t, row in enumerate(Xt):
        ph = phases(row)
        cs, sn = [mp.cos(a) for a in ph], [mp.sin(a) for a in ph]
        hs = [c * _h(code, mp.sqrt(mp.fsum(MI._dsq(row, xr)))) for xr in Xs]
        vrow, grow = [], []
        for q in range(N_PATHS):
            wq = [wr[q] for wr in wm]
            vrow.append(std * (fs * mp.fdot(cs, wq) + mp.fdot(ks[t], v[q])) + mean)
            ws = [a * bb for a, bb in zip(wq, sn)]
            hv = [a * bb for a, bb in zip(hs, v[q])]
            grow.append([float(std / ls[j] * (-fs * mp.fdot(ws, [o[j] for o in om])
                                                - mp.fdot(hv, [row[j] - xr[j] for xr in Xs]))) for j in range(d)])
        pv.append([float(a) for a in vrow])
        pg.append(grow)
    res["path_val"] = np.array(pv)                      # (m, q)
    res["path_grad"] = np.array(pg)  # (m, q, d)
    res["path_v"] = np.array([[float(a) for a in r] for r in v]).T  # (n, q)
    return res


# ---------------------------------------------------------------------------------------------------------------
# fp64 referee
# ---------------------------------------------------------------------------------------------------------------
def _grad_gp(case, X, y, P=None):
    """grad_oracle.GradGP of a case, conditioned on P with fp64 believer targets when P is given."""
    _tests_path()
    import grad_oracle as G

    args = (NU[case["kern"]], MI._ls_vec(case), case.get("const") or 1.0, case.get("white") or 0.0, case["alpha"])
    base = G.GradGP(X, y, *args)
    if P is None:
        return base
    mu_p = base.predict_grad(P)[0]
    aug = G.GradGP(np.vstack([X, P]), np.concatenate([base.y_norm, (mu_p - base.y_mean) / base.y_std]), *args,
                   normalize=False)
    aug.y_mean, aug.y_std = base.y_mean, base.y_std
    return aug


def referee(case, X, y, xt, seqs, draws, ystar):
    from scipy.linalg import cho_solve

    from oracle import gp_oracle as O

    _tests_path()
    import grad_oracle as G

    y_max = float(np.max(y))
    res = {}
    for s in SEQS:
        P = seqs[f"P_{s}"]
        for p in prefixes(s):
            aug, ym, ys, bel = sk_conditioned(case, X, y, P[:p])
            mu, sd = _sk_predict(aug, ym, ys, xt)
            res[f"sk_{s}_p{p}_mu"], res[f"sk_{s}_p{p}_sd"] = mu, sd
            for kind, code in (("ucb", O.ACQ_UCB), ("ei", O.ACQ_EI), ("poi", O.ACQ_POI)):
                with np.errstate(all="ignore"):
                    res[f"sk_{s}_p{p}_acq_{kind}"] = O.base_acq(code, mu, sd, kappa=KAPPA, xi=XI, y_max=y_max)
        res[f"sk_{s}_target"] = bel * ys + ym
        res[f"sk_{s}_pivot"] = np.diag(aug.L_)[len(X):]
    kinds = dict(ucb=(G.UCB, dict(kappa=KAPPA)), ei=(G.EI, dict(xi=XI, y_max=y_max)),
                 poi=(G.POI, dict(xi=XI, y_max=y_max)), mes=(G.MES, dict(ystar=ystar)))
    for gname in GPS:
        og = _grad_gp(case, X, y, None if gname == "orig" else seqs["P_incumbent"][:N_COND_GRAD])
        for kind, (code, kw) in kinds.items():
            with np.errstate(all="ignore"):
                v, g = G.acq_value_grad(code, og, xt, **kw)
            res[f"sk_gr_{gname}_{kind}_val"], res[f"sk_gr_{gname}_{kind}_grad"] = v, g
    og = _grad_gp(case, X, y)
    omega, b, w, eps = draws
    feat = np.sqrt(2.0 * og.const / N_FEATURES) * np.cos(og.Xs @ omega.T + b)
    V = cho_solve((og.L, True), og.y_norm[:, None] - feat @ w - eps)
    pv, pg = [], []
    for q in range(N_PATHS):
        v, g = G.path_value_grad(og, omega, b, w[:, q], V[:, q], xt)
        pv.append(v)
        pg.append(g)
    res["sk_path_val"] = np.stack(pv, axis=1)
    res["sk_path_grad"] = np.stack(pg, axis=1)
    return res


def make_case(name, inputs=None):
    """Every array of the fixture of one case.  `inputs`: a dict with X, y, xt, group, the pending sequences
    (P_incumbent, P_edge, P_believer, believer_idx) and the draws (omega, b, w, eps) instead of the builders'."""
    case = MI.CASES[name]
    if inputs is None:
        X, y, xt, group = MI.problem(case)
        inputs = dict(X=X, y=y, xt=xt, group=group, **pending_inputs(case, X, y, xt))
        inputs.update(zip(("omega", "b", "w", "eps"), path_draws(case, len(X))))
    inputs = {k: np.asarray(v) for k, v in inputs.items()}
    X, y, xt = inputs["X"], inputs["y"], inputs["xt"]
    draws = tuple(inputs[k] for k in ("omega", "b", "w", "eps"))
    res = exact_ext(case, X, y, xt, inputs, draws)
    res.update(referee(case, X, y, xt, inputs, draws, res["mes_ystar"]))
    res.update(inputs)
    return res


def _build(args):
    name, out = args
    res = make_case(name)
    np.savez_compressed(os.path.join(out, f"illext_{name}.npz"), **res)
    return (f"{name}: n={len(res['X'])} min pivot "
            + " ".join(f"{s} {np.min(res[f'{s}_pivot']):.1e}" for s in SEQS))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--only", nargs="*", default=None, help="case names (default: all)")
    ap.add_argument("--out", default=MI.GOLDEN)
    ap.add_argument("--jobs", type=int, default=os.cpu_count() or 1)
    a = ap.parse_args(argv)
    names = a.only or sorted(MI.CASES)
    with ProcessPoolExecutor(max_workers=max(1, min(a.jobs, len(names)))) as ex:
        for line in ex.map(_build, [(n, a.out) for n in names]):
            print(line, flush=True)


if __name__ == "__main__":
    main()

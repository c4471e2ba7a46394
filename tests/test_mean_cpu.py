"""The posterior-mean merit (B200BO_ACQ_MEAN, DESIGN.md 4.17) without a device: the numpy restatement
(tests/mean_oracle.py) against sklearn on every covariance variant, the bound B on adversarial GPs, the feasible-first
ranking, the gradient against central differences, the ABI constant, and recommend()'s no-device error."""
import os
import re
import warnings

import numpy as np
import pytest
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, WhiteKernel

import mean_oracle as MO
from grad_oracle import GradGP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALPHA = 1e-6
COVS = {"m05": 0.5, "m15": 1.5, "m25": 2.5, "rbf": np.inf}


def _sk_kernel(nu, ls, const, noise):
    base = RBF(ls) if nu == np.inf else Matern(ls, nu=nu)
    k = ConstantKernel(const) * base
    return k + WhiteKernel(noise) if noise else k


def _pair(nu, X, y, ls, const=1.0, noise=0.0):
    """The same GP as sklearn's regressor at fixed hyper-parameters and as the restatement's GradGP."""
    sk = GaussianProcessRegressor(_sk_kernel(nu, ls, const, noise), alpha=ALPHA, normalize_y=True,
                                  optimizer=None).fit(X, y)
    return sk, GradGP(X, y, nu, ls, const=const, noise=noise, alpha=ALPHA)


def _problem(rs, n, d):
    X = rs.uniform(size=(n, d))
    return X, np.sin(3 * X.sum(1)) + 0.1 * rs.randn(n)


@pytest.mark.parametrize("cov", sorted(COVS))
@pytest.mark.parametrize("ard", [False, True])
def test_restatement_matches_sklearn(cov, ard):
    rs = np.random.RandomState(7 + 2 * sorted(COVS).index(cov) + ard)
    d, n = 4, 60
    ls = np.geomspace(0.3, 2.0, d) if ard else 0.6
    X, y = _problem(rs, n, d)
    tgt = _pair(COVS[cov], X, y, ls, const=1.7, noise=1e-2)
    s = X.sum(1)
    cons = [_pair(COVS[cov], X, np.cos(2 * s), ls), _pair(COVS[cov], X, np.sin(s) + X[:, 0], ls, const=0.5)]
    bounds = [(-0.6, 0.6), (-np.inf, 1.5)]
    xt = np.vstack([rs.uniform(size=(400, d)), X[:5]])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mu_sk = [m.predict(xt) for m, _ in [tgt, *cons]]
    mu_or = [g.predict_grad(xt)[0] for _, g in [tgt, *cons]]
    for a, b in zip(mu_sk, mu_or):
        np.testing.assert_allclose(b, a, rtol=1e-9, atol=1e-12)
    # T from the restatement's alpha_ and sklearn's: the same bound
    g0 = tgt[1]
    T = MO.bound_T(g0.y_mean, g0.y_std, g0.const, g0.alpha_)
    T_sk = MO.bound_T(tgt[0]._y_train_mean, tgt[0]._y_train_std, 1.7, tgt[0].alpha_)
    assert T == pytest.approx(T_sk, rel=1e-9)
    lb, ub = [b[0] for b in bounds], [b[1] for b in bounds]
    v_sk = MO.value(mu_sk[0], mu_sk[1:], lb, ub, T_sk)
    v_or = MO.value(mu_or[0], mu_or[1:], lb, ub, T)
    feas_sk = MO.violation(mu_sk[1:], lb, ub, len(xt)) == 0
    feas_or = MO.violation(mu_or[1:], lb, ub, len(xt)) == 0
    # rows whose constraint means sit within round-off of a bound may fall either side
    edge = np.zeros(len(xt), bool)
    for mu, lo, hi in zip(mu_sk[1:], lb, ub):
        edge |= np.isclose(mu, lo, rtol=0, atol=1e-9) | np.isclose(mu, hi, rtol=0, atol=1e-9)
    assert np.array_equal(feas_sk[~edge], feas_or[~edge])
    assert 0 < feas_sk.sum() < len(xt)
    np.testing.assert_allclose(v_or[~edge], v_sk[~edge], rtol=1e-9, atol=1e-12)
    # unconstrained: -mu
    np.testing.assert_array_equal(MO.value(mu_or[0], T=T), -mu_or[0])


def test_bound_holds_on_adversarial_gps():
    rs = np.random.RandomState(3)
    d = 6
    for cov in sorted(COVS):
        # near-duplicate rows with opposite targets: a huge, oscillating alpha_; ARD over six decades
        base = rs.uniform(size=(30, d))
        X = np.vstack([base, base + 1e-6 * rs.randn(30, d)])
        y = np.concatenate([rs.randn(30), -rs.randn(30)]) * 50 + 3
        g = GradGP(X, y, COVS[cov], np.geomspace(1e-3, 1e3, d), const=2.3, alpha=1e-10)
        assert np.max(np.abs(g.alpha_)) > 1e3
        T = MO.bound_T(g.y_mean, g.y_std, g.const, g.alpha_)
        B = (T - 1.0) / 2.0
        xt = np.vstack([rs.uniform(size=(2000, d)), X, X + 1e-7, 1e3 * rs.uniform(size=(10, d))])
        mu = g.predict_grad(xt)[0]
        assert np.all(np.abs(mu) < B), cov


def test_feasible_rows_rank_first():
    rs = np.random.RandomState(11)
    m = 5000
    mu0 = rs.randn(m) * 1e3
    T = 2 * (np.max(np.abs(mu0)) + 1) + 1
    cm = [rs.randn(m), rs.randn(m) * 5]
    lb, ub = [-1.0, -np.inf], [0.8, 2.0]
    v = MO.value(mu0, cm, lb, ub, T)
    feas = MO.violation(cm, lb, ub, m) == 0
    assert 0 < feas.sum() < m
    assert v[feas].max() < v[~feas].min()
    # nothing feasible: the least violation ranks first, by violation alone
    cm2 = [np.abs(rs.randn(m)) + 1.0]
    viol = MO.violation(cm2, [-1.0], [0.5], m)
    v2 = MO.value(mu0, cm2, [-1.0], [0.5], T)
    assert np.all(viol > 0)
    order = np.argsort(v2, kind="stable")
    assert np.all(np.diff(viol[order]) >= 0)
    # boundary counts as feasible; a NaN constraint mean makes the value NaN; infinite bounds ignore it
    assert MO.value(np.array([2.0]), [np.array([0.5])], [-1.0], [0.5], T)[0] == -2.0
    assert np.isnan(MO.value(np.array([2.0]), [np.array([np.nan])], [-1.0], [0.5], T)[0])
    assert MO.value(np.array([2.0]), [np.array([np.nan])], [-np.inf], [np.inf], T)[0] == -2.0


@pytest.mark.parametrize("cov", ["m15", "m25", "rbf"])
def test_gradient_matches_central_differences(cov):
    rs = np.random.RandomState(5)
    d, n = 3, 40
    X, y = _problem(rs, n, d)
    s = X.sum(1)
    tgt = GradGP(X, y, COVS[cov], 0.5, const=1.3)
    cons = [(GradGP(X, np.cos(2 * s), COVS[cov], 0.7), -0.2, 0.3),
            (GradGP(X, X[:, 1] - X[:, 0], COVS[cov], 0.8), -np.inf, 0.1)]
    xt = rs.uniform(size=(200, d))
    val, grad = MO.value_grad(tgt, xt, cons)
    h = 1e-6

    def f(x):
        return MO.value_grad(tgt, x, cons)[0]

    checked = 0
    for i in range(len(xt)):
        x = xt[i]
        # away from the kinks: every constraint mean farther than the step's reach from its bounds
        mus = [g.predict_grad(x)[0][0] for g, _, _ in cons]
        if any(min(abs(mu - lo), abs(mu - hi)) < 1e-3 for mu, (_, lo, hi) in zip(mus, cons)):
            continue
        fd = np.array([(f(x + h * e) - f(x - h * e))[0] / (2 * h) for e in np.eye(d)])
        np.testing.assert_allclose(grad[i], fd, rtol=1e-5, atol=1e-6 * max(1.0, abs(val[i])))
        checked += 1
    assert checked > 100


def test_abi_constant():
    from bayesianoptimization_b200 import _lib as B

    with open(os.path.join(ROOT, "include", "b200bo.h")) as f:
        hdr = f.read()
    assert re.search(r"#define B200BO_ACQ_MEAN 12\b", hdr)
    assert B.ACQ_MEAN == 12
    src = open(os.path.join(ROOT, "bayesianoptimization_b200", "csrc", "predict16.cuh")).read()
    assert "predict_mean_kernel" in src
    lib = os.path.join(ROOT, "bayesianoptimization_b200", "libb200bo.so")
    if os.path.exists(lib):  # the built library carries the kernel (its name is in the embedded cubin)
        with open(lib, "rb") as f:
            assert b"predict_mean_kernel" in f.read()


def test_exports():
    import bayesianoptimization_b200 as bo

    assert "recommend" in bo.__all__ and "PosteriorMean" in bo.__all__


def test_recommend_without_a_device_touches_nothing():
    import torch

    if torch.cuda.is_available():
        pytest.skip("checks the no-device error")
    bayes_opt = pytest.importorskip("bayes_opt")
    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import _lib as B

    opt = bayes_opt.BayesianOptimization(f=None, pbounds={"x": (-1, 1), "y": (-1, 1)}, random_state=3,
                                         allow_duplicate_points=True)
    for i in range(4):
        opt.register(params={"x": 0.1 * i, "y": -0.2 * i}, target=float(i))
    state = opt._random_state.get_state(legacy=False)
    gp = opt._gp
    with pytest.raises(B.B200Error, match="no CUDA device"):
        bo.recommend(opt)
    assert opt._gp is gp and not hasattr(gp, "X_train_")
    after = opt._random_state.get_state(legacy=False)
    assert after["state"]["key"].tolist() == state["state"]["key"].tolist() and after["state"]["pos"] == state["state"]["pos"]

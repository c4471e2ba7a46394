"""Constrained noisy expected improvement on the device (DESIGN.md 4.15) against the numpy restatement
tests/cnei_oracle.py: CNEI / LogCNEI values of the 16-warp kernel on both bulk-copy pipes and of the small-batch kernels,
selection order, device-resident and Philox candidates, b200bo_gp_set_fantasy_incumbent with its floor, the reduction
to NEI x constraints with noiseless constraint GPs, the refusals, the reference's BayesianOptimization driven through
enable(), and a production-size ill-conditioned case."""
from __future__ import annotations

import ctypes as C
import types
import warnings

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import ConstantKernel, Matern, WhiteKernel

import cnei_oracle as CO
import nei_oracle as NO

pytestmark = pytest.mark.gpu

# (constant, length scale, WhiteKernel noise) of the target and of two constraint GPs
GPS = [(1.7, 0.35, 0.04), (0.9, 0.5, 0.02), (1.2, 0.45, 0.03)]
# one-sided then two-sided bounds
BOUNDS = [(-np.inf, 0.4), (-0.6, 0.7)]


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _fit(bo, X, y, c, ls, noise, alpha=1e-10):
    k = ConstantKernel(c) * Matern(length_scale=ls, nu=2.5)
    if noise > 0:
        k = k + WhiteKernel(noise)
    gp = bo.B200GaussianProcessRegressor(kernel=k, alpha=alpha, normalize_y=True, optimizer=None)
    return gp.fit(X, y)


def _problem(bo, n, d, J, seed=0, noisy_constraints=True):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    ys = [np.sin(3.0 * X.sum(1)), np.cos(2.0 * X[:, 0]) - 0.3, np.sin(2.0 * X[:, -1] + 1.0) * 0.8]
    gps = []
    for j in range(J + 1):
        c, ls, noise = GPS[j]
        if j > 0 and not noisy_constraints:
            noise = 0.0
        y = ys[j] + np.sqrt(GPS[j][2]) * rs.randn(n)
        gps.append(_fit(bo, X, y, c, ls, noise, alpha=1e-10 if noise > 0 else 1e-6))
    con = types.SimpleNamespace(model=gps[1:], lb=np.array([b[0] for b in BOUNDS[:J]]),
                                ub=np.array([b[1] for b in BOUNDS[:J]]))
    return X, gps, con


def _device_fantasies(bo, gps, con, S, seed, in_bounds=None):
    rs = np.random.RandomState(seed)
    fant = gps[0].noiseless_fantasies(S, random_state=rs)
    cf = [m.noiseless_fantasies(S, random_state=rs) for m in gps[1:]]
    n = gps[0].X_train_.shape[0]
    ok = CO.eligible(np.ones(n, bool) if in_bounds is None else in_bounds, [f.F for f in cf], con.lb, con.ub)
    best = np.empty(S)
    e = np.ascontiguousarray(ok, dtype=np.uint8)
    bo._lib.check(bo._lib.lib().b200bo_gp_set_fantasy_incumbent(fant.handle.ptr, e.ctypes.data_as(
        C.POINTER(C.c_uint8)), bo._lib.as_dp(best)))
    fant.best = best
    return fant, cf, ok


def _restatement(X, gps, con, S, seed, in_bounds=None):
    """Per GP (kc, Kc, tau, y_mean, y_std, F (normalised), A) from the same draws, then best_s by the rule."""
    n = X.shape[0]
    draws = CO.draws(np.random.RandomState(seed), n, S, len(gps) - 1)
    out = []
    for j, (gp, (Z, E)) in enumerate(zip(gps, draws)):
        c, ls, noise = GPS[j]
        kc = ConstantKernel(c) * Matern(length_scale=ls, nu=2.5)
        Kc = kc(X)
        noise = float(gp.kernel_.k2.noise_level) if isinstance(gp.kernel_.k2, WhiteKernel) else 0.0
        s2 = gp.alpha + noise
        tau = min(gp.alpha, 1e-6)
        ym, ys = float(gp._y_train_mean), float(gp._y_train_std)
        F, A, _ = NO.fantasies(Kc, (gp._y_raw - ym) / ys, s2, tau, Z, E, np.ones(n, bool), ym, ys)
        out.append((kc, Kc, tau, ym, ys, F, A))
    Fc = [o[4] * o[5] + o[3] for o in out[1:]]
    ok = CO.eligible(np.ones(n, bool) if in_bounds is None else in_bounds, Fc, con.lb, con.ub)
    best = CO.incumbents(out[0][4] * out[0][5] + out[0][3], ok)
    return out, best, ok


def _want(X, Xc, st, best, con, xi, log):
    (kc, Kc, tau, ym, ys, F, A), cons = st[0], st[1:]
    Ks = kc(Xc, X)
    sd = NO.noiseless_sd(Kc, tau, Ks, kc.k1.constant_value, ys)
    Kcs = [o[0](Xc, X) for o in cons]
    sdc = [NO.noiseless_sd(o[1], o[2], K, o[0].k1.constant_value, o[4]) for o, K in zip(cons, Kcs)]
    return -CO.cnei(Ks, A, best, sd, xi, Kcs, [o[6] for o in cons], sdc, con.lb, con.ub, ym, ys,
                    [o[3] for o in cons], [o[4] for o in cons], log=log)


@pytest.mark.parametrize("kind", ["cnei", "logcnei"])
@pytest.mark.parametrize("pipe", ["bulk", "bulk_nomc"])
@pytest.mark.parametrize("S", [1, 4, 16])
@pytest.mark.parametrize("d", [3, 20])
@pytest.mark.parametrize("J", [1, 2])
def test_values_match_the_restatement(bo, monkeypatch, kind, pipe, S, d, J):
    import torch

    monkeypatch.setenv("B200BO_PREDICT_PIPE", pipe)
    X, gps, con = _problem(bo, 300, d, J)
    fant, cf, ok = _device_fantasies(bo, gps, con, S, seed=3)
    st, best, ok_r = _restatement(X, gps, con, S, seed=3)
    assert np.array_equal(ok, ok_r)
    np.testing.assert_allclose(fant.best, best, rtol=1e-9, atol=1e-9)
    code = bo._lib.ACQ_CNEI if kind == "cnei" else bo._lib.ACQ_LOGCNEI
    xi = 0.01
    acq = bo.FusedAcquisition(code, gps[0], con, xi=xi, fantasies=fant, constraint_fantasies=cf)
    rs = np.random.RandomState(5)
    for m in (1000, 20):  # tiled kernel, small-batch kernels
        Xc = rs.uniform(size=(m, d))
        want = _want(X, Xc, st, fant.best, con, xi, kind == "logcnei")
        got = acq(Xc)
        np.testing.assert_allclose(got, want, rtol=1e-7, atol=1e-10)
        idx, val, top = acq.argmin_topk(Xc, 5)
        order = np.lexsort((np.arange(m), want))
        assert idx == order[0] and np.array_equal(top, order[:5])
        # device-resident candidates (b200bo_acq_eval_dev) give the host path's values bit for bit, on the tiled
        # kernel's bulk pipe and on the small-batch kernels
        Xd = torch.from_numpy(Xc).cuda()
        out = torch.empty(m, dtype=torch.float64, device="cuda")
        spec = acq.spec
        bo._lib.check(bo._lib.lib().b200bo_acq_eval_dev(C.byref(spec), Xd.data_ptr(), m, out.data_ptr(), None, None,
                                                        0, None, 0, None))
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), got)


@pytest.mark.parametrize("kind", ["cnei", "logcnei"])
def test_philox_candidates_match_the_restatement(bo, kind):
    X, gps, con = _problem(bo, 300, 3, 2)
    fant, cf, _ = _device_fantasies(bo, gps, con, 4, seed=2)
    st, best, _ = _restatement(X, gps, con, 4, seed=2)
    code = bo._lib.ACQ_CNEI if kind == "cnei" else bo._lib.ACQ_LOGCNEI
    acq = bo.FusedAcquisition(code, gps[0], con, xi=0.01, fantasies=fant, constraint_fantasies=cf)
    i, v, xb, ti, tx = acq.argmin_topk_philox(77, np.array([[0.0, 1.0]] * 3), 4000, 4)
    want = _want(X, tx, st, fant.best, con, 0.01, kind == "logcnei")
    np.testing.assert_allclose(v, want[0], rtol=1e-7, atol=1e-10)
    assert np.all(np.diff(want) >= -1e-9 * (np.abs(want[:-1]) + 1e-12))
    assert np.array_equal(xb, tx[0])


def test_set_fantasy_incumbent_rule_and_floor(bo):
    X, gps, con = _problem(bo, 200, 3, 1)
    fant = gps[0].noiseless_fantasies(4, random_state=1)
    F = fant.F
    ok = np.zeros(F.shape, bool)
    ok[::3, 0] = True
    ok[5, 2] = True
    ok[:, 3] = True  # sample 1 has no eligible row: the floor
    best = np.empty(4)
    e = np.ascontiguousarray(ok, dtype=np.uint8)
    L = bo._lib.lib()
    bo._lib.check(L.b200bo_gp_set_fantasy_incumbent(fant.handle.ptr, e.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                    bo._lib.as_dp(best)))
    assert np.array_equal(best, CO.incumbents(F, ok))
    assert best[1] == F[:, 1].min() and best[2] == F[5, 2] and best[3] == F[:, 3].max()
    # NEI on the same handle now measures against these incumbents
    acq = bo.FusedAcquisition(bo._lib.ACQ_NEI, gps[0], xi=0.0, fantasies=fant)
    kc = ConstantKernel(GPS[0][0]) * Matern(length_scale=GPS[0][1], nu=2.5)
    Xc = np.random.RandomState(2).uniform(size=(50, 3))
    st, _, _ = _restatement(X, gps[:1], types.SimpleNamespace(lb=[], ub=[]), 4, seed=1)
    _, Kc, tau, ym, ys, _, A = st[0]
    Ks = kc(Xc, X)
    want = -NO.nei(Ks, A, best, NO.noiseless_sd(Kc, tau, Ks, GPS[0][0], ys), 0.0, ym, ys)
    np.testing.assert_allclose(acq(Xc), want, rtol=1e-7, atol=1e-10)
    # refusals: a handle without fantasies, and fantasies conditioned on pending rows
    bare = _fit(bo, X, np.sin(X.sum(1)), 1.0, 0.5, 0.0, alpha=1e-6)
    assert L.b200bo_gp_set_fantasy_incumbent(bare._handle().ptr, e.ctypes.data_as(C.POINTER(C.c_uint8)),
                                             None) == bo._lib.ERR_STATE
    pend = gps[0].noiseless_fantasies(4, random_state=1, pending=X[:1] + 0.01)
    assert L.b200bo_gp_set_fantasy_incumbent(pend.handle.ptr, e.ctypes.data_as(C.POINTER(C.c_uint8)),
                                             None) == bo._lib.ERR_STATE


@pytest.mark.parametrize("log", [False, True])
def test_noiseless_constraints_equal_nei_times_constraints(bo, log):
    X, gps, con = _problem(bo, 400, 4, 2, seed=4, noisy_constraints=False)
    mask = np.ones(400, bool)
    for j, m in enumerate(gps[1:]):
        mask &= (con.lb[j] <= m._y_raw) & (m._y_raw <= con.ub[j])
    assert mask.any() and not mask.all()
    nei_f = gps[0].noiseless_fantasies(8, incumbent=mask, random_state=6)
    nei = bo.FusedAcquisition(bo._lib.ACQ_LOGNEI if log else bo._lib.ACQ_NEI, gps[0], con, xi=0.01, fantasies=nei_f)
    fant, cf, ok = _device_fantasies(bo, gps, con, 8, seed=6)
    assert np.array_equal(ok, np.repeat(mask[:, None], 8, axis=1))
    assert np.array_equal(fant.best, nei_f.best)
    cnei = bo.FusedAcquisition(bo._lib.ACQ_LOGCNEI if log else bo._lib.ACQ_CNEI, gps[0], con, xi=0.01, fantasies=fant,
                               constraint_fantasies=cf)
    Xc = np.random.RandomState(7).uniform(size=(3000, 4))
    a, b = cnei(Xc), nei(Xc)
    # the constraint means come from A_j = K0_j^-1 y_n here and from alpha_ there: equal to solve round-off
    np.testing.assert_allclose(a, b, rtol=1e-8, atol=1e-9 if log else 1e-13)
    ia, _, ta = cnei.argmin_topk(Xc, 8)
    ib, _, tb = nei.argmin_topk(Xc, 8)
    assert ia == ib and np.array_equal(ta, tb)


def test_refusals(bo, monkeypatch):
    X, gps, con = _problem(bo, 300, 3, 2)
    fant, cf, _ = _device_fantasies(bo, gps, con, 2, seed=0)
    acq = bo.FusedAcquisition(bo._lib.ACQ_CNEI, gps[0], con, fantasies=fant, constraint_fantasies=cf)
    Xc = np.random.RandomState(1).uniform(size=(5000, 3))
    for env, val in (("B200BO_PREDICT_WARPS", "8"), ("B200BO_PREDICT_IMPL", "dfma"), ("B200BO_PREDICT_IMPL", "tf32"),
                     ("B200BO_PREDICT_PIPE", "cpasync"), ("B200BO_PREDICT_MMA", "884")):
        with monkeypatch.context() as mp:
            mp.setenv(env, val)
            with pytest.raises(NotImplementedError):
                acq(Xc)
    assert np.all(np.isfinite(acq(Xc)))
    L, spec = bo._lib.lib(), acq.spec
    mu = np.empty(10)
    xs = np.ascontiguousarray(Xc[:10])
    out = np.empty(10)
    assert L.b200bo_acq_eval_dev(C.byref(spec), None, 0, None, bo._lib.as_dp(mu), None, 0, None, 0, None) == \
        bo._lib.ERR_ARG
    # mismatched S, a handle without fantasies
    cf_s = [gps[1].noiseless_fantasies(3, random_state=0), cf[1]]
    bad = bo.FusedAcquisition(bo._lib.ACQ_CNEI, gps[0], con, fantasies=fant, constraint_fantasies=cf_s)
    assert L.b200bo_acq_eval(C.byref(bad.spec), bo._lib.as_dp(xs), 10, bo._lib.as_dp(out)) == bo._lib.ERR_ARG
    fresh = _fit(bo, X, np.cos(X.sum(1)), 1.0, 0.5, 0.0, alpha=1e-6)
    sp = bad.spec
    sp.gps[1] = fresh._handle().ptr.value
    assert L.b200bo_acq_eval(C.byref(sp), bo._lib.as_dp(xs), 10, bo._lib.as_dp(out)) == bo._lib.ERR_STATE
    # mismatched n
    Xs = X[:200]
    small = _fit(bo, Xs, np.cos(Xs.sum(1)), 1.0, 0.5, 0.0, alpha=1e-6)
    small_f = small.noiseless_fantasies(2, random_state=0)
    bad_n = bo.FusedAcquisition(bo._lib.ACQ_CNEI, gps[0], con, fantasies=fant, constraint_fantasies=[small_f, cf[1]])
    assert L.b200bo_acq_eval(C.byref(bad_n.spec), bo._lib.as_dp(xs), 10, bo._lib.as_dp(out)) == bo._lib.ERR_ARG
    with pytest.raises(ValueError):
        bo.FusedAcquisition(bo._lib.ACQ_CNEI, gps[0], con, fantasies=fant, constraint_fantasies=cf[:1])


def _noisy_opt(bo, ref, acq, constraint, seed=1):
    rs = np.random.RandomState(seed)

    def f(x, y):
        return -(x - 0.3) ** 2 - (y + 0.2) ** 2 + 0.05 * rs.randn()

    opt = ref.BayesianOptimization(f=f, pbounds={"x": (-1, 1), "y": (-1, 1)}, acquisition_function=acq,
                                   constraint=constraint, random_state=seed, verbose=0)
    opt.set_gp_params(alpha=2e-3)
    bo.enable(opt, refine="analytic")  # the refinement on CNEI's device gradient
    for m in opt.constraint.model:  # noisy constraint GPs
        m.set_params(kernel=Matern(nu=2.5) + WhiteKernel(1e-3))
    return opt


@pytest.mark.parametrize("cls", ["ConstrainedNoisyExpectedImprovement", "LogConstrainedNoisyExpectedImprovement"])
def test_bayesian_optimization_with_noisy_constraints(bo, ref, cls, tmp_path):
    from scipy.optimize import NonlinearConstraint

    rs = np.random.RandomState(3)
    con = NonlinearConstraint(lambda x, y: x + y + 0.05 * rs.randn(), -np.inf, 0.5)
    acq = getattr(bo, cls)(xi=0.0, n_samples=4)
    opt = _noisy_opt(bo, ref, acq, con)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt.maximize(init_points=5, n_iter=3)
    assert len(opt.space) == 8 and acq.fantasies is not None and len(acq.constraint_fantasies) == 1
    path = tmp_path / "state.json"
    opt.save_state(str(path))
    acq2 = getattr(bo, cls)(xi=0.5, n_samples=2, jitter=1e-3)
    opt2 = _noisy_opt(bo, ref, acq2, con)
    opt2.load_state(str(path))
    assert (acq2.n_samples, acq2.jitter, acq2.xi) == (4, 1e-6, 0.0)


def test_suggests_without_a_feasible_point_where_nei_cannot(bo, ref):
    from bayes_opt.exception import NoValidPointRegisteredError
    from scipy.optimize import NonlinearConstraint

    never = NonlinearConstraint(lambda x, y: x + y, 5.0, 6.0)
    opt = _noisy_opt(bo, ref, bo.NoisyExpectedImprovement(xi=0.0, n_samples=2), never)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(NoValidPointRegisteredError):
            opt.maximize(init_points=3, n_iter=1)
    acq = bo.ConstrainedNoisyExpectedImprovement(xi=0.0, n_samples=4)
    opt = _noisy_opt(bo, ref, acq, never)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt.maximize(init_points=3, n_iter=2)
    assert len(opt.space) == 5
    # every sample fell back to the floor: the smallest target fantasy
    assert np.array_equal(acq.fantasies.best, acq.fantasies.F.min(axis=0))


def test_int_space_with_a_noisy_constraint(bo, ref):
    """A mixed-integer space: the noisy constraint kernel keeps the reference's wrap_kernel transform."""
    from bayes_opt.parameter import wrap_kernel
    from scipy.optimize import NonlinearConstraint

    def f(x, k):
        return -(x - 0.2) ** 2 - 0.1 * (k - 2) ** 2

    con = NonlinearConstraint(lambda x, k: x + 0.1 * k, -np.inf, 0.6)
    acq = bo.LogConstrainedNoisyExpectedImprovement(xi=0.0, n_samples=3)
    opt = ref.BayesianOptimization(f=f, pbounds={"x": (-1.0, 1.0), "k": (0, 5, int)}, acquisition_function=acq,
                                   constraint=con, random_state=3, verbose=0)
    opt.set_gp_params(alpha=1e-3)
    bo.enable(opt)
    for m in opt.constraint.model:
        m.set_params(kernel=wrap_kernel(Matern(nu=2.5) + WhiteKernel(1e-3), opt._space.kernel_transform))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt.maximize(init_points=4, n_iter=2)
    assert len(opt.space) == 6


def test_production_size_ill_conditioned(bo):
    """N = 2048, d = 16, J = 2, S = 16, clustered inputs (cond(K0) >~ 1e8): values at 4096 candidates and at 1e-7
    neighbours of registered rows against the fp64 restatement.  LogCNEI: within 1e-6 relative.  CNEI: within 1e-6 of
    |want| + 1e-3 max|want| - a candidate whose value is tiny next to the largest (far in a constraint's tail) is held
    to an absolute floor, since its P_js amplify the round-off of the constraint means; the pure relative error over
    the values above 1e-3 max|want| is reported as well."""
    rs = np.random.RandomState(11)
    n, d, S = 2048, 16, 16
    centers = rs.uniform(size=(64, d))
    X = centers[rs.randint(0, 64, n)] + 0.02 * rs.standard_normal((n, d))
    ys = [np.sin(X.sum(1)), np.cos(X[:, 0] + X[:, 1]), np.sin(2.0 * X[:, 2])]
    gps = []
    for j in range(3):
        c, ls, noise = GPS[j]
        gps.append(_fit(bo, X, ys[j] + np.sqrt(noise) * rs.randn(n), c, 2.0, noise, alpha=1e-6))
    GPS_LS = 2.0
    con = types.SimpleNamespace(model=gps[1:], lb=np.array([b[0] for b in BOUNDS]), ub=np.array([b[1] for b in BOUNDS]))
    fant, cf, ok = _device_fantasies(bo, gps, con, S, seed=9)
    draws = CO.draws(np.random.RandomState(9), n, S, 2)
    st = []
    for j, (gp, (Z, E)) in enumerate(zip(gps, draws)):
        kc = ConstantKernel(GPS[j][0]) * Matern(length_scale=GPS_LS, nu=2.5)
        Kc = kc(X)
        ym, ysd = float(gp._y_train_mean), float(gp._y_train_std)
        F, A, _ = NO.fantasies(Kc, (gp._y_raw - ym) / ysd, gp.alpha + GPS[j][2], min(gp.alpha, 1e-6), Z, E,
                               np.ones(n, bool), ym, ysd)
        st.append((kc, Kc, min(gp.alpha, 1e-6), ym, ysd, F, A))
    assert np.linalg.cond(st[0][1] + st[0][2] * np.eye(n)) > 1e8
    Xc = np.vstack([rs.uniform(size=(4096, d)) * 0.9 + 0.05, X[:64] + 1e-7])
    worst = 0.0
    for kind, log in ((bo._lib.ACQ_CNEI, False), (bo._lib.ACQ_LOGCNEI, True)):
        acq = bo.FusedAcquisition(kind, gps[0], con, xi=0.0, fantasies=fant, constraint_fantasies=cf)
        want = _want(X, Xc, st, fant.best, con, 0.0, log)
        got = acq(Xc)
        big = np.max(np.abs(want))
        scale = np.abs(want) + (big * 1e-3 if not log else 0.0)
        err = np.max(np.abs(got - want) / scale)
        worst = max(worst, err)
        sel = np.abs(want) >= 1e-3 * big
        pure = np.max(np.abs(got - want)[sel] / np.abs(want[sel]))
        print(f"production size, {'LogCNEI' if log else 'CNEI'}: largest error {err:.2e} (pure relative over "
              f"|want| >= 1e-3 max|want|: {pure:.2e})")
    assert worst < 1e-6


def _cd5(f, rows, h):
    """Fourth-order central differences of f at rows, one column per input dimension."""
    cols = []
    for e in np.eye(rows.shape[1]):
        cols.append((8 * (f(rows + h * e) - f(rows - h * e)) - (f(rows + 2 * h * e) - f(rows - 2 * h * e))) / (12 * h))
    return np.stack(cols, axis=1)


@pytest.mark.parametrize("kind", ["cnei", "logcnei"])
@pytest.mark.parametrize("S", [1, 4, 16])
def test_gradient_matches_central_differences(bo, kind, S):
    """b200bo_acq_value_grad of CNEI / LogCNEI with two constraints: the value equals the restatement and the
    evaluation path's value, the gradient five-point central differences of the value in refine_mode()."""
    X, gps, con = _problem(bo, 300, 3, 2)
    fant, cf, _ = _device_fantasies(bo, gps, con, S, seed=8)
    st, _, _ = _restatement(X, gps, con, S, seed=8)
    code = bo._lib.ACQ_CNEI if kind == "cnei" else bo._lib.ACQ_LOGCNEI
    acq = bo.FusedAcquisition(code, gps[0], con, xi=0.01, fantasies=fant, constraint_fantasies=cf)
    rows = np.random.RandomState(6).uniform(0.05, 0.95, size=(12, 3))
    val, grad = acq.value_and_grad(rows)
    np.testing.assert_allclose(val, _want(X, rows, st, fant.best, con, 0.01, kind == "logcnei"), rtol=1e-7,
                               atol=1e-10)
    with acq.refine_mode():
        np.testing.assert_allclose(val, acq(rows), rtol=1e-12, atol=1e-15)
        cd = _cd5(acq, rows, 1e-5)
    assert np.all(np.isfinite(grad))
    np.testing.assert_allclose(grad, cd, rtol=2e-5, atol=1e-6 * (1.0 + np.abs(cd).max()))


def test_closure_eligibility_uses_the_bounds_and_draws_in_order(bo, ref):
    """The class's own closure: a registered row outside the bounds is never an incumbent, the incumbents follow the
    rule over the constraint fantasies, and the RandomState is left where Z, E, Z_1, E_1, Z_2, E_2 leave it."""
    X, gps, con = _problem(bo, 200, 3, 2)
    outside = np.zeros(200, bool)
    outside[:20] = True
    params = X.copy()
    params[outside, 0] = 1.5  # outside the bounds [0, 1] of dimension 0 (the GPs keep their own inputs)
    space = types.SimpleNamespace(params=params, bounds=np.array([[0.0, 1.0]] * 3))
    acq = bo.ConstrainedNoisyExpectedImprovement(xi=0.0, n_samples=4)
    rs = np.random.RandomState(21)
    acq._path_rng, acq._suggest_space = rs, space
    closure = acq._get_acq(gps[0], con)
    st, best, ok = _restatement(X, gps, con, 4, seed=21, in_bounds=~outside)
    assert not ok[outside].any()
    np.testing.assert_allclose(acq.fantasies.best, best, rtol=1e-9, atol=1e-9)
    rs2 = np.random.RandomState(21)
    CO.draws(rs2, 200, 4, 2)
    assert rs.randint(1 << 30) == rs2.randint(1 << 30)
    Xc = np.random.RandomState(22).uniform(size=(50, 3))
    np.testing.assert_allclose(closure(Xc), _want(X, Xc, st, best, con, 0.0, False), rtol=1e-7, atol=1e-10)

"""Constrained NEI with pending points without a GPU: the restatement tests/cnei_batch_oracle.py against independent forms
(the full Cholesky factor of X u P, a brute-force Monte-Carlo of E[1{c(x) feasible} (f(x) - best(X u P))+] from the joint
covariances), its identities, the class's draw order and its refusals before any draw, and the new export."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest
from scipy.linalg import cho_factor, cho_solve, cholesky
from sklearn.gaussian_process.kernels import ConstantKernel, Matern

import cnei_batch_oracle as CB
import cnei_oracle as CO
import nei_batch_oracle as NB
import nei_oracle as NO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAU = 1e-6
BOX = np.array([[0.0, 1.0], [0.0, 1.0]])


def _gps(X, rs, J=2, s2=(0.05, 0.04, 0.03), ym=(0.0, 0.0, 0.0), ys=(1.0, 1.0, 1.0)):
    """Target and J constraint GPs as dicts (cnei_batch_oracle.grown's layout)."""
    fs = [np.sin(3 * X.sum(1)), np.cos(2 * X[:, 0]) - 0.2, np.sin(2 * X[:, 1] + 1.0) * 0.8]
    out = []
    for g in range(J + 1):
        kc = ConstantKernel(1.3 - 0.2 * g) * Matern(length_scale=0.4 + 0.1 * g, nu=2.5)
        y = fs[g] + np.sqrt(max(s2[g], 1e-4)) * rs.randn(X.shape[0])
        out.append({"kc": kc, "y_n": (y - ym[g]) / ys[g], "s2": s2[g], "tau": TAU, "y_mean": ym[g], "y_std": ys[g]})
    return out


def _problem(n=12, p=3, J=2, seed=0, **kw):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, 2))
    P = rs.uniform(size=(p, 2))
    return X, P, _gps(X, rs, J, **kw)


LB, UB = np.array([-np.inf, -0.6]), np.array([0.3, 0.7])


def test_restatement_equals_the_full_factor_form():
    """Every GP's F' over X u P from the Cholesky factor of X u P at once; best' by the definition, row by row."""
    X, P, gps = _problem(p=4)
    n, p, S = X.shape[0], P.shape[0], 5
    inb = np.ones(n + p, bool)
    inb[[2, n + 1]] = False  # a registered and a pending row outside the bounds
    out, best, ok, d = CB.pipeline(gps, X, P, np.random.RandomState(1), S, 0, inb, LB, UB)
    Xa = np.vstack([X, P])
    for g, (Fd, A), (Z, E, Zp) in zip(gps, out, d):
        L = cholesky(g["kc"](Xa) + TAU * np.eye(n + p), lower=True)
        W = NB.residual_solve(g["kc"](X), g["y_n"], g["s2"], TAU, Z, E)
        F, _, _ = NO.fantasies(g["kc"](X), g["y_n"], g["s2"], TAU, Z, E, np.ones(n, bool))
        want = np.vstack([F, (L @ np.vstack([Z, Zp]))[n:] + g["kc"](P, X) @ W])
        np.testing.assert_allclose(Fd, g["y_std"] * want + g["y_mean"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(A, cho_solve(cho_factor(g["kc"](Xa) + TAU * np.eye(n + p), lower=True), want),
                                   atol=1e-9)
    for s in range(S):
        elig = [i for i in range(n + p) if inb[i] and all(LB[j] <= out[1 + j][0][i, s] <= UB[j] for j in range(2))]
        assert np.array_equal(ok[:, s], np.isin(np.arange(n + p), elig))
        want = max(out[0][0][i, s] for i in elig) if elig else out[0][0][:, s].min()
        assert best[s] == want
    assert not ok[[2, n + 1]].any()


@pytest.mark.parametrize("log", [False, True])
def test_cnei_matches_a_brute_force_monte_carlo(log):
    """CNEI on the grown noiseless GPs against E[prod_j 1{lb_j <= c_j(x) <= ub_j} (f(x) - best(X u P))+], best the
    largest g_tau over the in-bounds rows of X u P that the draws of g_tau,j call feasible, or the smallest over all rows
    when none is: every GP drawn directly from the joint posterior of (g_tau(X u P), g(x)) given its data, no Matheron
    step, the GPs independent."""
    X, P, gps = _problem(n=10, p=2, J=2, seed=4)
    n, p, S = X.shape[0], P.shape[0], 200_000
    inb = np.ones(n + p, bool)
    inb[3] = False
    lb, ub = np.array([-np.inf, -0.3]), np.array([0.5, 0.9])
    xc = np.array([[0.3, 0.6], [0.8, 0.2]])
    out, best, _, _ = CB.pipeline(gps, X, P, np.random.RandomState(5), S, 0, inb, lb, ub)
    Xa = np.vstack([X, P])
    got = CB.cnei(gps, Xa, [o[1] for o in out], best, xc, 0.0, lb, ub, log=log)
    assert np.all(np.isfinite(got))
    rs = np.random.RandomState(6)
    for i, x in enumerate(xc):
        T = np.vstack([Xa, x[None]])
        G = []
        for g in gps:
            Kf = cho_factor(g["kc"](X) + g["s2"] * np.eye(n), lower=True)
            prior = g["kc"](T) + np.diag(np.r_[np.full(n + p, TAU), 0.0])
            cross = g["kc"](T, X)
            m = cross @ cho_solve(Kf, g["y_n"])
            Cv = prior - cross @ cho_solve(Kf, cross.T)
            w, V = np.linalg.eigh(Cv)
            G.append(g["y_std"] * (m + (rs.standard_normal((S, len(m))) * np.sqrt(np.maximum(w, 0.0))) @ V.T)
                     + g["y_mean"])
        feas_rows = inb[None, :] & np.all([(lb[j] <= G[1 + j][:, :-1]) & (G[1 + j][:, :-1] <= ub[j])
                                           for j in range(2)], axis=0)
        inc = np.where(feas_rows.any(axis=1), np.where(feas_rows, G[0][:, :-1], -np.inf).max(axis=1),
                       G[0][:, :-1].min(axis=1))
        feas_x = np.all([(lb[j] <= G[1 + j][:, -1]) & (G[1 + j][:, -1] <= ub[j]) for j in range(2)], axis=0)
        imp = feas_x * np.maximum(G[0][:, -1] - inc, 0.0)
        want, se = imp.mean(), imp.std() / np.sqrt(S)
        val = np.exp(got[i]) if log else got[i]
        # two independent Monte-Carlo estimates: their difference within 4 combined standard errors
        assert abs(val - want) <= 4 * np.sqrt(2.0) * se, (i, val, want, se)


def test_no_pending_rows_is_cnei():
    """p = 0: the same draws, F, A, incumbents and values as tests/cnei_oracle.py's pipeline."""
    X, P, gps = _problem()
    n, S = X.shape[0], 4
    out, best, ok, _ = CB.pipeline(gps, X, P[:0], np.random.RandomState(2), S, 0, np.ones(n, bool), LB, UB)
    draws = CO.draws(np.random.RandomState(2), n, S, 2)
    Fs = []
    for g, (Z, E), (Fd, A) in zip(gps, draws, out):
        F, A0, _ = NO.fantasies(g["kc"](X), g["y_n"], g["s2"], TAU, Z, E, np.ones(n, bool))
        assert np.array_equal(Fd, F)
        np.testing.assert_allclose(A, A0, rtol=1e-12, atol=1e-12)
        Fs.append(F)
    ok0 = CO.eligible(np.ones(n, bool), Fs[1:], LB, UB)
    assert np.array_equal(ok, ok0) and np.array_equal(best, CO.incumbents(Fs[0], ok0))


def test_no_constraint_and_unbounded_constraints_are_pending_nei():
    """J = 0, and constraints with bounds (-inf, inf) with every row in bounds: best' is PendingNEI's bit for bit (the
    largest fantasy over X u P), and the values are NEI's on the grown GP."""
    X, P, gps = _problem(p=3)
    n, p, S = X.shape[0], P.shape[0], 4
    Xa = np.vstack([X, P])
    xc = np.random.RandomState(9).uniform(size=(40, 2))
    g0 = gps[0]
    Z, E, Zp = NB.draws(np.random.RandomState(3), n, S, p)
    Fa, A, best_nei = NB.pending_fantasies(g0["kc"], X, P, g0["y_n"], g0["s2"], TAU, Z, E, Zp, np.ones(n, bool))
    out, best, _, _ = CB.pipeline(gps[:1], X, P, np.random.RandomState(3), S, 0, np.ones(n + p, bool), [], [])
    assert np.array_equal(best, best_nei)
    inf = np.full(2, np.inf)
    out2, best2, ok2, _ = CB.pipeline(gps, X, P, np.random.RandomState(3), S, 0, np.ones(n + p, bool), -inf, inf)
    assert ok2.all() and np.array_equal(best2, best_nei)
    for log in (False, True):
        want = NB.nei(g0["kc"], Xa, A, best_nei, TAU, xc, 0.01, log=log)
        np.testing.assert_array_equal(CB.cnei(gps[:1], Xa, [out[0][1]], best, xc, 0.01, [], [], log=log), want)
        got = CB.cnei(gps, Xa, [o[1] for o in out2], best2, xc, 0.01, -inf, inf, log=log)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-15)


def test_noiseless_constraints_observe_registered_rows_and_draw_pending_ones():
    """sigma_n^2 = tau on the constraint GPs: their registered fantasies are the observations in every sample, the pending
    ones are draws that differ across the samples."""
    X, P, gps = _problem(p=3, s2=(0.05, TAU, TAU))
    n, S = X.shape[0], 6
    out, _, _, _ = CB.pipeline(gps, X, P, np.random.RandomState(8), S, 0, np.ones(n + 3, bool), LB, UB)
    for j in (1, 2):
        F = out[j][0]
        assert np.array_equal(F[:n], np.repeat(gps[j]["y_n"][:, None], S, axis=1))
        assert np.all(np.std(F[n:], axis=1) > 1e-4)


def test_draw_order_per_gp_then_the_candidates():
    rs = np.random.RandomState(7)
    d = CB.draws(rs, 5, 3, 2, 4)
    rs2 = np.random.RandomState(7)
    for Z, E, Zp in d:
        assert np.array_equal(Z, rs2.standard_normal((5, 3)))
        assert np.array_equal(E, rs2.standard_normal((5, 3)))
        assert np.array_equal(Zp, rs2.standard_normal((4, 3)))
    assert rs.randint(1 << 30) == rs2.randint(1 << 30)
    # p = 0 and q = 1: no z rows, cnei_oracle's stream
    rs, rs2 = np.random.RandomState(7), np.random.RandomState(7)
    CB.draws(rs, 5, 3, 2, 0)
    CO.draws(rs2, 5, 3, 2)
    assert rs.randint(1 << 30) == rs2.randint(1 << 30)


class _Recorder:
    """Stands in for a device GP: noiseless_fantasies consumes the stream as the real one does and records its call."""

    def __init__(self, log, name, n):
        self.log, self.name, self.n = log, name, n
        self.__dict__["_b200_device_fitted"] = True

    def device_list(self):
        return [0]

    def _ensure_device_fit(self):
        pass

    def noiseless_fantasies(self, S, jitter, random_state=None, pending=None, extra_rows=0):
        rows = (0 if pending is None else len(pending)) + extra_rows
        self.log.append((self.name, 0 if pending is None else len(pending), extra_rows))
        random_state.standard_normal((self.n, S))
        random_state.standard_normal((self.n, S))
        if rows:
            random_state.standard_normal((rows, S))
        return self.name


def test_class_draws_target_then_each_constraint(monkeypatch, ref):
    """The closure's calls of noiseless_fantasies: the target first, then each constraint in constraint.model order, each
    with the pending rows and q - 1 extra rows; the stream ends where cnei_batch_oracle.draws leaves it."""
    import types

    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import acquisition as A

    log, n, S = [], 6, 3
    gp = _Recorder(log, "target", n)
    con = types.SimpleNamespace(model=[_Recorder(log, f"c{j}", n) for j in range(2)], lb=LB, ub=UB)
    monkeypatch.setattr(A, "_as_b200_gp", lambda g: g)
    monkeypatch.setattr(A._ConstrainedNoisyEI, "_set_incumbent", lambda self: None)
    monkeypatch.setattr(A, "FusedAcquisition", lambda *a, **k: "closure")
    space = types.SimpleNamespace(params=np.random.RandomState(0).uniform(size=(n, 2)), bounds=BOX)
    acq = bo.LogConstrainedNoisyExpectedImprovement(n_samples=S)
    rs = np.random.RandomState(4)
    acq._path_rng = rs
    P = np.array([[0.2, 0.3], [1.5, 0.1]])
    assert acq._closure(gp, con, space, pending=P, extra_rows=3) == "closure"
    assert log == [("target", 2, 3), ("c0", 2, 3), ("c1", 2, 3)]
    assert np.array_equal(acq._in_bounds_mask, np.r_[np.ones(n, bool), True, False])
    rs2 = np.random.RandomState(4)
    CB.draws(rs2, n, S, 2, 5)
    assert rs.randint(1 << 30) == rs2.randint(1 << 30)
    assert acq._extender(con) == acq.condition_on_pending
    log.clear()
    acq._closure(gp, con, space)  # no pending rows, q = 1: no z rows
    assert log == [("target", 0, 0), ("c0", 0, 0), ("c1", 0, 0)]


def _gp_on_host(bo, devices=None, xform="device"):
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), devices=devices)
    gp.X_train_ = np.zeros((3, 2))
    gp.__dict__["_b200_device_fitted"] = True
    gp.__dict__["_b200_xform"] = (xform, None)
    return gp


@pytest.mark.parametrize("what", ["too_many", "multi_device_target", "multi_device_constraint", "host_xform"])
def test_refusals_before_any_draw(ref, what):
    import types

    import bayesianoptimization_b200 as bo

    J = 8 if what == "too_many" else 2
    models = [_gp_on_host(bo) for _ in range(J)]
    gp = _gp_on_host(bo, devices=[0, 1] if what == "multi_device_target" else None)
    if what == "multi_device_constraint":
        models[1] = _gp_on_host(bo, devices=[0, 1])
    if what == "host_xform":
        models[1] = _gp_on_host(bo, xform="host")
    con = types.SimpleNamespace(model=models, lb=np.full(J, -np.inf), ub=np.zeros(J))
    space = types.SimpleNamespace(params=np.zeros((3, 2)), bounds=BOX)
    acq = bo.ConstrainedNoisyExpectedImprovement(n_samples=2)
    rs = np.random.RandomState(0)
    acq._path_rng, acq._suggest_space = rs, space
    with pytest.raises(NotImplementedError):
        acq._closure(gp, con, space, pending=np.full((1, 2), 0.5), extra_rows=1)
    assert np.array_equal(rs.get_state()[1], np.random.RandomState(0).get_state()[1])


def test_pending_nei_accepts_constraints_with_a_cnei_base_only(ref):
    from bayes_opt.constraint import ConstraintModel
    from bayes_opt.exception import ConstraintNotSupportedError
    from bayes_opt.target_space import TargetSpace

    import bayesianoptimization_b200 as bo

    pb = {"a": (0.0, 1.0), "b": (0.0, 1.0)}
    space = TargetSpace(None, pb, constraint=ConstraintModel(lambda a, b: a - b, -np.inf, 0.0))
    space.register(np.array([0.2, 0.4]), 1.0, constraint_value=-0.2)
    for cls in (bo.ConstrainedNoisyExpectedImprovement, bo.LogConstrainedNoisyExpectedImprovement):
        assert bo.PendingNEI(cls(n_samples=2))._serves_constraints()
    for cls in (bo.NoisyExpectedImprovement, bo.LogNoisyExpectedImprovement):
        acq = bo.PendingNEI(cls(n_samples=2))
        assert not acq._serves_constraints()
        with pytest.raises(ConstraintNotSupportedError):
            acq.suggest_batch(None, space, 2)
    with pytest.raises(TypeError):
        bo.KrigingBeliever(bo.ConstrainedNoisyExpectedImprovement())


def test_new_export():
    from bayesianoptimization_b200 import _lib as B

    assert "b200bo_gp_set_constrained_incumbent" in B.EXPORTS
    with open(os.path.join(ROOT, "include", "b200bo.h")) as f:
        h = f.read()
    assert "int b200bo_gp_set_constrained_incumbent(b200bo_gp* target, b200bo_gp* const* constraints" in h
    if not os.path.exists(B.LIB_PATH):
        pytest.skip("library not built")
    assert hasattr(C.CDLL(B.LIB_PATH), "b200bo_gp_set_constrained_incumbent")

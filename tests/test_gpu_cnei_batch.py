"""Constrained NEI with pending points and batches on the device (DESIGN.md 4.16) against the numpy restatement
tests/cnei_batch_oracle.py: b200bo_gp_set_constrained_incumbent bit for bit against the host rule, CNEI / LogCNEI values
and selection on the grown handles (both bulk-copy pipes, the small-batch kernels, device and Philox candidates),
row-by-row against one-call extension, gradients, PendingNEI's q = 1 identity, a restated q = 4 batch, the fitted GPs
left unchanged, a live asynchronous BayesianOptimization loop, the refusals and a production-size case."""
from __future__ import annotations

import ctypes as C
import types
import warnings

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import ConstantKernel, Matern, Sum, WhiteKernel

import cnei_batch_oracle as CB
import cnei_oracle as CO

pytestmark = pytest.mark.gpu

# (constant, length scale, WhiteKernel noise) of the target and of two constraint GPs
GPS = [(1.7, 0.35, 0.04), (0.9, 0.5, 0.02), (1.2, 0.45, 0.03)]
BOUNDS = [(-np.inf, 0.4), (-0.6, 0.7)]


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


def _fit(bo, X, y, c, ls, noise, alpha=1e-10):
    k = ConstantKernel(c) * Matern(length_scale=ls, nu=2.5)
    if noise > 0:
        k = k + WhiteKernel(noise)
    gp = bo.B200GaussianProcessRegressor(kernel=k, alpha=alpha, normalize_y=True, optimizer=None)
    return gp.fit(X, y)


def _problem(bo, n, d, J, seed=0, p=3, ls=None, X=None, alpha=1e-10):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d)) if X is None else X
    ys = [np.sin(3.0 * X.sum(1)), np.cos(2.0 * X[:, 0]) - 0.3, np.sin(2.0 * X[:, -1] + 1.0) * 0.8]
    gps = [_fit(bo, X, ys[j] + np.sqrt(GPS[j][2]) * rs.randn(n), GPS[j][0], ls or GPS[j][1], GPS[j][2], alpha)
           for j in range(J + 1)]
    con = types.SimpleNamespace(model=gps[1:], lb=np.array([b[0] for b in BOUNDS[:J]]),
                                ub=np.array([b[1] for b in BOUNDS[:J]]))
    P = rs.uniform(size=(p, d))
    P[0] = X[7] + 1e-3  # near a training row
    return X, gps, con, P


def _as_dict(gp):
    """A fitted device GP in cnei_batch_oracle's layout."""
    k = gp.kernel_
    kc, noise = (k.k1, float(k.k2.noise_level)) if isinstance(k, Sum) and isinstance(k.k2, WhiteKernel) else (k, 0.0)
    ym, ys = float(gp._y_train_mean), float(gp._y_train_std)
    return {"kc": kc, "y_n": (gp._y_raw - ym) / ys, "s2": float(gp.alpha) + noise, "tau": min(float(gp.alpha), 1e-6),
            "y_mean": ym, "y_std": ys}


def _closure(bo, gps, con, X, P, S, seed, box=None, extra=0, log=False):
    """The class's own closure over the pending rows P (its draws, the grown handles, the device incumbents)."""
    cls = bo.LogConstrainedNoisyExpectedImprovement if log else bo.ConstrainedNoisyExpectedImprovement
    acq = cls(xi=0.01, n_samples=S)
    space = types.SimpleNamespace(params=X, bounds=np.array([[0.0, 1.0]] * X.shape[1]) if box is None else box)
    acq._path_rng, acq._suggest_space = np.random.RandomState(seed), space
    closure = acq._closure(gps[0], con, space, pending=P, extra_rows=extra)
    return acq, closure, space


def _entry(bo, fant, cfant, lb, ub, inb):
    L = bo._lib
    handles = (C.c_void_p * max(len(cfant), 1))(*[f.handle.ptr.value for f in cfant])
    best = np.empty(fant.n_samples)
    m = np.ascontiguousarray(inb, dtype=np.uint8)
    rc = L.lib().b200bo_gp_set_constrained_incumbent(fant.handle.ptr, handles, len(cfant), L.as_dp(L.c_f64(lb)),
                                                     L.as_dp(L.c_f64(ub)), m.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                     L.as_dp(best))
    return rc, best


# ---- the incumbent entry ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0, 4])
def test_incumbent_entry_is_the_host_rule_bit_for_bit(bo, p):
    """best_s from the device equals the rule on the host copies of F (NoiselessFantasies.F), bit for bit, with a
    registered and a pending row outside the bounds and a constraint fantasy exactly on a bound; unconditioned, it
    also equals b200bo_gp_set_fantasy_incumbent(cnei_eligible(...))."""
    from bayesianoptimization_b200.acquisition import cnei_eligible

    X, gps, con, P = _problem(bo, 300, 3, 2, p=max(p, 1))
    n, S = X.shape[0], 8
    rs = np.random.RandomState(4)
    kw = {"pending": P[:p]} if p else {}
    fants = [g.noiseless_fantasies(S, random_state=rs, **kw) for g in gps]
    fant, cf = fants[0], fants[1:]
    inb = np.ones(n + p, bool)
    inb[[5, n + p - 1]] = False
    lb, ub = con.lb.copy(), con.ub.copy()
    r = n + p - 2
    s = int(np.argmin(np.abs(cf[1].F[r])))
    lb[1], ub[1] = cf[1].F[r, s], max(ub[1], cf[1].F[r, s] + 1.0)  # exactly on the lower bound: feasible there
    ok = CO.eligible(inb, [f.F for f in cf], lb, ub)
    assert ok[r, s] == (cf[0].F[r, s] <= ub[0])
    rc, best = _entry(bo, fant, cf, lb, ub, inb)
    assert rc == bo._lib.OK
    assert np.array_equal(best, CO.incumbents(fant.F, ok))
    # NEI on the target handle now measures against these incumbents: the handle's device copy is best
    acq = bo.FusedAcquisition(bo._lib.ACQ_CNEI, gps[0], con, xi=0.0, fantasies=fant, constraint_fantasies=cf)
    assert np.all(np.isfinite(acq(np.random.RandomState(1).uniform(size=(30, 3)))))
    if p == 0:
        e = np.ascontiguousarray(cnei_eligible(inb, [f.F for f in cf], lb, ub), dtype=np.uint8)
        host = np.empty(S)
        bo._lib.check(bo._lib.lib().b200bo_gp_set_fantasy_incumbent(fant.handle.ptr, e.ctypes.data_as(
            C.POINTER(C.c_uint8)), bo._lib.as_dp(host)))
        assert np.array_equal(best, host)
    # every sample falls to the floor when nothing is in bounds
    rc, floor = _entry(bo, fant, cf, lb, ub, np.zeros(n + p, bool))
    assert rc == bo._lib.OK and np.array_equal(floor, fant.F.min(axis=0))


def test_incumbent_entry_errors(bo):
    X, gps, con, P = _problem(bo, 200, 3, 2)
    rs = np.random.RandomState(0)
    fants = [g.noiseless_fantasies(4, random_state=rs) for g in gps]
    n = X.shape[0]
    inb = np.ones(n, bool)
    L = bo._lib
    assert _entry(bo, fants[0], fants[1:], con.lb, con.ub, inb)[0] == L.OK
    assert _entry(bo, fants[0], fants[1:], con.ub, con.ub, inb)[0] == L.ERR_ARG  # lb >= ub
    assert _entry(bo, fants[0], fants[1:] * 4, np.full(8, -1.0), np.full(8, 1.0), inb)[0] == L.ERR_ARG  # 8
    other = gps[1].noiseless_fantasies(3, random_state=1)  # another S
    assert _entry(bo, fants[0], [other, fants[2]], con.lb, con.ub, inb)[0] == L.ERR_ARG
    grown = gps[1].noiseless_fantasies(4, random_state=1, pending=P[:1])  # another n
    assert _entry(bo, fants[0], [grown, fants[2]], con.lb, con.ub, inb)[0] == L.ERR_ARG
    bare = _fit(bo, X, np.cos(X.sum(1)), 1.0, 0.5, 0.0, alpha=1e-6)
    bare_f = types.SimpleNamespace(handle=bare._handle(), n_samples=4)
    assert _entry(bo, fants[0], [bare_f, fants[2]], con.lb, con.ub, inb)[0] == L.ERR_STATE
    assert L.lib().b200bo_gp_set_constrained_incumbent(fants[0].handle.ptr, None, 2, None, None, None, None) == \
        L.ERR_ARG


# ---- values on the grown handles -------------------------------------------------------------------------------
def _restated(gps, X, P, S, seed, inb, con, extra=0):
    ds = [_as_dict(g) for g in gps]
    out, best, ok, _ = CB.pipeline(ds, X, P, np.random.RandomState(seed), S, extra, inb, con.lb, con.ub)
    return ds, out, best, ok


@pytest.mark.parametrize("kind", ["cnei", "logcnei"])
@pytest.mark.parametrize("pipe", ["bulk", "bulk_nomc"])
@pytest.mark.parametrize("S", [1, 4, 16])
@pytest.mark.parametrize("d", [3, 20])
@pytest.mark.parametrize("J", [1, 2])
@pytest.mark.parametrize("p", [1, 7])
def test_values_match_the_restatement(bo, monkeypatch, kind, pipe, S, d, J, p):
    import torch

    monkeypatch.setenv("B200BO_PREDICT_PIPE", pipe)
    X, gps, con, P = _problem(bo, 300, d, J, p=p)
    n = X.shape[0]
    log = kind == "logcnei"
    acq, closure, space = _closure(bo, gps, con, X, P, S, seed=3, log=log)
    inb = np.ones(n + p, bool)
    ds, out, best, ok = _restated(gps, X, P, S, 3, inb, con)
    for f, (Fd, _) in zip([acq.fantasies, *acq.constraint_fantasies], out):
        assert np.all(np.abs(f.F - Fd) <= 1e-8 * (np.abs(Fd) + 1.0))
    assert np.array_equal(CO.eligible(inb, [f.F for f in acq.constraint_fantasies], con.lb, con.ub), ok)
    np.testing.assert_allclose(acq.fantasies.best, best, rtol=1e-9, atol=1e-9)
    Xa = np.vstack([X, P])
    As = [o[1] for o in out]
    rs = np.random.RandomState(5)
    for m in (1000, 20):  # tiled kernel, small-batch kernels
        r = m - 2 * p
        Xc = np.vstack([rs.uniform(size=(r, d)), P, P + 1e-7])  # then the pending rows and their neighbours
        want = -CB.cnei(ds, Xa, As, acq.fantasies.best, Xc, 0.01, con.lb, con.ub, log=log)
        got = closure(Xc)
        fin = np.isfinite(want)
        assert np.array_equal(fin, np.isfinite(got))
        np.testing.assert_allclose(got[:r], want[:r], rtol=1e-7, atol=1e-10)
        # at and next to the pending rows K0' is ill-conditioned: DESIGN.md 4.14's bar, and in LogCNEI's deep tail
        # (log values below -1e3, where sigma0 ~ sqrt(tau) and the log value ~ -z^2 / 2 doubles sigma0's relative
        # error) 1e-3
        tail = np.abs(want[r:]) >= 1e3 if log else np.zeros(2 * p, bool)
        near = fin[r:] & ~tail
        np.testing.assert_allclose(got[r:][near], want[r:][near], rtol=1e-5, atol=1e-10)
        np.testing.assert_allclose(got[r:][tail], want[r:][tail], rtol=1e-3)
        idx, val, top = closure.argmin_topk(Xc[:r], 5)
        order = np.lexsort((np.arange(r), want[:r]))
        assert idx == order[0] and np.array_equal(top, order[:5])
        Xd = torch.from_numpy(np.ascontiguousarray(Xc)).cuda()  # device-resident candidates: the host values
        outd = torch.empty(m, dtype=torch.float64, device="cuda")
        spec = closure.spec
        bo._lib.check(bo._lib.lib().b200bo_acq_eval_dev(C.byref(spec), Xd.data_ptr(), m, outd.data_ptr(), None, None,
                                                        0, None, 0, None))
        torch.cuda.synchronize()
        assert np.array_equal(outd.cpu().numpy(), got)


@pytest.mark.parametrize("kind", ["cnei", "logcnei"])
def test_philox_candidates_match_the_restatement(bo, kind):
    X, gps, con, P = _problem(bo, 300, 3, 2, p=5)
    log = kind == "logcnei"
    acq, closure, _ = _closure(bo, gps, con, X, P, 4, seed=2, log=log)
    ds, out, _, _ = _restated(gps, X, P, 4, 2, np.ones(305, bool), con)
    i, v, xb, ti, tx = closure.argmin_topk_philox(77, np.array([[0.0, 1.0]] * 3), 4000, 4)
    want = -CB.cnei(ds, np.vstack([X, P]), [o[1] for o in out], acq.fantasies.best, tx, 0.01, con.lb, con.ub, log=log)
    np.testing.assert_allclose(v, want[0], rtol=1e-7, atol=1e-10)
    assert np.all(np.diff(want) >= -1e-9 * (np.abs(want[:-1]) + 1e-12))
    assert np.array_equal(xb, tx[0])


def test_rows_one_by_one_equal_one_call(bo):
    """The class's extender, pick by pick, against one closure over all the rows: bit-equal fantasies, incumbents and
    values (each GP uses its pre-drawn z rows in order)."""
    X, gps, con, P = _problem(bo, 300, 3, 2, p=5)
    a, ca, _ = _closure(bo, gps, con, X, P, 4, seed=6)
    b, cb, _ = _closure(bo, gps, con, X, P[:1], 4, seed=6, extra=4)
    for row in P[1:]:
        b.condition_on_pending(row)
    for fa, fb in zip([a.fantasies, *a.constraint_fantasies], [b.fantasies, *b.constraint_fantasies]):
        assert np.array_equal(fa.F, fb.F) and np.array_equal(fa.best, fb.best)
    Xc = np.random.RandomState(2).uniform(size=(700, 3))
    assert np.array_equal(ca(Xc), cb(Xc))


def test_no_pending_rows_is_todays_cnei(bo):
    """p = 0: the closure equals the one-GP-at-a-time path of DESIGN.md 4.15 (set_fantasy_incumbent over cnei_eligible),
    the same draws and bit-equal incumbents and values."""
    from bayesianoptimization_b200.acquisition import _in_bounds, cnei_eligible

    X, gps, con, _ = _problem(bo, 300, 3, 2)
    X2 = X.copy()
    X2[:10, 0] = 1.5  # registered rows outside the bounds
    acq, closure, space = _closure(bo, gps, con, X2, None, 4, seed=8)
    rs = np.random.RandomState(8)
    fants = [g.noiseless_fantasies(4, random_state=rs) for g in gps]
    e = np.ascontiguousarray(cnei_eligible(_in_bounds(space), [f.F for f in fants[1:]], con.lb, con.ub), np.uint8)
    best = np.empty(4)
    bo._lib.check(bo._lib.lib().b200bo_gp_set_fantasy_incumbent(fants[0].handle.ptr, e.ctypes.data_as(
        C.POINTER(C.c_uint8)), bo._lib.as_dp(best)))
    assert np.array_equal(acq.fantasies.best, best)
    assert np.array_equal(acq._path_rng.randint(1 << 30), rs.randint(1 << 30))
    old = bo.FusedAcquisition(bo._lib.ACQ_CNEI, gps[0], con, xi=0.01, fantasies=fants[0], constraint_fantasies=fants[1:])
    Xc = np.random.RandomState(3).uniform(size=(500, 3))
    assert np.array_equal(closure(Xc), old(Xc))


@pytest.mark.parametrize("log", [False, True])
def test_unbounded_constraints_are_pending_nei(bo, log):
    """Every constraint with bounds (-inf, inf) and every row in bounds: best' is PendingNEI(NEI)'s largest fantasy over
    X u P.  PendingNEI raises best_s at a pending row on the device with a contracted FMA (fantasy_row_kernel), CNEI from
    the separately rounded values: bit-equal where the largest row is registered, within one rounding otherwise.  The
    values agree to round-off, with the same argmin and top-k."""
    X, gps, con, P = _problem(bo, 300, 3, 2, p=6)
    P[1] = X[int(np.argmax(gps[0]._y_raw))]  # a pending row at the incumbent's input
    con.lb, con.ub = np.full(2, -np.inf), np.full(2, np.inf)
    acq, closure, _ = _closure(bo, gps, con, X, P, 8, seed=9, log=log)
    nei = (bo.LogNoisyExpectedImprovement if log else bo.NoisyExpectedImprovement)(xi=0.01, n_samples=8)
    nei._path_rng = np.random.RandomState(9)
    nclosure = nei._closure(gps[0], None, types.SimpleNamespace(mask=np.ones(300, bool)), pending=P)
    F = acq.fantasies.F
    assert np.array_equal(F, nei.fantasies.F)
    assert np.array_equal(acq.fantasies.best, F.max(axis=0))
    top_reg = F[:300].max(axis=0) >= F[300:].max(axis=0)
    assert np.array_equal(acq.fantasies.best[top_reg], nei.fantasies.best[top_reg])
    ym = float(gps[0]._y_train_mean)
    assert np.all(np.abs(acq.fantasies.best - nei.fantasies.best) <= 4 * np.finfo(float).eps *
                  (np.abs(acq.fantasies.best) + abs(ym)))
    Xc = np.random.RandomState(4).uniform(size=(2000, 3))
    a, b = closure(Xc), nclosure(Xc)
    np.testing.assert_allclose(a, b, rtol=1e-10, atol=1e-13)
    ia, _, ta = closure.argmin_topk(Xc, 8)
    ib, _, tb = nclosure.argmin_topk(Xc, 8)
    assert ia == ib and np.array_equal(ta, tb)


def _cd5(f, rows, h):
    cols = []
    for e in np.eye(rows.shape[1]):
        cols.append((8 * (f(rows + h * e) - f(rows - h * e)) - (f(rows + 2 * h * e) - f(rows - 2 * h * e))) / (12 * h))
    return np.stack(cols, axis=1)


@pytest.mark.parametrize("kind", ["cnei", "logcnei"])
def test_gradient_matches_central_differences(bo, kind):
    X, gps, con, P = _problem(bo, 300, 3, 2, p=4)
    log = kind == "logcnei"
    acq, closure, _ = _closure(bo, gps, con, X, P, 4, seed=10, log=log)
    ds, out, _, _ = _restated(gps, X, P, 4, 10, np.ones(304, bool), con)
    Xa, As = np.vstack([X, P]), [o[1] for o in out]

    def f(rows):
        return -CB.cnei(ds, Xa, As, acq.fantasies.best, rows, 0.01, con.lb, con.ub, log=log)

    rows = np.random.RandomState(6).uniform(0.05, 0.95, size=(12, 3))
    val, grad = closure.value_and_grad(rows)
    np.testing.assert_allclose(val, f(rows), rtol=1e-7, atol=1e-10)
    with closure.refine_mode():
        cd = _cd5(closure, rows, 1e-5)
    assert np.all(np.isfinite(grad))
    np.testing.assert_allclose(grad, cd, rtol=2e-5, atol=1e-6 * (1.0 + np.abs(cd).max()))


def test_non_pd_pending_point_names_jitter_and_the_gp(bo):
    """A constraint GP with alpha = 0 (tau = 0) and one training row: a pending point on it gives the pivot 0."""
    from sklearn.gaussian_process.kernels import RBF

    X = np.array([[0.25, 0.5]])
    gp = _fit(bo, X, [1.0], 1.0, 0.5, 0.04, alpha=1e-6)
    c = bo.B200GaussianProcessRegressor(kernel=RBF(1.0), alpha=0.0, optimizer=None).fit(X, [0.1])
    con = types.SimpleNamespace(model=[c], lb=np.array([-np.inf]), ub=np.array([0.5]))
    with pytest.raises(np.linalg.LinAlgError, match=r"jitter.*constraint GP 0"):
        _closure(bo, [gp, c], con, X, X.copy(), 2, seed=0)


def test_host_side_transform_is_refused_before_any_draw(bo):
    X, gps, con, P = _problem(bo, 200, 3, 2)
    gps[2].__dict__["_b200_xform"] = ("host", None)  # as a categorical kernel transform leaves it
    acq = bo.ConstrainedNoisyExpectedImprovement(n_samples=2)
    rs = np.random.RandomState(0)
    space = types.SimpleNamespace(params=X, bounds=np.array([[0.0, 1.0]] * 3))
    acq._path_rng = rs
    with pytest.raises(NotImplementedError, match="host-side"):
        acq._closure(gps[0], con, space, pending=P[:1])
    assert np.array_equal(rs.get_state()[1], np.random.RandomState(0).get_state()[1])


def test_production_size_clustered(bo):
    """The C4 shape: N = 2048, d = 16, J = 2, S = 16, p = 15 pending rows, clustered inputs (cond(K0) >~ 1e8): LogCNEI
    and CNEI at 4096 candidates within 1e-6 relative of the restatement (CNEI held to |want| + 1e-3 max|want|, as in
    DESIGN.md 4.15)."""
    rs = np.random.RandomState(11)
    n, d, S, p = 2048, 16, 16, 15
    centers = rs.uniform(size=(64, d))
    X = centers[rs.randint(0, 64, n)] + 0.02 * rs.standard_normal((n, d))
    _, gps, con, _ = _problem(bo, n, d, 2, seed=12, ls=2.0, X=X, alpha=1e-6)
    P = np.vstack([X[:4] + 1e-3, rs.uniform(size=(p - 4, d)) * 0.9 + 0.05])
    box = np.array([[-1.0, 2.0]] * d)
    worst = 0.0
    for log in (False, True):
        acq, closure, _ = _closure(bo, gps, con, X, P, S, seed=9, box=box, log=log)
        ds, out, best, ok = _restated(gps, X, P, S, 9, np.ones(n + p, bool), con)
        assert np.linalg.cond(ds[0]["kc"](X) + 1e-6 * np.eye(n)) > 1e8
        Xc = rs.uniform(size=(4096, d)) * 0.9 + 0.05
        want = -CB.cnei(ds, np.vstack([X, P]), [o[1] for o in out], acq.fantasies.best, Xc, 0.01, con.lb, con.ub,
                        log=log)
        got = closure(Xc)
        big = np.max(np.abs(want))
        err = np.max(np.abs(got - want) / (np.abs(want) + (0.0 if log else 1e-3 * big)))
        print(f"production size, {'LogCNEI' if log else 'CNEI'} with {p} pending rows: largest error {err:.2e}")
        worst = max(worst, err)
    assert worst < 1e-6


# ---- the acquisition in the batch loop ---------------------------------------------------------------------------
PB = {f"x{j}": (0.0, 1.0) for j in range(3)}
CON = [(0.9, 0.5, 0.01), (1.1, 0.45, 0.02)]  # (constant, length scale, noise) of the constraint GPs


def _cfuns(x):
    return np.array([x[0] + x[1] - 0.8, x[2] - x[0]])


def _cspace(bo, J=2, n=40, seed=3, lb=(-np.inf, -0.5), ub=(0.3, 0.4)):
    from bayes_opt.target_space import TargetSpace
    from scipy.optimize import NonlinearConstraint

    from bayesianoptimization_b200.gpr import to_b200_gp

    space = TargetSpace(None, PB, constraint=NonlinearConstraint(lambda *a: 0.0, np.array(lb[:J]), np.array(ub[:J])))
    cm = space.constraint
    cm._model = [to_b200_gp(m) for m in cm.model]  # as enable(optimizer) does
    for m, (c, ls, noise) in zip(cm.model, CON):
        m.set_params(kernel=ConstantKernel(c) * Matern(length_scale=ls, nu=2.5) + WhiteKernel(noise), optimizer=None)
    rs = np.random.RandomState(seed)
    for _ in range(n):
        x = space.random_sample(random_state=rs)
        cv = _cfuns(x)[:J] + 0.05 * rs.randn(J)
        space.register(x, float(np.sin(5 * x.sum()) + np.cos(3 * x[0]) + 0.2 * rs.randn()),
                       constraint_value=cv if J > 1 else float(cv[0]))
    return space


def _gp(bo):
    k = ConstantKernel(1.0) * Matern(length_scale=0.4, nu=2.5) + WhiteKernel(0.04)
    return bo.B200GaussianProcessRegressor(kernel=k, alpha=1e-10, normalize_y=True, optimizer=None)


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
def test_q1_equals_suggest(bo, ref, source):
    space, out = _cspace(bo), []
    for batch in (True, False):
        base = bo.LogConstrainedNoisyExpectedImprovement(n_samples=4)
        base.b200_candidate_source = source
        rs = np.random.RandomState(11)
        if batch:
            x = _quiet(bo.PendingNEI(base).suggest_batch, _gp(bo), space, 1, n_random=5000, n_smart=3,
                       random_state=rs)[0]
        else:
            x = _quiet(base.suggest, _gp(bo), space, n_random=5000, n_smart=3, random_state=rs)
        out.append((x, rs.get_state()))
    assert np.array_equal(out[0][0], out[1][0])
    assert np.array_equal(out[0][1][1], out[1][1][1]) and out[0][1][2:] == out[1][1][2:]


def test_batch_reaches_the_optimum_of_a_restated_pipeline(bo, ref):
    """Round j of the restatement: every GP's fantasies conditioned on the device's picks 0..j-1 from the same stream
    (per GP Z, E, its q - 1 z rows, then the candidates), best' by the rule, the same random stage, SciPy L-BFGS-B from
    its top n_smart: the restated LogCNEI at the device's pick j is at least the round's best, to 1e-4 relative."""
    from scipy.optimize import minimize

    q, S = 4, 4
    space = _cspace(bo)
    gp = _gp(bo)
    acq = bo.PendingNEI(bo.LogConstrainedNoisyExpectedImprovement(n_samples=S))
    picks = _quiet(acq.suggest_batch, gp, space, q, n_random=3000, n_smart=3, random_state=np.random.RandomState(5))
    assert picks.shape == (q, 3) and len({p.tobytes() for p in picks}) == q and len(acq.dummies) == q
    X, n = space.params, len(space)
    cm = space.constraint
    ds = [_as_dict(gp)] + [_as_dict(m) for m in cm.model]
    rs = np.random.RandomState(5)
    draws = CB.draws(rs, n, S, 2, q - 1)
    cand = space.random_sample(3000, random_state=rs)
    for j in range(q):
        P = picks[:j]
        grown = [CB.grown(g, X, P, *dr) for g, dr in zip(ds, draws)]
        Fd = [CB.data_units(F, g) for (F, _), g in zip(grown, ds)]
        best, _ = CB.incumbents(Fd[0], Fd[1:], np.ones(n + j, bool), cm.lb, cm.ub)
        Xa, As = np.vstack([X, P]), [A for _, A in grown]

        def neg(x, Xa=Xa, As=As, best=best):
            return -CB.cnei(ds, Xa, As, best, np.atleast_2d(x), 0.0, cm.lb, cm.ub, log=True)

        vals = neg(cand)
        best_v = float(vals.min())
        for s in cand[np.argsort(vals)[:3]]:
            r = minimize(lambda x: float(neg(x)[0]), s, bounds=space.bounds, method="L-BFGS-B")
            best_v = min(best_v, float(r.fun))
        got = float(neg(picks[j])[0])
        assert got <= best_v + 1e-4 * (abs(best_v) + 1e-3), (j, got, best_v)


def _state(bo, h, n):
    L = bo._lib
    out = []
    for what, size in ((L.GET_L, n * n), (L.GET_ALPHA, n), (L.GET_LINV, n * n), (L.GET_K, n * n)):
        buf = np.empty(size)
        L.check(L.lib().b200bo_gp_get(h.ptr, what, buf.ctypes.data_as(C.POINTER(C.c_double)), size))
        out.append(buf)
    return out


def test_batch_leaves_every_gp_and_noiseless_regressor_unchanged(bo, ref):
    space = _cspace(bo)
    n = len(space)
    gp = _gp(bo).fit(space.params, space.target)
    space.constraint.fit(space.params, space._constraint_values)
    gps = [gp, *space.constraint.model]
    Xq = np.random.RandomState(1).uniform(size=(50, 3))
    preds = [g.predict(Xq, return_std=True) for g in gps]
    nls = [g.noiseless_fantasies(4, random_state=0).gp for g in gps]
    before = [_state(bo, nl._handle(), n) for nl in nls]
    acq = bo.PendingNEI(bo.ConstrainedNoisyExpectedImprovement(n_samples=4))
    acq.dummies = [np.full(3, 0.31)]
    picks = _quiet(acq.suggest_batch, gp, space, 4, n_random=2000, n_smart=2, fit_gp=False, random_state=3)
    assert picks.shape == (4, 3) and len(acq.dummies) == 5
    for g, (mu0, sd0), nl, b in zip(gps, preds, nls, before):
        mu1, sd1 = g.predict(Xq, return_std=True)
        assert np.array_equal(mu0, mu1) and np.array_equal(sd0, sd1) and g.X_train_.shape[0] == n
        assert g.__dict__["_b200_noiseless"]._handle().ptr.value == nl._handle().ptr.value
        for u, v in zip(b, _state(bo, nl._handle(), n)):
            assert np.array_equal(u, v)


def test_suggests_without_a_feasible_point(bo, ref):
    space = _cspace(bo, J=1, lb=(5.0,), ub=(6.0,))
    acq = bo.PendingNEI(bo.LogConstrainedNoisyExpectedImprovement(n_samples=4))
    picks = _quiet(acq.suggest_batch, _gp(bo), space, 3, n_random=2000, n_smart=2, random_state=4)
    assert picks.shape == (3, 3) and np.all(np.isfinite(picks))
    f = acq.base_acquisition.fantasies
    assert np.array_equal(f.best, f.F.min(axis=0))  # every sample at the floor, over X u P


def test_live_optimizer_async_pattern_and_state_round_trip(bo, ref, tmp_path):
    from scipy.optimize import NonlinearConstraint

    con = NonlinearConstraint(lambda x0, x1, x2: x0 + x1, -np.inf, 1.1)

    def make():
        opt = ref.BayesianOptimization(f=None, pbounds=PB, constraint=con, random_state=4, verbose=0,
                                       acquisition_function=bo.PendingNEI(bo.LogConstrainedNoisyExpectedImprovement(
                                           n_samples=4)))
        opt.set_gp_params(alpha=2e-3)
        bo.enable(opt)
        opt._gp.set_params(optimizer=None)
        for m in opt.constraint.model:  # noisy constraint GPs
            m.set_params(kernel=Matern(nu=2.5) + WhiteKernel(1e-3), optimizer=None)
        return opt

    opt = make()
    rs = np.random.RandomState(0)
    for _ in range(20):
        x = rs.uniform(size=3)
        opt.register(params=x, target=float(np.sin(5 * x.sum()) + 0.05 * rs.randn()),
                     constraint_value=float(x[0] + x[1] + 0.05 * rs.randn()))
    xs = [_quiet(opt.suggest) for _ in range(3)]  # three workers, nothing registered in between
    arr = [opt._space.params_to_array(x) for x in xs]
    assert len({a.tobytes() for a in arr}) == 3 and len(opt._acquisition_function.dummies) == 3
    opt.register(params=xs[0], target=0.3, constraint_value=0.5)  # worker 0 reports: its dummy expires
    _quiet(opt.suggest)
    dummies = opt._acquisition_function.dummies
    assert len(dummies) == 3 and not any(np.allclose(d, arr[0]) for d in dummies)
    path = tmp_path / "state.json"
    opt.save_state(path)
    other = make()
    other.load_state(path)
    assert [d.tolist() for d in other._acquisition_function.dummies] == [d.tolist() for d in dummies]
    Xb = _quiet(bo.suggest_batch, other, 5)
    assert len(Xb) == 5 and len(other._acquisition_function.dummies) == 8

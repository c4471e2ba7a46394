"""NEI with pending points on the device (DESIGN.md 4.14) against the numpy restatement tests/nei_batch_oracle.py: the
pending fantasies and best_s of b200bo_gp_condition_fantasies, bit-equality of row-by-row and one-call conditioning,
the fork's fantasy state, NEI / LogNEI values, selection and gradients on the grown handle, PendingNEI's batches and
its async loop in the reference's BayesianOptimization."""
from __future__ import annotations

import warnings

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import ConstantKernel, Matern, WhiteKernel

import nei_batch_oracle as NB
import nei_oracle as NO

pytestmark = pytest.mark.gpu

C0, LS, NOISE = 1.7, 0.35, 0.04
CASES = {"white": (NOISE, 1e-8), "tau": (0.0, 1e-6)}  # (WhiteKernel noise, alpha): sigma_n^2 > tau, sigma_n^2 = tau


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


def _fit(bo, case, n=300, d=3, seed=0):
    noise, alpha = CASES[case]
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    y = np.sin(3.0 * X.sum(1)) + np.sqrt(NOISE) * rs.randn(n)
    k = ConstantKernel(C0) * Matern(length_scale=LS, nu=2.5)
    if noise > 0:
        k = k + WhiteKernel(noise)
    gp = bo.B200GaussianProcessRegressor(kernel=k, alpha=alpha, normalize_y=True, optimizer=None)
    gp.fit(X, y)
    P = rs.uniform(size=(6, d))
    P[1] = X[7] + 1e-3  # near a training row
    P[2] = X[int(np.argmax(y))]  # at the incumbent's input
    return gp, X, P


def _oracle(gp, case, X, P, S, seed, rows, mask=None):
    noise, alpha = CASES[case]
    kc = ConstantKernel(C0) * Matern(length_scale=LS, nu=2.5)
    tau = min(alpha, 1e-6)
    ym, ys = float(gp._y_train_mean), float(gp._y_train_std)
    y_n = (gp._y_raw - ym) / ys
    Z, E, Zp = NB.draws(np.random.RandomState(seed), len(y_n), S, rows)
    mask = np.ones(len(y_n), bool) if mask is None else mask
    Fa, A, best = NB.pending_fantasies(kc, X, P, y_n, alpha + noise, tau, Z, E, Zp, mask, ym, ys)
    return kc, tau, ym, ys, Fa, A, best


def _state(bo, h, n):
    import ctypes as C

    L = bo._lib
    out = []
    for what, size in ((L.GET_L, n * n), (L.GET_ALPHA, n), (L.GET_LINV, n * n), (L.GET_K, n * n)):
        buf = np.empty(size)
        L.check(L.lib().b200bo_gp_get(h.ptr, what, buf.ctypes.data_as(C.POINTER(C.c_double)), size))
        out.append(buf)
    return out


@pytest.mark.parametrize("case", list(CASES))
def test_pending_fantasies_match_the_restatement(bo, case):
    gp, X, P = _fit(bo, case)
    n, S = X.shape[0], 4
    mask = np.ones(n, bool)
    mask[::3] = False
    fant0 = gp.noiseless_fantasies(S, incumbent=mask, random_state=11)
    nl = fant0.gp
    before = _state(bo, nl._handle(), n)
    Xq = np.random.RandomState(1).uniform(size=(50, 3))
    mu0, sd0 = gp.predict(Xq, return_std=True)
    fant = gp.noiseless_fantasies(S, incumbent=mask, random_state=11, pending=P[:4], extra_rows=2)
    fant.condition_on_pending(P[4:])
    kc, tau, ym, ys, Fa, A, best = _oracle(gp, case, X, P, S, 11, 6, mask)
    want = ys * Fa + ym
    assert fant.F.shape == (n + 6, S)
    assert np.all(np.abs(fant.F - want) <= 1e-8 * (np.abs(want) + ys))
    assert np.all(np.abs(fant.best - best) <= 1e-8 * (np.abs(best) + ys))
    assert np.all(fant.best >= fant0.best)
    np.testing.assert_array_equal(fant.F[:n], fant0.F)
    # the caller's GP and the noiseless regressor are bit-unchanged
    mu1, sd1 = gp.predict(Xq, return_std=True)
    assert np.array_equal(mu0, mu1) and np.array_equal(sd0, sd1)
    for a, b in zip(before, _state(bo, nl._handle(), n)):
        assert np.array_equal(a, b)
    assert fant.gp is not gp and fant.gp is not nl and gp.X_train_.shape[0] == n
    with pytest.raises(ValueError, match="pre-drawn"):
        fant.condition_on_pending(P[:1])


@pytest.mark.parametrize("case", list(CASES))
def test_single_rows_are_bit_equal_to_one_call(bo, case):
    gp, X, P = _fit(bo, case)
    fa = gp.noiseless_fantasies(4, random_state=3, extra_rows=6)
    fb = gp.noiseless_fantasies(4, random_state=3, extra_rows=6)
    fa.condition_on_pending(P)
    for row in P:
        fb.condition_on_pending(row)
    assert np.array_equal(fa.F, fb.F) and np.array_equal(fa.best, fb.best)
    Xc = np.random.RandomState(2).uniform(size=(700, 3))
    for code in (bo._lib.ACQ_NEI, bo._lib.ACQ_LOGNEI):
        va = bo.FusedAcquisition(code, gp, xi=0.01, fantasies=fa)(Xc)
        vb = bo.FusedAcquisition(code, gp, xi=0.01, fantasies=fb)(Xc)
        assert np.array_equal(va, vb)


@pytest.mark.parametrize("case", list(CASES))
def test_fork_without_rows_equals_its_source(bo, case):
    gp, X, P = _fit(bo, case)  # n = 300: capacity 384
    Xc = np.random.RandomState(4).uniform(size=(900, 3))
    vals = {}
    for extra in (0, 10, 200):  # the source itself, a fork at the same capacity, a re-pitched fork
        fant = gp.noiseless_fantasies(4, random_state=5, extra_rows=extra)
        acq = bo.FusedAcquisition(bo._lib.ACQ_LOGNEI, gp, xi=0.01, fantasies=fant)
        vals[extra] = (acq(Xc), fant.F, fant.best)
    assert all(np.array_equal(a, b) for a, b in zip(vals[0], vals[10]))
    np.testing.assert_allclose(vals[200][0], vals[0][0], rtol=1e-10, atol=1e-12)
    assert np.array_equal(vals[200][1], vals[0][1]) and np.array_equal(vals[200][2], vals[0][2])


@pytest.mark.parametrize("kind", ["nei", "lognei"])
@pytest.mark.parametrize("pipe", ["bulk", "bulk_nomc"])
@pytest.mark.parametrize("case", list(CASES))
def test_values_and_selection_match_the_restatement(bo, monkeypatch, kind, pipe, case):
    monkeypatch.setenv("B200BO_PREDICT_PIPE", pipe)
    gp, X, P = _fit(bo, case)
    S = 4
    fant = gp.noiseless_fantasies(S, random_state=7, pending=P)
    kc, tau, ym, ys, Fa, A, best = _oracle(gp, case, X, P, S, 7, len(P))
    Xa = np.vstack([X, P])
    code = bo._lib.ACQ_NEI if kind == "nei" else bo._lib.ACQ_LOGNEI
    acq = bo.FusedAcquisition(code, gp, xi=0.01, fantasies=fant)
    rs = np.random.RandomState(8)
    for m in (1000, 20):  # tiled kernel, small-batch kernels
        Xc = np.vstack([rs.uniform(size=(m - 2 * len(P), 3)), P, P + 1e-7])  # the pending rows and their neighbours
        want = -NB.nei(kc, Xa, A, best, tau, Xc, 0.01, ym, ys, log=(kind == "lognei"))
        got = acq(Xc)
        ok = np.isfinite(want)
        assert np.array_equal(ok, np.isfinite(got))
        r = m - 2 * len(P)  # random rows; then the pending rows and their neighbours, where K0' is ill-conditioned
        np.testing.assert_allclose(got[:r], want[:r], rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(got[r:][ok[r:]], want[r:][ok[r:]], rtol=1e-5, atol=1e-10)
        idx, val, top = acq.argmin_topk(Xc[:m - 2 * len(P)], 5)
        order = np.lexsort((np.arange(m - 2 * len(P)), want[:m - 2 * len(P)]))
        assert idx == order[0] and np.array_equal(top, order[:5])


def _cd5(f, rows, h):
    cols = []
    for e in np.eye(rows.shape[1]):
        cols.append((8 * (f(rows + h * e) - f(rows - h * e)) - (f(rows + 2 * h * e) - f(rows - 2 * h * e))) / (12 * h))
    return np.stack(cols, axis=1)


@pytest.mark.parametrize("kind", ["nei", "lognei"])
def test_gradient_matches_central_differences(bo, kind):
    gp, X, P = _fit(bo, "white")
    fant = gp.noiseless_fantasies(4, random_state=9, pending=P)
    kc, tau, ym, ys, Fa, A, best = _oracle(gp, "white", X, P, 4, 9, len(P))
    Xa = np.vstack([X, P])
    code = bo._lib.ACQ_NEI if kind == "nei" else bo._lib.ACQ_LOGNEI
    acq = bo.FusedAcquisition(code, gp, xi=0.01, fantasies=fant)

    def f(rows):
        return -NB.nei(kc, Xa, A, best, tau, rows, 0.01, ym, ys, log=(kind == "lognei"))

    rows = np.random.RandomState(6).uniform(0.05, 0.95, size=(12, 3))
    val, grad = acq.value_and_grad(rows)
    np.testing.assert_allclose(val, f(rows), rtol=1e-7, atol=1e-10)
    cd = _cd5(f, rows, 1e-6)
    np.testing.assert_allclose(grad, cd, rtol=2e-5, atol=1e-6 * (1.0 + np.abs(cd).max()))


def test_non_pd_pending_point_raises_linalg_error_naming_jitter(bo):
    """One training point, alpha = 0 (tau = 0), unit variance: a pending point on it gives the pivot 1 - 1 = 0."""
    from sklearn.gaussian_process.kernels import RBF

    gp = bo.B200GaussianProcessRegressor(kernel=RBF(1.0), alpha=0.0, optimizer=None).fit(np.array([[0.25, 0.5]]), [1.0])
    mu0 = gp.predict(np.array([[0.9, 0.1]]))
    with pytest.raises(np.linalg.LinAlgError, match="jitter"):
        gp.noiseless_fantasies(2, random_state=0, pending=np.array([[0.25, 0.5]]))
    assert np.array_equal(gp.predict(np.array([[0.9, 0.1]])), mu0)


# ---- the acquisition ------------------------------------------------------------------------------------------
PB = {f"x{j}": (0.0, 1.0) for j in range(3)}


def _space(n=50, seed=3):
    from bayes_opt.target_space import TargetSpace

    space = TargetSpace(None, PB)
    rs = np.random.RandomState(seed)
    for _ in range(n):
        x = space.random_sample(random_state=rs)
        space.register(x, float(np.sin(5 * x.sum()) + np.cos(3 * x[0]) + 0.2 * rs.randn()))
    return space


def _gp(bo):
    k = ConstantKernel(1.0) * Matern(length_scale=0.4, nu=2.5) + WhiteKernel(0.04)
    return bo.B200GaussianProcessRegressor(kernel=k, alpha=1e-10, normalize_y=True, optimizer=None)


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
@pytest.mark.parametrize("cls", ["NoisyExpectedImprovement", "LogNoisyExpectedImprovement"])
def test_q1_equals_suggest(bo, ref, cls, source):
    space, out = _space(), []
    for batch in (True, False):
        base = getattr(bo, cls)(n_samples=4)
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
    """Round j of the restatement: the fantasies conditioned on the device's picks 0..j-1 drawn from the same stream
    (Z, E, the q - 1 z rows, then the candidates), the same random stage, SciPy L-BFGS-B from its top n_smart.  The
    check is not equality of the picks (two L-BFGS-B implementations stop at different points of a flat optimum):
    the restated LogNEI at the device's pick j is at least the restated round's best, to 1e-4 relative; the picks are
    distinct."""
    from scipy.optimize import minimize

    q, S = 4, 4
    space = _space()
    gp = _gp(bo)
    acq = bo.PendingNEI(bo.LogNoisyExpectedImprovement(n_samples=S))
    rs = np.random.RandomState(5)
    picks = _quiet(acq.suggest_batch, gp, space, q, n_random=3000, n_smart=3, random_state=rs)
    assert picks.shape == (q, 3) and len({p.tobytes() for p in picks}) == q
    assert len(acq.dummies) == q
    X = space.params
    n = X.shape[0]
    kc = gp.kernel_.k1
    tau, s2 = 1e-10, 1e-10 + float(gp.kernel_.k2.noise_level)
    ym, ys = float(gp._y_train_mean), float(gp._y_train_std)
    y_n = (space.target - ym) / ys
    rs = np.random.RandomState(5)
    Z, E, Zp = NB.draws(rs, n, S, q - 1)
    cand = space.random_sample(3000, random_state=rs)
    for j in range(q):
        P = picks[:j]
        _, A, best = NB.pending_fantasies(kc, X, P, y_n, s2, tau, Z, E, Zp, np.ones(n, bool), ym, ys)
        Xa = np.vstack([X, P])

        def neg(x, A=A, best=best, Xa=Xa):
            return -NB.nei(kc, Xa, A, best, tau, np.atleast_2d(x), 0.0, ym, ys, log=True)

        vals = neg(cand)
        best_v = float(vals.min())
        for s in cand[np.argsort(vals)[:3]]:
            r = minimize(lambda x: float(neg(x)[0]), s, bounds=space.bounds, method="L-BFGS-B")
            best_v = min(best_v, float(r.fun))
        got = float(neg(picks[j])[0])
        assert got <= best_v + 1e-4 * (abs(best_v) + 1e-3), (j, got, best_v)


def test_live_optimizer_async_pattern_and_state_round_trip(bo, ref, tmp_path):
    def make():
        opt = ref.BayesianOptimization(f=None, pbounds=PB, random_state=4, verbose=0,
                                       acquisition_function=bo.PendingNEI(bo.NoisyExpectedImprovement(n_samples=4)))
        opt.set_gp_params(alpha=2e-3)  # noise through alpha: the noiseless GP is a second handle
        bo.enable(opt)
        opt._gp.set_params(optimizer=None)
        return opt

    opt = make()
    rs = np.random.RandomState(0)
    for _ in range(20):
        x = rs.uniform(size=3)
        opt.register(params=x, target=float(np.sin(5 * x.sum()) + 0.05 * rs.randn()))
    xs = [_quiet(opt.suggest) for _ in range(3)]  # three workers, nothing registered in between
    arr = [opt._space.params_to_array(x) for x in xs]
    assert len({a.tobytes() for a in arr}) == 3 and len(opt._acquisition_function.dummies) == 3
    opt.register(params=xs[0], target=0.3)  # worker 0 reports: its dummy expires at the next suggest
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


def test_batch_leaves_the_gp_and_the_noiseless_regressor_unchanged(bo, ref):
    space = _space()
    gp = _gp(bo).fit(space.params, space.target)
    Xq = np.random.RandomState(1).uniform(size=(50, 3))
    mu0, sd0 = gp.predict(Xq, return_std=True)
    nl = gp.noiseless_fantasies(4, random_state=0).gp
    before = _state(bo, nl._handle(), len(space))
    acq = bo.PendingNEI(bo.LogNoisyExpectedImprovement(n_samples=4))
    acq.dummies = [np.full(3, 0.31)]
    picks = _quiet(acq.suggest_batch, gp, space, 4, n_random=2000, n_smart=2, fit_gp=False, random_state=3)
    assert picks.shape == (4, 3) and len(acq.dummies) == 5
    mu1, sd1 = gp.predict(Xq, return_std=True)
    assert np.array_equal(mu0, mu1) and np.array_equal(sd0, sd1) and gp.X_train_.shape[0] == len(space)
    assert gp.__dict__["_b200_noiseless"]._handle().ptr.value == nl._handle().ptr.value
    for a, b in zip(before, _state(bo, nl._handle(), len(space))):
        assert np.array_equal(a, b)


def test_host_side_transform_with_pending_rows_is_refused(bo):
    gp, X, P = _fit(bo, "white")
    gp.__dict__["_b200_xform"] = ("host", None)  # as a categorical kernel transform leaves it
    with pytest.raises(NotImplementedError, match="host-side"):
        gp.noiseless_fantasies(4, random_state=0, pending=P[:1])

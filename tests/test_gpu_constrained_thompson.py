"""Constrained Thompson sampling on the device (paths.ConstrainedPaths, ConstrainedThompsonSampling): the raw values
of every set, the combine rule restated in numpy on the device's own values (bit for bit), parity with an independent
restatement of the paths on identical draws, the fused selection against numpy, the Philox source, suggest() against
a host implementation, and runs through the reference's BayesianOptimization driver."""
import ctypes as C
import warnings

import numpy as np
import pytest
from scipy.linalg import cho_solve, cholesky
from sklearn.gaussian_process.kernels import RBF, Matern

import thompson_oracle as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def merit_rule(raw, lb, ub, bound):
    """The combine rule restated: raw (M, G, q), lb / ub (G-1,), bound (q,) -> (M, q) merit.  Same operations in the
    same order as the kernel (adds, subtracts, NaN-propagating max, one multiply)."""
    f = raw[:, 0, :]
    viol = np.zeros_like(f)
    for j in range(1, raw.shape[1]):
        c = raw[:, j, :]
        viol = viol + (np.maximum(0.0, lb[j - 1] - c) + np.maximum(0.0, c - ub[j - 1]))
    t = 2.0 * bound + 1.0
    return np.where(viol == 0.0, f, -(t * (1.0 + viol)))


NUS = [2.5, 1.5, 0.5, np.inf]  # the covariance family of set g is NUS[g % 4]: every set has its own


def _kernel(nu, ls):
    return RBF(ls) if nu == np.inf else Matern(ls, nu=nu)


def _fit_sets(bo, G, n=300, d=3, seed=1, ls=0.5, alpha=1e-6):
    """G device GPs on the same inputs: the target (g = 0) and G-1 constraint functions."""
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    gps, ys = [], []
    for g in range(G):
        y = np.sin(3 * X.sum(1) + g) + 0.3 * g * X[:, 0] + 0.05 * rs.randn(n)
        gps.append(bo.B200GaussianProcessRegressor(kernel=_kernel(NUS[g % 4], ls), alpha=alpha, normalize_y=True,
                                                   optimizer=None).fit(X, y))
        ys.append(y)
    return X, ys, gps, rs


def _bounds_from(vals):
    """Bounds of J constraints that each hold on most rows: one-sided lower, one-sided upper, two-sided in turn."""
    J = vals.shape[1] - 1
    lb, ub = np.full(J, -np.inf), np.full(J, np.inf)
    for j in range(J):
        c = vals[:, j + 1, :].ravel()
        lo, hi = np.quantile(c, 0.15), np.quantile(c, 0.85)
        if j % 3 == 0:
            lb[j] = lo
        elif j % 3 == 1:
            ub[j] = hi
        else:
            lb[j], ub[j] = lo, hi
    return lb, ub


def _constrained(bo, gps, q, L, seed, lb=None, ub=None, Xb=None):
    from bayesianoptimization_b200.paths import ConstrainedPaths

    sets = [g.sample_paths(q, L, random_state=seed + i) for i, g in enumerate(gps)]
    if lb is None:  # bounds from the constraint paths' values on Xb
        vals = np.stack([s(Xb) for s in sets], axis=1)
        lb, ub = _bounds_from(vals)
    return ConstrainedPaths(sets[0], sets[1:], lb, ub), sets, lb, ub


@pytest.mark.parametrize("J,q", [(1, 1), (2, 3), (7, 16), (2, 16), (7, 1)])
def test_raw_values_and_combine_rule_are_bit_exact(bo, J, q):
    X, ys, gps, rs = _fit_sets(bo, J + 1, seed=J * 10 + q)
    Xc = rs.uniform(-0.1, 1.1, size=(3000, 3))
    cp, sets, lb, ub = _constrained(bo, gps, q, 512, 7, Xb=Xc)
    raw = cp.raw(Xc)
    assert raw.shape == (3000, J + 1, q)
    for g, s in enumerate(sets):  # 1. every set's values are exactly PosteriorPaths.__call__'s
        assert np.array_equal(raw[:, g, :], s(Xc))
    merit = cp(Xc)
    want = merit_rule(raw, lb, ub, sets[0].bound())
    assert np.array_equal(merit, want)  # 2. bit for bit
    feas = merit == raw[:, 0, :]
    print(f"J={J} q={q}: {feas.mean():.2f} of (row, path) pairs feasible")
    assert 0.05 < feas.mean() < 0.95  # both tiers are exercised
    for p in range(q):  # the tiers never mix
        assert np.all(merit[~feas[:, p], p] < merit[feas[:, p], p].min())


def _restated_bound(X, y, dr, kind, nu, ls, const, alpha, normalize=True):
    """B_p restated from scratch: |y_mean| + s_y (sqrt(2c/L) sum_l |w_lp| + c sum_i |v_ip|), v = K^-1 r."""
    from oracle.gp_oracle import kernel_train

    m, s = (float(np.mean(y)), float(np.std(y))) if normalize else (0.0, 1.0)
    omega, b, w, eps = dr
    K = kernel_train(X, kind=kind, nu=nu, length_scale=ls, const=const)
    K[np.diag_indices_from(K)] += alpha
    r = (y - m)[:, None] / s - T.features(X / ls, omega, b, const) @ w - eps
    v = cho_solve((cholesky(K, lower=True), True), r)
    return abs(m) + s * (np.sqrt(2.0 * const / w.shape[0]) * np.abs(w).sum(0) + const * np.abs(v).sum(0))


@pytest.mark.parametrize("J,q", [(1, 1), (2, 3), (7, 16)])
def test_parity_with_an_independent_restatement_on_identical_draws(bo, J, q):
    n, d, L, ls, alpha = 300, 3, 512, 0.5, 1e-6
    X, ys, gps, rs = _fit_sets(bo, J + 1, n=n, d=d, seed=J + 100, ls=ls, alpha=alpha)
    Xc = rs.uniform(-0.1, 1.1, size=(3000, d))
    cp, sets, lb, ub = _constrained(bo, gps, q, L, 7, Xb=Xc)
    oracle_vals, bounds, s_y = [], [], []
    for g in range(J + 1):
        nu = NUS[g % 4]
        kind = T.KIND_RBF if nu == np.inf else T.KIND_MATERN
        dr = T.draws(np.random.RandomState(7 + g), q, L, d, nu, n, alpha)
        oracle_vals.append(T.make_paths(X, ys[g], dr, kind=kind, nu=nu, length_scale=ls, alpha=alpha)(Xc))
        bounds.append(_restated_bound(X, ys[g], dr, kind, nu, ls, 1.0, alpha))
        s_y.append(float(np.std(ys[g])))
    berr = np.max(np.abs(sets[0].bound() - bounds[0]) / bounds[0])
    assert berr <= 1e-8
    ov = np.stack(oracle_vals, axis=1)
    want = merit_rule(ov, lb, ub, bounds[0])
    got = cp(Xc)
    # rows whose every constraint value is clear of its finite bounds: the two computations classify them alike
    clear = np.ones(ov.shape[0], dtype=bool)
    for j in range(1, J + 1):
        c, margin = ov[:, j, :], 1e-7 * (np.abs(ov[:, j, :]) + s_y[j])
        for bnd in (lb[j - 1], ub[j - 1]):
            if np.isfinite(bnd):
                clear &= np.all(np.abs(c - bnd) > margin, axis=1)
    err = np.max(np.abs(got[clear] - want[clear]) / (np.abs(want[clear]) + s_y[0]))
    print(f"J={J} q={q}: B_p rel err {berr:.1e}, merit err {err:.1e}, {np.sum(~clear)} rows inside the margin")
    assert err <= 1e-8
    assert np.sum(~clear) <= 5


def _chunk_rows():
    import torch

    return 8 * 128 * torch.cuda.get_device_properties(0).multi_processor_count


def _np_select(ys, k):
    return int(np.argmin(ys)), np.argsort(ys, kind="stable")[:k]


def _check_selection(cp, Xc, k):
    ys = -cp(Xc)
    idx, val, tops = cp.argmin_topk(Xc, k)
    for p in range(cp.n_paths):
        ri, rtop = _np_select(ys[:, p], k)
        assert idx[p] == ri and val[p] == ys[ri, p]
        assert list(tops[p]) == list(rtop)
    return ys, idx


# (chunks of the streamed upload, extra rows, J, q): one launch; two chunks with a ragged tail; four chunks
@pytest.mark.parametrize("chunks,extra,J,q", [(0, 5000, 2, 3), (1, 77, 1, 1), (3, 5, 2, 16)])
def test_selection_equals_numpy(bo, chunks, extra, J, q):
    X, ys, gps, rs = _fit_sets(bo, J + 1, n=400, d=4, seed=chunks + 3)
    m = chunks * _chunk_rows() + extra
    Xc = rs.uniform(size=(m, 4))
    Xc[m // 2] = Xc[3]  # exact ties across tiles and chunks
    Xc[m - 1] = Xc[3]
    if m > _chunk_rows():
        Xc[_chunk_rows()] = Xc[3]
    cp, *_ = _constrained(bo, gps, q, 1024, 2, Xb=Xc[:5000])
    _check_selection(cp, Xc, 10)


def test_ties_at_the_winner(bo):
    X, ys, gps, rs = _fit_sets(bo, 3, n=200, d=2, seed=4)
    Xc = rs.uniform(size=(2 * _chunk_rows() + 300, 2))
    cp, *_ = _constrained(bo, gps, 2, 512, 3, Xb=Xc[:4000])
    win = cp.argmin_topk(Xc, 1)[0]
    for p in range(2):  # copies of every path's winner in later tiles and chunks
        for at in (5, 129, _chunk_rows() + 1, len(Xc) - 1):
            if at != win[p]:
                Xc[at] = Xc[win[p]]
    _check_selection(cp, Xc, 12)


def test_no_feasible_candidate_picks_the_least_violation(bo):
    X, ys, gps, rs = _fit_sets(bo, 3, n=300, d=3, seed=5)
    Xc = rs.uniform(size=(_chunk_rows() + 999, 3))
    cp, sets, lb, ub = _constrained(bo, gps, 3, 512, 4, lb=[50.0, -np.inf], ub=[60.0, -50.0])
    raw = cp.raw(Xc)
    viol = np.maximum(0.0, lb[0] - raw[:, 1, :]) + np.maximum(0.0, raw[:, 2, :] - ub[1])
    assert np.all(viol > 0)
    ys, idx = _check_selection(cp, Xc, 10)
    for p in range(3):
        assert idx[p] == np.argmin(viol[:, p])


def test_a_feasible_row_beats_an_infeasible_row_of_larger_value(bo):
    X, ys, gps, rs = _fit_sets(bo, 1, n=300, d=3, seed=6)
    Xc = rs.uniform(size=(20_000, 3))
    from bayesianoptimization_b200.paths import ConstrainedPaths

    target = gps[0].sample_paths(2, 512, random_state=8)
    same = gps[0].sample_paths(2, 512, random_state=8)  # the constraint IS the target path: f <= median
    med = float(np.median(target(Xc)[:, 0]))
    cp = ConstrainedPaths(target, [same], [-np.inf], [med])
    _, idx = _check_selection(cp, Xc, 10)
    raw = cp.raw(Xc)
    f, feas = raw[:, 0, 0], raw[:, 1, 0] <= med
    w = idx[0]
    assert feas[w] and f[w] == f[feas].max()
    assert np.any(~feas & (f > f[w]))  # rows of larger value exist, and are infeasible


def test_philox_source_equals_host_evaluation_of_its_rows(bo):
    from bayesianoptimization_b200 import _lib as B

    X, ys, gps, _ = _fit_sets(bo, 3, n=200, d=3, seed=7)
    bounds = np.array([[-1.0, 1.0], [0.0, 2.0], [0.5, 0.75]])
    lo, hi = np.ascontiguousarray(bounds[:, 0]), np.ascontiguousarray(bounds[:, 1])
    m, k, seed, base = _chunk_rows() + 40_000, 8, 0x1234_5678_9ABC, 1000  # two Philox chunks
    gidx = np.arange(base, base + m, dtype=np.int64)
    rows = np.empty((m, 3))
    B.check(B.lib().b200bo_philox_rows(0, seed, B.as_dp(lo), B.as_dp(hi), 3, gidx.ctypes.data_as(C.POINTER(C.c_int64)),
                                       m, B.as_dp(rows)))
    cp, *_ = _constrained(bo, gps, 3, 512, 3, Xb=rows[:5000])
    idx, val, bx, ti, tx = cp.argmin_topk_philox(seed, bounds, m, k, index_base=base)
    ys = -cp(rows)
    for j in range(3):
        ri, rtop = _np_select(ys[:, j], k)
        assert idx[j] == base + ri and val[j] == ys[ri, j]
        assert list(ti[j]) == list(base + rtop)
        assert np.array_equal(bx[j], rows[ri]) and np.array_equal(tx[j], rows[rtop])


def test_nonfinite_candidates_are_rejected(bo):
    X, ys, gps, rs = _fit_sets(bo, 2, n=100, d=2, seed=8)
    Xc = rs.uniform(size=(500, 2))
    cp, *_ = _constrained(bo, gps, 1, 128, 1, lb=[-np.inf], ub=[0.0])
    Xc[77, 1] = np.nan
    for call in (lambda: cp(Xc), lambda: cp.argmin_topk(Xc, 3)):
        with pytest.raises(ValueError, match="NaN or infinity"):
            call()


def test_suggest_equals_host_constrained_thompson_sampling_on_the_same_draws(bo, ref):
    """End to end at fixed theta: device ConstrainedThompsonSampling.suggest vs a host acquisition whose closure is
    the restated rule on the same draws (target, then the constraint, from the suggest RandomState)."""
    from types import SimpleNamespace

    from bayes_opt.target_space import TargetSpace

    pb = {"x": (-2.0, 2.0), "y": (-1.0, 3.0)}
    space = TargetSpace(lambda x, y: -(x**2) - (y - 1) ** 2 + 1, pb)
    rs0 = np.random.RandomState(21)
    for _ in range(12):
        space.probe(space.random_sample(random_state=rs0))
    X = space.params
    cy = X[:, 0] + X[:, 1]
    L, ls, alpha, ub = 1024, 0.9, 1e-6, 1.5
    mk = lambda y: bo.B200GaussianProcessRegressor(kernel=Matern(ls, nu=2.5), alpha=alpha,  # noqa: E731
                                                   normalize_y=True, optimizer=None).fit(X, y)
    gp, cgp = mk(space.target), mk(cy)
    cons = SimpleNamespace(model=[cgp], lb=np.array([-np.inf]), ub=np.array([ub]))
    stage = {}

    class DeviceCTS(bo.ConstrainedThompsonSampling):
        def _get_acq(self, gp, constraint=None):
            return super()._get_acq(gp, constraint=cons)

        def _random_sample_minimize(self, acq, sp, random_state, n_random, n_x_seeds=0):
            out = super()._random_sample_minimize(acq, sp, random_state, n_random, n_x_seeds)
            stage["dev"] = out[0]
            return out

    class HostCTS(ref.acquisition.AcquisitionFunction):
        def base_acq(self, *a, **k):
            raise NotImplementedError

        def suggest(self, gp, target_space, n_random=10_000, n_smart=10, fit_gp=True, random_state=None):
            self.rs = random_state
            return super().suggest(gp, target_space, n_random, n_smart, fit_gp, random_state)

        def _get_acq(self, gp, constraint=None):
            n = len(cy)
            dt, dc = T.draws(self.rs, 1, L, 2, 2.5, n, alpha), T.draws(self.rs, 1, L, 2, 2.5, n, alpha)
            f = T.make_paths(X, space.target, dt, length_scale=ls, alpha=alpha)
            c = T.make_paths(X, cy, dc, length_scale=ls, alpha=alpha)
            bound = _restated_bound(X, space.target, dt, T.KIND_MATERN, 2.5, ls, 1.0, alpha)

            def acq(x):
                x = np.asarray(x).reshape(-1, 2)
                return -merit_rule(np.stack([f(x), c(x)], axis=1), [-np.inf], [ub], bound)[:, 0]

            return acq

        def _random_sample_minimize(self, acq, sp, random_state, n_random, n_x_seeds=0):
            out = super()._random_sample_minimize(acq, sp, random_state, n_random, n_x_seeds)
            stage["host"] = out[0]
            return out

    ra, rb = np.random.RandomState(5), np.random.RandomState(5)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        xd = DeviceCTS(n_features=L).suggest(gp, space, n_random=5000, n_smart=5, fit_gp=False, random_state=ra)
        xh = HostCTS().suggest(gp, space, n_random=5000, n_smart=5, fit_gp=False, random_state=rb)
    assert np.array_equal(stage["dev"], stage["host"])
    sa, sb = ra.get_state(), rb.get_state()
    assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]
    assert np.allclose(xd, xh, rtol=0, atol=1e-3 * 4)  # optimiser tolerance on a span of 4


def _target(x, y):
    return -(x**2) - (y - 1) ** 2 + 1


def _cfun(x, y):
    return (x - 3.5) ** 2 + (y - 2.0) ** 2


def _optimizer(bo, ref, seed=5):
    from scipy.optimize import NonlinearConstraint

    opt = ref.BayesianOptimization(f=_target, pbounds={"x": (2.0, 4.0), "y": (-3.0, 3.0)},
                                   constraint=NonlinearConstraint(_cfun, -np.inf, 0.8**2),
                                   acquisition_function=bo.ConstrainedThompsonSampling(n_features=1024),
                                   random_state=seed, verbose=0)
    return bo.enable(opt)


def test_constrained_thompson_sampling_through_the_reference_driver(bo, ref, tmp_path):
    a, b = _optimizer(bo, ref), _optimizer(bo, ref)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        a.maximize(init_points=3, n_iter=10)
        b.maximize(init_points=3, n_iter=10)
    assert len(a.space) == 13 and isinstance(a._acquisition_function, bo.ConstrainedThompsonSampling)
    assert np.array_equal(a.space.params, b.space.params)  # suggestion1 == suggestion2, every step
    path = tmp_path / "state.json"
    a.save_state(path)
    c = _optimizer(bo, ref)
    c.load_state(path)
    assert c._acquisition_function.n_features == 1024
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sa, sc = a.suggest(), c.suggest()
    assert sa == sc


def test_suggests_without_a_feasible_point_where_ei_cannot(bo, ref):
    from bayes_opt.exception import NoValidPointRegisteredError

    opt = _optimizer(bo, ref, seed=11)
    for x, y in [(2.2, -2.5), (3.0, -1.0), (2.5, 0.5)]:  # all far outside the disc around (3.5, 2)
        opt.probe({"x": x, "y": y}, lazy=False)
    assert not opt.space.mask.any()
    with pytest.raises(NoValidPointRegisteredError):
        bo.ExpectedImprovement(xi=0.01).suggest(opt._gp, opt.space, random_state=np.random.RandomState(1))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt.maximize(init_points=0, n_iter=15)
    assert len(opt.space) == 18
    n_feasible = int(opt.space.mask.sum())
    print(f"feasible points registered in 15 iterations: {n_feasible}")
    assert n_feasible >= 1

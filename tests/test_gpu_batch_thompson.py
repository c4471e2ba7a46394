"""Batch Thompson sampling on the device: the row-mode evaluation (b200bo_paths_eval_rows / b200bo_cpaths_eval_rows)
is bit-equal to the columns of the full evaluation; suggest_batch(q=1) is suggest; for q > 1 every point is what a
per-path restatement (numpy ranking of -paths(X)[:, p] over the same candidates, SciPy L-BFGS-B on that path alone)
finds; and b200.suggest_batch drives a live BayesianOptimization."""
import ctypes as C
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
from scipy.optimize import minimize
from sklearn.gaussian_process.kernels import RBF, Matern

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _kernel(nu, ls):
    return RBF(ls) if nu == np.inf else Matern(ls, nu=nu)


def _gp(bo, X, y, nu=2.5, ls=0.5, alpha=1e-6):
    return bo.B200GaussianProcessRegressor(kernel=_kernel(nu, ls), alpha=alpha, normalize_y=True,
                                           optimizer=None).fit(X, y)


def _data(n, d, seed, g=0):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    y = np.sin(3 * X.sum(1) + g) + 0.3 * g * X[:, 0] + 0.05 * rs.randn(n)
    return X, y, rs


def _check_rows(p, Xc, rs):
    full = p(Xc)
    q, m = p.n_paths, len(Xc)
    pidx = rs.randint(0, q, m)
    assert np.array_equal(p.eval_rows(Xc, pidx), full[np.arange(m), pidx])
    for j in range(q):  # one path for every row, and a single row (against the full evaluation of the same batch:
        # the reference's categorical one-hot transform depends on the batch it is given)
        assert np.array_equal(p.eval_rows(Xc, np.full(m, j)), full[:, j])
        assert np.array_equal(p.eval_rows(Xc[5:6], [j]), p(Xc[5:6])[:, j])


# (q, covariance nu, d): every register class of the full evaluation (QT = 1, 4, 16), every covariance code, d even,
# odd and > 16
ROWS = [(1, 2.5, 2), (4, 1.5, 3), (16, 0.5, 17), (16, np.inf, 4), (4, np.inf, 33), (1, 0.5, 5), (4, 2.5, 18),
        (16, 1.5, 1), (3, 2.5, 7)]


@pytest.mark.parametrize("q,nu,d", ROWS)
def test_eval_rows_is_bit_equal_to_the_columns(bo, q, nu, d):
    X, y, rs = _data(300, d, q * 100 + d)
    gp = _gp(bo, X, y, nu=nu, ls=0.4 * np.sqrt(d))
    p = gp.sample_paths(q, 700, random_state=3)
    Xc = rs.uniform(-0.1, 1.1, size=(1500, d))  # several tiles of 128, a ragged tail
    Xc[:4] = X[:4]
    _check_rows(p, Xc, rs)


@pytest.mark.parametrize("transform", ["int", "categorical"])
def test_eval_rows_with_kernel_transforms(bo, ref, transform):
    """np.round on the device (int) and the host-side one-hot (categorical) reach row mode as they reach the full
    evaluation."""
    from bayes_opt.parameter import wrap_kernel
    from bayes_opt.target_space import TargetSpace

    pb = {"x": (0.0, 1.0), "n": (0, 5, int)} if transform == "int" else {"x": (0.0, 1.0), "c": ["a", "b", "c"]}
    space = TargetSpace(None, pb)
    rs = np.random.RandomState(4)
    X = space.random_sample(200, random_state=rs)
    y = np.sin(3 * X.sum(1))
    gp = bo.B200GaussianProcessRegressor(kernel=wrap_kernel(Matern(0.8, nu=2.5), space.kernel_transform), alpha=1e-4,
                                         normalize_y=True, optimizer=None).fit(X, y)
    p = gp.sample_paths(4, 512, random_state=5)
    _check_rows(p, space.random_sample(900, random_state=rs), rs)


@pytest.mark.parametrize("J,q", [(1, 4), (3, 16), (3, 1), (1, 7)])
def test_constrained_eval_rows_is_bit_equal_to_the_columns(bo, J, q):
    from bayesianoptimization_b200.paths import ConstrainedPaths

    X, _, rs = _data(250, 3, J * 10 + q)
    gps = [_gp(bo, X, _data(250, 3, J * 10 + q, g)[1], nu=[2.5, 1.5, 0.5, np.inf][g % 4]) for g in range(J + 1)]
    sets = [g.sample_paths(q, 512, random_state=11 + i) for i, g in enumerate(gps)]
    Xc = rs.uniform(-0.1, 1.1, size=(2000, 3))
    lb = np.array([np.quantile(s(Xc), 0.2) for s in sets[1:]])  # both tiers present
    cp = ConstrainedPaths(sets[0], sets[1:], lb, np.full(J, np.inf))
    merit = cp(Xc)
    assert 0.02 < np.mean(merit == cp.raw(Xc)[:, 0, :]) < 0.98
    _check_rows(cp, Xc, rs)


def test_out_of_range_path_idx_is_rejected(bo):
    from bayesianoptimization_b200 import _lib as B
    from bayesianoptimization_b200.paths import ConstrainedPaths

    X, y, rs = _data(100, 2, 1)
    gp = _gp(bo, X, y)
    p = gp.sample_paths(3, 256, random_state=1)
    Xc = B.c_f64(rs.uniform(size=(10, 2)))
    for bad in (3, -1, 2**40, 16):
        pidx = np.zeros(10, dtype=np.int64)
        pidx[7] = bad
        with pytest.raises(ValueError, match="out of range"):
            p.eval_rows(Xc, pidx)
    raw = np.array([0, 1, 2, 3, 0, 0, 0, 0, 0, 0], dtype=np.int32)  # straight through the ABI
    out = np.empty(10)
    rc = B.lib().b200bo_paths_eval_rows(p._handle.ptr, B.as_dp(Xc), raw.ctypes.data_as(C.POINTER(C.c_int32)), 10,
                                        B.as_dp(out))
    assert rc == B.ERR_ARG
    cp = ConstrainedPaths(p, [gp.sample_paths(3, 256, random_state=2)], [0.0], [1.0])
    rc = B.lib().b200bo_cpaths_eval_rows(*cp._args(), B.as_dp(Xc), raw.ctypes.data_as(C.POINTER(C.c_int32)), 10,
                                         B.as_dp(out))
    assert rc == B.ERR_ARG
    with pytest.raises(ValueError, match="out of range"):
        cp.eval_rows(Xc, raw)
    assert np.array_equal(p.eval_rows(Xc, np.full(10, 2)), p(Xc)[:, 2])  # the handle still works


# ---- suggest_batch ----------------------------------------------------------------------------------------------
PB = {"x": (-2.0, 2.0), "y": (-1.0, 3.0), "z": (0.0, 1.0)}


def _f(x, y, z):
    return -(x**2) - (y - 1) ** 2 + np.sin(4 * z) + 1


def _space(ref, n=14, constraint=False):
    from bayes_opt.target_space import TargetSpace

    space = TargetSpace(_f, PB)
    rs = np.random.RandomState(21)
    for _ in range(n):
        space.probe(space.random_sample(random_state=rs))
    return space


def _with_infeasible_constraint(bo, space):
    """A constraint GP c(x) = x + y with the bound c >= 4.5: no registered point is feasible."""
    c = space.params[:, 0] + space.params[:, 1]
    assert np.all(c < 4.5)
    cgp = _gp(bo, space.params, c, ls=1.0)
    space._constraint = SimpleNamespace(model=[cgp], lb=np.array([4.5]), ub=np.array([np.inf]))
    return cgp


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
@pytest.mark.parametrize("constrained", [False, True])
def test_q1_is_suggest_bit_for_bit(bo, ref, source, constrained):
    space = _space(ref)
    gp = _gp(bo, space.params, space.target, ls=0.9)
    if constrained:
        _with_infeasible_constraint(bo, space)
    cls = bo.ConstrainedThompsonSampling if constrained else bo.ThompsonSampling
    a, b = cls(n_features=1024), cls(n_features=1024)
    a.b200_candidate_source = b.b200_candidate_source = source
    ra, rb = np.random.RandomState(5), np.random.RandomState(5)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        xa = a.suggest_batch(gp, space, 1, n_random=20_000, n_smart=6, fit_gp=False, random_state=ra)
        xb = b.suggest(gp, space, n_random=20_000, n_smart=6, fit_gp=False, random_state=rb)
    assert xa.shape == (1, 3) and np.array_equal(xa[0], xb)
    sa, sb = ra.get_state(), rb.get_state()
    assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


def _restated(bo, gp, space, rs, q, L, n, k, source, cgp=None):
    """The per-path pipeline restated on the same draws: numpy ranks -paths(X)[:, p] over the same candidates, SciPy
    refines every seed on that single path, the reference's rule picks."""
    from bayesianoptimization_b200 import _lib as B
    from bayesianoptimization_b200.acquisition import _philox_seed
    from bayesianoptimization_b200.paths import ConstrainedPaths

    paths = gp.sample_paths(q, L, random_state=rs)
    if cgp is not None:
        c = space.constraint
        paths = ConstrainedPaths(paths, [cgp.sample_paths(q, L, random_state=rs)], c.lb, c.ub)
    if source == "device_philox":
        seed = _philox_seed(rs)
        lo, hi = B.c_f64(space.bounds[:, 0]), B.c_f64(space.bounds[:, 1])
        gidx = np.arange(n, dtype=np.int64)
        X = np.empty((n, 3))
        B.check(B.lib().b200bo_philox_rows(0, seed, B.as_dp(lo), B.as_dp(hi), 3,
                                           gidx.ctypes.data_as(C.POINTER(C.c_int64)), n, B.as_dp(X)))
    else:
        X = space.random_sample(n, random_state=rs)
    ys = -paths(X)
    out = []
    for p in range(q):
        i = int(np.argmin(ys[:, p]))
        best_x, best_f = X[i], ys[i, p]
        fun = lambda x, p=p: -paths(np.asarray(x).reshape(1, -1))[:, p]  # noqa: E731
        runs = [minimize(fun, s, bounds=space.bounds, method="L-BFGS-B")
                for s in X[np.argsort(ys[:, p], kind="stable")[:k]]]
        runs = [r for r in runs if r.success]
        if runs:
            r = min(runs, key=lambda r: float(np.squeeze(r.fun)))
            if best_f > np.squeeze(r.fun):
                best_x = np.clip(r.x, space.bounds[:, 0], space.bounds[:, 1])
        out.append(best_x)
    return np.array(out), ys


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
@pytest.mark.parametrize("q", [4, 16])
def test_each_point_matches_the_per_path_restatement(bo, ref, q, source):
    space = _space(ref)
    gp = _gp(bo, space.params, space.target, ls=0.9)
    ts = bo.ThompsonSampling(n_features=1024)
    ts.b200_candidate_source = source
    ra, rb = np.random.RandomState(7), np.random.RandomState(7)
    n, k = 30_000, 5
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        X = ts.suggest_batch(gp, space, q, n_random=n, n_smart=k, fit_gp=False, random_state=ra)
        want, _ = _restated(bo, gp, space, rb, q, 1024, n, k, source)
    assert X.shape == (q, 3)
    span = space.bounds[:, 1] - space.bounds[:, 0]
    assert np.all(np.abs(X - want) <= 1e-3 * span), np.abs(X - want).max(axis=0)
    sa, sb = ra.get_state(), rb.get_state()
    assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]
    assert len({x.tobytes() for x in X}) == q


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
def test_constrained_points_match_the_restatement_without_a_feasible_point(bo, ref, source):
    space = _space(ref)
    gp = _gp(bo, space.params, space.target, ls=0.9)
    cgp = _with_infeasible_constraint(bo, space)
    ts = bo.ConstrainedThompsonSampling(n_features=1024)
    ts.b200_candidate_source = source
    ra, rb = np.random.RandomState(8), np.random.RandomState(8)
    q, n, k = 8, 30_000, 5
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        X = ts.suggest_batch(gp, space, q, n_random=n, n_smart=k, fit_gp=False, random_state=ra)
        want, _ = _restated(bo, gp, space, rb, q, 1024, n, k, source, cgp=cgp)
    span = space.bounds[:, 1] - space.bounds[:, 0]
    assert np.all(np.abs(X - want) <= 1e-3 * span), np.abs(X - want).max(axis=0)
    sa, sb = ra.get_state(), rb.get_state()
    assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


def _live(ref, bo, tmp_path, f, pb, seed):
    def mk():
        opt = ref.BayesianOptimization(f=f, pbounds=pb, acquisition_function=bo.ThompsonSampling(n_features=1024),
                                       random_state=seed, verbose=0)
        return bo.enable(opt)

    a, restored = mk(), None
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        first = bo.suggest_batch(a, 4)  # empty space: random_sample(4)
        for p in first:
            a.register(params=p, target=f(**p))
        for rnd in range(5):
            batch = bo.suggest_batch(a, 4)
            assert len(batch) == 4 and all(set(p) == set(pb) for p in batch)
            if restored is not None:  # the optimizer restored from save_state proposes the same batch
                assert bo.suggest_batch(restored, 4) == batch
                restored = None
            for p in batch:
                a.register(params=p, target=f(**p))  # NotUniqueError on a duplicate
            if rnd == 1:
                path = tmp_path / "state.json"
                a.save_state(path)
                restored = mk()
                restored.load_state(path)
    assert len(a.space) == 24
    return a


def test_live_optimizer_continuous(bo, ref, tmp_path):
    a = _live(ref, bo, tmp_path, _f, PB, 3)
    assert isinstance(a._acquisition_function, bo.ThompsonSampling) and a._acquisition_function.i == 5


def test_live_optimizer_int_and_categorical(bo, ref, tmp_path):
    def f(x, k, c):
        return -((x - 2.0) ** 2) - 0.3 * (k - 3) ** 2 + {"a": 0.0, "b": 1.0, "c": -0.5}[c]

    a = _live(ref, bo, tmp_path, f, {"x": (0.0, 5.0), "k": (0, 6, int), "c": ["a", "b", "c"]}, 11)
    assert all(isinstance(p["c"], str) for p in [a.space.array_to_params(x) for x in a.space.params])

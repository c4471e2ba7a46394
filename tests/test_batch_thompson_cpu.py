"""Batch Thompson sampling without a GPU: the host logic of ThompsonSampling.suggest_batch and b200.suggest_batch over a
stub that keeps the PosteriorPaths interface (numpy paths whose shape comes from the draws of draw_path_inputs, so
they consume the RandomState exactly as device paths do).  Checked: the order in which the RandomState is consumed
(host and Philox candidates, with and without constraints), q validation, the duplicate rule, the empty-space branch
of b200.suggest_batch and its TypeError for other acquisition functions."""
import ctypes as C
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

PB = {"x": (0.0, 1.0), "y": (-1.0, 2.0)}
L_FEAT, NU = 8, 2.5


@pytest.fixture(scope="module")
def bo():
    import __graft_entry__ as g

    g.build()
    import bayesianoptimization_b200 as bo

    return bo


class StubPaths:
    """q smooth paths f_p(x) = -|x - c_p|^2 + h_p with c_p, h_p taken from the weights w of draw_path_inputs.  Records
    the candidate sets and Philox seeds it is asked to rank."""

    def __init__(self, rs, q, n, lo, hi, scale=1.0):
        from bayesianoptimization_b200.paths import draw_path_inputs

        d = len(lo)
        _, _, w, _ = draw_path_inputs(rs, q, L_FEAT, d, NU, n, 1e-6)
        self.c = lo + (hi - lo) * (0.5 + 0.4 * np.tanh(w[:d].T))  # (q, d), inside the box
        self.h = scale * w[d]
        self.n_paths, self.dim, self.device, self.devices = q, d, 0, [0]
        self._xform = ("device", None)
        self._handle = SimpleNamespace(ptr=C.c_void_p(0))
        self.ranked, self.seeds = [], []

    def __call__(self, X):
        X = np.asarray(X, dtype=np.float64).reshape(-1, self.dim)
        return -((X[:, None, :] - self.c[None]) ** 2).sum(-1) + self.h

    def eval_rows(self, X, path_idx):
        X = np.asarray(X, dtype=np.float64).reshape(-1, self.dim)
        return self(X)[np.arange(len(X)), np.asarray(path_idx)]

    def _select(self, X, k):
        ys = -self(X)
        order = [np.argsort(ys[:, p], kind="stable")[:k] for p in range(self.n_paths)]
        return ys.argmin(axis=0), ys.min(axis=0), order

    def argmin_topk(self, X, k):
        self.ranked.append(np.array(X))
        return self._select(X, k)

    def argmin_topk_philox(self, seed, bounds, m, k, index_base=0):
        self.seeds.append(seed)
        b = np.asarray(bounds)
        X = np.random.RandomState(seed % 2**32).uniform(b[:, 0], b[:, 1], (m, self.dim))
        idx, vals, order = self._select(X, k)
        return idx, vals, X[idx], [o + index_base for o in order], [X[o] for o in order]

    def bound(self):
        return np.abs(self.h) + 10.0


class StubConstrained(StubPaths):
    """ConstrainedPaths' interface over stub sets: merit = f if every c_j in [lb_j, ub_j], else -T (1 + viol)."""

    def __init__(self, target, constraints, lb, ub):
        self.t, self.cs, self.lb, self.ub = target, constraints, np.asarray(lb), np.asarray(ub)
        self.n_paths, self.dim, self.device, self.devices = target.n_paths, target.dim, 0, [0]
        self._xform = target._xform
        self.ranked, self.seeds = target.ranked, target.seeds

    def __call__(self, X):
        f = self.t(X)
        viol = sum(np.maximum(0, lb - c(X)) + np.maximum(0, c(X) - ub) for c, lb, ub in zip(self.cs, self.lb, self.ub))
        return np.where(viol == 0, f, -(2 * self.t.bound() + 1) * (1 + viol))


def _stub_gp(bo, draws, scale=1.0):
    """A B200GaussianProcessRegressor whose sample_paths draws from the RandomState like the device's and returns a
    StubPaths.  ``draws`` records every call."""
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=NU), optimizer=None)
    lo, hi = np.array([v[0] for v in PB.values()]), np.array([v[1] for v in PB.values()])

    def sample_paths(n_paths=1, n_features=4096, random_state=None):
        assert n_features == L_FEAT
        draws.append(n_paths)
        return StubPaths(random_state, n_paths, 5, lo, hi, scale)

    gp.sample_paths = sample_paths
    return gp


def _space(ref, n=5, seed=1):
    from bayes_opt.target_space import TargetSpace

    space = TargetSpace(None, PB)
    rs = np.random.RandomState(seed)
    for _ in range(n):
        space.register(space.random_sample(random_state=rs), float(rs.uniform()))
    return space


def _same_state(a, b):
    sa, sb = a.get_state(), b.get_state()
    return np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
@pytest.mark.parametrize("n_constraints", [0, 2])
@pytest.mark.parametrize("n_smart", [0, 3, 65])
def test_random_state_is_consumed_in_the_documented_order(bo, ref, monkeypatch, source, n_constraints, n_smart):
    """paths of the target, then q paths per constraint GP in constraint order, then ONE candidate set (or one Philox
    seed) shared by every path - and nothing more on a continuous space.  n_smart = 65 exceeds the device's top-k:
    host candidates, numpy selection."""
    import bayesianoptimization_b200.paths as P
    from bayesianoptimization_b200.acquisition import _philox_seed
    from bayesianoptimization_b200.paths import draw_path_inputs

    monkeypatch.setattr(P, "ConstrainedPaths", StubConstrained)
    q, n_random = 3, 400
    draws = []
    gp = _stub_gp(bo, draws)
    cgps = [_stub_gp(bo, draws) for _ in range(n_constraints)]
    space = _space(ref)
    if n_constraints:
        space._constraint = SimpleNamespace(model=cgps, lb=np.full(n_constraints, -10.0), ub=np.full(n_constraints, 10.0))
    ts = (bo.ConstrainedThompsonSampling if n_constraints else bo.ThompsonSampling)(n_features=L_FEAT)
    ts.b200_candidate_source = source
    ra, rb = np.random.RandomState(9), np.random.RandomState(9)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        X = ts.suggest_batch(gp, space, q, n_random=n_random, n_smart=n_smart, fit_gp=False, random_state=ra)
    assert X.shape == (q, 2) and ts.i == 1
    assert draws == [q] * (1 + n_constraints)  # one sample_paths(q) per GP
    for _ in range(1 + n_constraints):
        draw_path_inputs(rb, q, L_FEAT, 2, NU, 5, 1e-6)
    target = LAST[0]  # the target's stub: a constrained stub records on it too
    if source == "device_philox" and n_smart <= 64:
        seed = _philox_seed(rb)
        assert len(target.ranked) == 0 and target.seeds == [seed]
    else:
        want = space.random_sample(max(n_random, n_smart), random_state=rb)
        if n_smart <= 64:  # (beyond, the numpy selection evaluates the same rows through __call__)
            assert len(target.ranked) == 1 and np.array_equal(target.ranked[0], want)
    assert _same_state(ra, rb)
    if n_smart and not n_constraints:
        # every path's answer is its own maximiser: the refinement evaluated each run on its own path
        assert np.allclose(X, target.c, atol=1e-4)


LAST = []


@pytest.fixture(autouse=True)
def _track_paths(monkeypatch):
    """Keep the first StubPaths of a test (the target's) reachable as LAST[0]."""
    LAST.clear()
    orig = StubPaths.__init__

    def init(self, *a, **k):
        orig(self, *a, **k)
        if not LAST:
            LAST.append(self)

    monkeypatch.setattr(StubPaths, "__init__", init)


def test_q1_equals_suggest(bo, ref):
    """q = 1 through suggest_batch: the point of suggest, bit for bit, and the same RandomState after."""
    space = _space(ref, seed=4)
    ra, rb = np.random.RandomState(3), np.random.RandomState(3)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        xa = bo.ThompsonSampling(n_features=L_FEAT).suggest_batch(_stub_gp(bo, []), space, 1, n_random=300, n_smart=4,
                                                                  fit_gp=False, random_state=ra)
        xb = bo.ThompsonSampling(n_features=L_FEAT).suggest(_stub_gp(bo, []), space, n_random=300, n_smart=4,
                                                            fit_gp=False, random_state=rb)
    assert xa.shape == (1, 2) and np.array_equal(xa[0], xb)
    assert _same_state(ra, rb)


def test_mixed_integer_space_takes_the_reference_branch_per_path(bo, ref):
    """With an int parameter the refinement is the reference's differential evolution, per path, in path order:
    q = 1 matches suggest bit for bit and q = 3 gives one point per path."""
    from bayes_opt.target_space import TargetSpace

    pb = {"x": (0.0, 1.0), "y": (-1, 2, int)}
    space = TargetSpace(None, pb)
    rs = np.random.RandomState(2)
    for _ in range(4):
        space.register(space.random_sample(random_state=rs), float(rs.uniform()))
    ra, rb = np.random.RandomState(6), np.random.RandomState(6)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        xa = bo.ThompsonSampling(n_features=L_FEAT).suggest_batch(_stub_gp(bo, []), space, 1, n_random=200, n_smart=3,
                                                                  fit_gp=False, random_state=ra)
        xb = bo.ThompsonSampling(n_features=L_FEAT).suggest(_stub_gp(bo, []), space, n_random=200, n_smart=3,
                                                            fit_gp=False, random_state=rb)
        assert np.array_equal(xa[0], xb) and _same_state(ra, rb)
        X = bo.ThompsonSampling(n_features=L_FEAT).suggest_batch(_stub_gp(bo, []), space, 3, n_random=200, n_smart=3,
                                                                 fit_gp=False, random_state=ra)
    assert X.shape == (3, 2) and np.all((X >= space.bounds[:, 0]) & (X <= space.bounds[:, 1]))


@pytest.mark.parametrize("bad", [0, 17, -1, 1.5, 2.0, True, False, "3", None])
def test_q_validation(bo, ref, bad):
    ts = bo.ThompsonSampling(n_features=L_FEAT)
    rs = np.random.RandomState(0)
    before = rs.get_state()
    with pytest.raises(ValueError, match="q must be"):
        ts.suggest_batch(_stub_gp(bo, []), _space(ref), bad, fit_gp=False, random_state=rs)
    after = rs.get_state()
    assert np.array_equal(before[1], after[1]) and ts.i == 0  # refused before anything is drawn or counted
    opt = ref.BayesianOptimization(f=None, pbounds=PB, acquisition_function=ts, verbose=0)
    with pytest.raises(ValueError, match="q must be"):
        bo.suggest_batch(opt, bad)
    assert bo.ThompsonSampling.suggest_batch is bo.ConstrainedThompsonSampling.suggest_batch


def test_q_accepts_numpy_integers(bo, ref):
    X = bo.ThompsonSampling(n_features=L_FEAT).suggest_batch(_stub_gp(bo, []), _space(ref), np.int64(2), n_random=50,
                                                             n_smart=0, fit_gp=False, random_state=1)
    assert X.shape == (2, 2)


def _a(*v):
    return np.array(v, dtype=np.float64)


def test_duplicate_rule_on_synthetic_top_k_lists():
    from bayesianoptimization_b200.acquisition import distinct_picks

    a, b, c, d = _a(0, 0), _a(1, 0), _a(2, 0), _a(3, 0)
    # distinct picks are kept as they are
    out = distinct_picks([a, b, c], [[a], [b], [c]])
    assert all(np.array_equal(x, y) for x, y in zip(out, [a, b, c]))
    # path 1 repeats path 0: its best top-k row not taken (a is taken, c is not)
    out = distinct_picks([a, a], [[a, b], [a, c, d]])
    assert np.array_equal(out[1], c)
    # path 2 repeats; its top-k holds only taken rows and then d
    out = distinct_picks([a, b, a], [[a], [b], [a, b, d]])
    assert np.array_equal(out[2], d)
    # nothing left: the duplicate stays
    out = distinct_picks([a, a], [[a], [a]])
    assert np.array_equal(out[1], a)
    out = distinct_picks([a, a], [[a], []])
    assert np.array_equal(out[1], a)
    # a replacement counts as taken for later paths; earlier paths are never changed
    out = distinct_picks([a, a, a], [[a, b], [a, b, c], [b, a, c, d]])
    assert [tuple(x) for x in out] == [tuple(a), tuple(b), tuple(c)]
    # bit-equality: -0.0 and 0.0 are different points to the rule
    out = distinct_picks([_a(0.0, 1), _a(-0.0, 1)], [[], []])
    assert np.signbit(out[1][0])


def test_duplicates_of_the_random_stage_are_replaced_in_suggest_batch(bo, ref):
    """Identical paths (h = 0, same centre for all) and no refinement: every path wins on the same candidate, so paths
    1.. take the next rows of their own top-k."""
    space = _space(ref)

    def same_paths(n_paths=1, n_features=4096, random_state=None):
        p = StubPaths(random_state, n_paths, 5, np.zeros(2), np.ones(2), scale=0.0)
        p.c[:] = p.c[0]
        return p

    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=NU), optimizer=None)
    gp.sample_paths = same_paths
    X = bo.ThompsonSampling(n_features=L_FEAT).suggest_batch(gp, space, 4, n_random=500, n_smart=0, fit_gp=False,
                                                             random_state=5)
    assert all(np.array_equal(X[0], x) for x in X)  # n_smart = 0: no top-k to draw replacements from
    Y = bo.ThompsonSampling(n_features=L_FEAT).suggest_batch(gp, space, 4, n_random=500, n_smart=4, fit_gp=False,
                                                             random_state=5)
    assert len({y.tobytes() for y in Y}) == 4


def test_empty_space_draws_what_random_sample_draws(bo, ref):
    mk = lambda: ref.BayesianOptimization(f=None, pbounds=PB, acquisition_function=bo.ThompsonSampling(),  # noqa: E731
                                          random_state=3, verbose=0)
    a, b = mk(), mk()
    got = bo.suggest_batch(a, 4)
    want = b.random_sample(4)
    assert got == want and len(got) == 4
    assert _same_state(a._random_state, b._random_state)


def test_type_error_for_other_acquisition_functions(bo, ref):
    accs = [bo.ExpectedImprovement(xi=0.01), bo.UpperConfidenceBound(kappa=2.0),
            bo.ConstantLiar(bo.ExpectedImprovement(xi=0.01)),
            bo.GPHedge([bo.ExpectedImprovement(xi=0.01), bo.UpperConfidenceBound()]),
            ref.acquisition.ExpectedImprovement(xi=0.01), ref.acquisition.UpperConfidenceBound()]
    for acq in accs:
        opt = ref.BayesianOptimization(f=None, pbounds=PB, acquisition_function=acq, random_state=1, verbose=0)
        with pytest.raises(TypeError, match="ConstantLiar"):
            bo.suggest_batch(opt, 2)


def test_lockstep_driver_routes_each_run_to_its_path(bo, monkeypatch):
    """The three L-BFGS-B drivers (batched, thread-per-run, sequential) give every run of a multi-path closure its own
    path, and agree with scipy's minimize on that path alone."""
    from scipy.optimize import minimize

    from bayesianoptimization_b200.fused import lockstep_lbfgsb
    from bayesianoptimization_b200.paths import PathBatchAcquisition

    p = StubPaths(np.random.RandomState(1), 3, 5, np.zeros(2), np.ones(2))
    acq = PathBatchAcquisition(p)
    bounds = np.array([[0.0, 1.0], [0.0, 1.0]])
    seeds = [_a(0.1, 0.2), _a(0.9, 0.9), _a(0.5, 0.1), _a(0.3, 0.7)]
    owner = [2, 0, 1, 2]
    want = [minimize(acq.path(o), s, bounds=bounds, method="L-BFGS-B") for s, o in zip(seeds, owner)]
    for driver in ("batched", "threads"):
        monkeypatch.setenv("B200BO_LBFGSB_DRIVER", driver)
        got = lockstep_lbfgsb(acq, seeds, bounds, run_paths=owner)
        for g, w in zip(got, want):
            assert np.allclose(g.x, w.x, atol=1e-6) and g.success
    got = lockstep_lbfgsb(acq, seeds[:1], bounds, run_paths=owner[:1])
    assert np.allclose(got[0].x, p.c[owner[0]], atol=1e-4)

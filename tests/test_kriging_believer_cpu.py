"""KrigingBeliever without a GPU: the host logic of suggest / suggest_batch over a stub GP and a stub closure that keep
the interfaces of B200GaussianProcessRegressor.condition_on_pending and FusedAcquisition.  Checked: the order in which
the RandomState is consumed, q = 1 parity with the base acquisition, the batch accounting, the dummies (expiry and the
save_state round trip), argument and refusal errors, the unchanged TypeError of b200.suggest_batch, and the numpy
restatement of the conditioned posterior (tests/believer_oracle.py) against sklearn."""
import contextlib
import json
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

PB = {"x": (0.0, 1.0), "y": (-1.0, 2.0)}
CENTRE = np.array([0.3, 0.5])


@pytest.fixture(scope="module")
def bo():
    import __graft_entry__ as g

    g.build()
    import bayesianoptimization_b200 as bo

    return bo


def _stub_gp_class(bo):
    class StubGP(bo.B200GaussianProcessRegressor):
        """Records every condition_on_pending call in ``log``; conditions in place once conditioned, as the device GP
        does while its capacity holds the rows."""

        def condition_on_pending(self, X, extra_rows=0):
            X = np.asarray(X, dtype=np.float64).reshape(-1, 2)
            self.log.append((len(X), extra_rows, self.__dict__.get("_b200_conditioned") is not None))
            out = self
            if self.__dict__.get("_b200_conditioned") is None:
                out = StubGP(kernel=Matern(nu=2.5), optimizer=None)
                out.log, out.pending = self.log, list(self.pending)
                out.__dict__["_b200_conditioned"] = 5
            out.pending.extend(X)
            return out

    return StubGP


def _stub_gp(bo, log=None):
    gp = _stub_gp_class(bo)(kernel=Matern(nu=2.5), optimizer=None)
    gp.log = [] if log is None else log
    gp.pending = []
    return gp


class StubClosure:
    """-acq(x) = |x - c|^2 + sum over the GP's pending points p of 5 exp(-|x - p|^2 / 0.02): a bowl whose bottom the
    pending points fill in.  Records the candidate sets and Philox seeds it ranks."""

    ranked, seeds = [], []

    def __init__(self, kind, gp, constraint=None, owner=None, max_values=None, **kw):
        self.gp, self.dim, self.devices = gp, 2, [0]

    def __call__(self, X):
        X = np.asarray(X, dtype=np.float64).reshape(-1, 2)
        v = ((X - CENTRE) ** 2).sum(1)
        for p in self.gp.pending:
            v = v + 5.0 * np.exp(-((X - p) ** 2).sum(1) / 0.02)
        return v

    def refine_mode(self):
        return contextlib.nullcontext(self)

    def argmin_topk(self, X, k):
        StubClosure.ranked.append(np.array(X))
        ys = self(X)
        return int(ys.argmin()), float(ys.min()), np.argsort(ys, kind="stable")[:k]

    def argmin_topk_philox(self, seed, bounds, m, k, index_base=0):
        StubClosure.seeds.append(seed)
        b = np.asarray(bounds)
        X = np.random.RandomState(seed % 2**32).uniform(b[:, 0], b[:, 1], (m, 2))
        ys = self(X)
        order = np.argsort(ys, kind="stable")[:k]
        return int(ys.argmin()), float(ys.min()), X[ys.argmin()], order, X[order]


@pytest.fixture(autouse=True)
def _stub_closure(monkeypatch):
    import bayesianoptimization_b200.acquisition as A

    monkeypatch.setattr(A, "FusedAcquisition", StubClosure)
    StubClosure.ranked, StubClosure.seeds = [], []


def _space(n=5, seed=1):
    from bayes_opt.target_space import TargetSpace

    space = TargetSpace(None, PB)
    rs = np.random.RandomState(seed)
    for _ in range(n):
        space.register(space.random_sample(random_state=rs), float(rs.uniform()))
    return space


def _same_state(a, b):
    sa, sb = a.get_state(), b.get_state()
    return np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


def _bases(bo):
    return [bo.UpperConfidenceBound(kappa=2.0, exploration_decay=0.9), bo.ExpectedImprovement(xi=0.01),
            bo.ProbabilityOfImprovement(xi=0.01, exploration_decay=0.8)]


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
@pytest.mark.parametrize("n_smart", [0, 3, 65])
def test_random_state_is_consumed_in_the_documented_order(bo, ref, source, n_smart):
    """ONE candidate set (or one Philox seed) shared by every round - and nothing more on a continuous space; the GP is
    forked once with room for the batch, then conditioned in place on every pick but the last."""
    from bayesianoptimization_b200.acquisition import _philox_seed

    q, n_random = 4, 400
    kb = bo.KrigingBeliever(bo.ExpectedImprovement(xi=0.01))
    kb.base_acquisition.b200_candidate_source = source
    gp, space = _stub_gp(bo), _space()
    ra, rb = np.random.RandomState(9), np.random.RandomState(9)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        X = kb.suggest_batch(gp, space, q, n_random=n_random, n_smart=n_smart, fit_gp=False, random_state=ra)
    assert X.shape == (q, 2) and kb.base_acquisition.i == 1
    assert gp.log == [(0, q, False)] + [(1, 0, True)] * (q - 1)
    if source == "device_philox" and n_smart <= 64:
        assert StubClosure.seeds == [_philox_seed(rb)] * q and not StubClosure.ranked
    else:
        want = space.random_sample(max(n_random, n_smart), random_state=rb)
        if n_smart <= 64:  # (beyond, the numpy selection evaluates the same rows through __call__)
            assert len(StubClosure.ranked) == q and all(np.array_equal(r, want) for r in StubClosure.ranked)
    assert _same_state(ra, rb)
    assert len({x.tobytes() for x in X}) == q  # the pending points push the later rounds away
    assert [d.tobytes() for d in kb.dummies] == [x.tobytes() for x in X]


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
@pytest.mark.parametrize("which", [0, 1, 2])
def test_q1_and_suggest_equal_the_base_acquisition(bo, ref, source, which):
    """Without dummies, suggest_batch(q=1) and suggest() return the base acquisition's point bit for bit, leave the
    RandomState where it does and count / decay as it does; nothing is conditioned."""
    space = _space(seed=4)
    outs = []
    for mode in ("batch", "suggest", "base"):
        base = _bases(bo)[which]
        base.b200_candidate_source = source
        gp, rs = _stub_gp(bo), np.random.RandomState(3)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            if mode == "base":
                x = base.suggest(gp, space, n_random=300, n_smart=4, fit_gp=False, random_state=rs)
            elif mode == "batch":
                x = bo.KrigingBeliever(base).suggest_batch(gp, space, 1, n_random=300, n_smart=4, fit_gp=False,
                                                           random_state=rs)[0]
            else:
                x = bo.KrigingBeliever(base).suggest(gp, space, n_random=300, n_smart=4, fit_gp=False, random_state=rs)
        assert gp.log == []
        outs.append((x, rs, base.get_acquisition_params(), base.i))
    for x, rs, params, i in outs[:2]:
        assert np.array_equal(x, outs[2][0]) and _same_state(rs, outs[2][1])
        assert params == outs[2][2] and i == outs[2][3] == 1


def test_a_batch_counts_and_decays_once(bo, ref):
    kb = bo.KrigingBeliever(bo.UpperConfidenceBound(kappa=2.0, exploration_decay=0.5))
    X = kb.suggest_batch(_stub_gp(bo), _space(), 5, n_random=200, n_smart=2, fit_gp=False, random_state=1)
    assert X.shape == (5, 2) and kb.base_acquisition.i == 1 and kb.base_acquisition.kappa == 1.0
    assert len(kb.dummies) == 5


def test_dummies_expire_and_survive_a_state_round_trip(bo, ref):
    """Three suggest() calls without registering: distinct points, each conditioned on the ones before.  Registering
    a point at a dummy expires it (ConstantLiar's rule, inherited); the dummies go through get/set_acquisition_params
    (what save_state / load_state use) as JSON."""
    kb = bo.KrigingBeliever(bo.ExpectedImprovement(xi=0.01), atol=1e-5, rtol=1e-8)
    space, log = _space(), []
    xs = [kb.suggest(_stub_gp(bo, log), space, n_random=300, n_smart=2, fit_gp=False, random_state=i)
          for i in range(3)]
    assert len({x.tobytes() for x in xs}) == 3 and len(kb.dummies) == 3
    assert log == [(1, 0, False), (2, 0, False)]  # nothing to condition on at the first call
    space.register(xs[0] + 1e-7, 0.5)  # within atol of dummy 0
    log.clear()
    kb.suggest(_stub_gp(bo, log), space, n_random=300, n_smart=2, fit_gp=False, random_state=7)
    assert log == [(2, 0, False)] and len(kb.dummies) == 3
    assert not any(np.array_equal(d, xs[0]) for d in kb.dummies)
    params = json.loads(json.dumps(kb.get_acquisition_params()))
    kb2 = bo.KrigingBeliever(bo.ExpectedImprovement(xi=0.5))
    kb2.set_acquisition_params(params)
    assert [d.tolist() for d in kb2.dummies] == [d.tolist() for d in kb.dummies]
    assert kb2.base_acquisition.xi == kb.base_acquisition.xi and (kb2.atol, kb2.rtol) == (1e-5, 1e-8)


@pytest.mark.parametrize("bad", [0, -1, 1.5, 2.0, True, False, "3", None])
def test_q_validation(bo, ref, bad):
    kb = bo.KrigingBeliever(bo.ExpectedImprovement(xi=0.01))
    rs = np.random.RandomState(0)
    before = rs.get_state()
    with pytest.raises(ValueError, match="q must be"):
        kb.suggest_batch(_stub_gp(bo), _space(), bad, fit_gp=False, random_state=rs)
    assert np.array_equal(before[1], rs.get_state()[1]) and kb.base_acquisition.i == 0 and not kb.dummies
    opt = ref.BayesianOptimization(f=None, pbounds=PB, acquisition_function=kb, verbose=0)
    with pytest.raises(ValueError, match="q must be"):
        bo.suggest_batch(opt, bad)


def test_q_has_no_upper_limit(bo, ref):
    kb = bo.KrigingBeliever(bo.UpperConfidenceBound())
    X = kb.suggest_batch(_stub_gp(bo), _space(), np.int64(20), n_random=100, n_smart=0, fit_gp=False, random_state=1)
    assert X.shape == (20, 2)


def test_refusals(bo, ref):
    from bayes_opt.exception import ConstraintNotSupportedError, TargetSpaceEmptyError
    from bayes_opt.target_space import TargetSpace

    for base in (bo.ThompsonSampling(), bo.ConstantLiar(bo.ExpectedImprovement(xi=0.01)),
                 bo.GPHedge([bo.ExpectedImprovement(xi=0.01), bo.UpperConfidenceBound()]), object()):
        with pytest.raises(TypeError, match="KrigingBeliever needs"):
            bo.KrigingBeliever(base)
    bo.KrigingBeliever(bo.MaxValueEntropySearch())
    kb = bo.KrigingBeliever(ref.acquisition.ExpectedImprovement(xi=0.01))  # a reference object gets the hooks
    assert isinstance(kb.base_acquisition, bo.DeviceHooks) and isinstance(kb, ref.acquisition.ConstantLiar)
    with pytest.raises(TargetSpaceEmptyError):
        kb.suggest(_stub_gp(bo), TargetSpace(None, PB), fit_gp=False, random_state=1)
    space = _space()
    space._constraint = SimpleNamespace(model=[], lb=np.zeros(1), ub=np.ones(1))
    for call in (kb.suggest, lambda *a, **k: kb.suggest_batch(*a, q=2, **k)):
        with pytest.raises(ConstraintNotSupportedError):
            call(_stub_gp(bo), space, fit_gp=False, random_state=1)
    assert kb.base_acquisition.i == 0 and not kb.dummies


def test_condition_on_pending_argument_errors(bo):
    """Checked on the host before any device work."""
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), optimizer=None, devices=[0, 1])
    gp.X_train_ = np.zeros((4, 2))
    with pytest.raises(ValueError, match="n_pending, d"):
        gp.condition_on_pending(np.zeros((2, 3)))
    with pytest.raises(ValueError, match="NaN"):
        gp.condition_on_pending(np.array([[0.1, np.nan]]))
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError, match="extra_rows"):
            gp.condition_on_pending(np.zeros((1, 2)), extra_rows=bad)
    with pytest.raises(NotImplementedError, match="multi-device"):
        gp.condition_on_pending(np.zeros((1, 2)))
    with pytest.raises(ValueError, match="fitted"):
        bo.B200GaussianProcessRegressor().condition_on_pending(np.zeros((1, 2)))


def test_suggest_batch_type_error_is_unchanged(bo, ref):
    accs = [bo.ExpectedImprovement(xi=0.01), bo.UpperConfidenceBound(kappa=2.0),
            bo.ConstantLiar(bo.ExpectedImprovement(xi=0.01)),
            bo.GPHedge([bo.ExpectedImprovement(xi=0.01), bo.UpperConfidenceBound()]),
            ref.acquisition.ExpectedImprovement(xi=0.01), bo.MaxValueEntropySearch()]
    for acq in accs:
        opt = ref.BayesianOptimization(f=None, pbounds=PB, acquisition_function=acq, random_state=1, verbose=0)
        with pytest.raises(TypeError, match="ConstantLiar"):
            bo.suggest_batch(opt, 2)


def test_empty_space_and_enable(bo, ref):
    mk = lambda: ref.BayesianOptimization(  # noqa: E731
        f=None, pbounds=PB, acquisition_function=bo.KrigingBeliever(bo.ExpectedImprovement(xi=0.01)), random_state=3,
        verbose=0)
    a, b = mk(), mk()
    assert bo.suggest_batch(a, 20) == b.random_sample(20)
    assert _same_state(a._random_state, b._random_state) and not a._acquisition_function.dummies
    opt = ref.BayesianOptimization(f=None, pbounds=PB, verbose=0,
                                   acquisition_function=ref.acquisition.ExpectedImprovement(xi=0.01))
    kb = bo.KrigingBeliever(opt._acquisition_function)
    opt._acquisition_function = kb
    bo.enable(opt, candidate_source="device_philox", refine="analytic")
    assert opt._acquisition_function is kb and kb.base_acquisition.b200_candidate_source == "device_philox"
    assert kb.base_acquisition.b200_refine == "analytic"
    assert isinstance(kb, bo.AcquisitionFunction)


@pytest.mark.parametrize("kern", ["m25", "rbf_white", "m15_ard_norm"])
def test_believer_oracle_matches_the_closed_form(kern):
    """The numpy restatement (augmented set, believer targets, fresh Cholesky) against the Schur complement of the
    original GP's joint predictive covariance from sklearn: same mean as the original GP, the same variance; the
    augmented alpha_ is [alpha_; 0]."""
    from sklearn.gaussian_process import GaussianProcessRegressor
    from sklearn.gaussian_process.kernels import RBF, ConstantKernel, WhiteKernel

    from believer_oracle import closed_form, conditioned_posterior

    rs = np.random.RandomState(5)
    d = 3
    X = rs.uniform(size=(60, d))
    y = np.sin(3 * X.sum(1)) + 0.05 * rs.randn(60)
    k = {"m25": Matern(0.5, nu=2.5), "rbf_white": ConstantKernel(1.7) * RBF(0.6) + WhiteKernel(1e-2),
         "m15_ard_norm": Matern([0.3, 0.6, 1.2], nu=1.5)}[kern]
    gp = GaussianProcessRegressor(k, alpha=1e-6, optimizer=None, normalize_y=kern.endswith("norm")).fit(X, y)
    Xq = np.vstack([rs.uniform(size=(40, d)), X[:3] + 1e-3])
    for p in (1, 7):
        P = rs.uniform(size=(p, d))
        mu, sd, a = conditioned_posterior(gp, P, Xq)
        mu_c, sd_c = closed_form(gp, P, Xq)
        mu0, sd0 = gp.predict(Xq, return_std=True)
        scale = float(np.ravel(gp._y_train_std)[0])
        assert np.max(np.abs(mu - mu_c)) / scale < 1e-9 and np.max(np.abs(mu - mu0)) / scale < 1e-9
        assert np.max(np.abs(sd**2 - sd_c**2)) / scale**2 < 1e-9
        assert np.all(sd <= sd0 + 1e-9 * scale) and np.allclose(a[:60], gp.alpha_, rtol=1e-6, atol=1e-8 * np.abs(gp.alpha_).max())
        assert np.max(np.abs(a[60:])) < 1e-6 * np.abs(gp.alpha_).max()

"""Max-value entropy search without a GPU: the numpy oracle against an independent high-precision evaluation over
g in [-40, 40] and the sigma = 0 rule, the order in which MaxValueEntropySearch draws from the suggest RandomState
(a GP whose sample paths are recorded instead of uploaded), the floor of the y* samples, the argument checks and the
parameter round trip."""
from types import SimpleNamespace

import ctypes as C
import os

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

import mes_oracle as MO
import thompson_oracle as T


@pytest.fixture(scope="module")
def bo():
    import __graft_entry__ as g

    g.build()
    import bayesianoptimization_b200 as bo

    return bo


def _exact_term(g):
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 60
    x = mp.mpf(float(g))
    P = mp.erfc(-x / mp.sqrt(2)) / 2
    lnP = mp.log(P) if x < 0 else mp.log1p(-mp.erfc(x / mp.sqrt(2)) / 2)  # 1 - Psi exactly in the upper tail
    return float(x * mp.npdf(x) / (2 * P) - lnP)


GAMMA = np.concatenate([np.linspace(-40.0, 40.0, 801), [-38.5, -37.9, -1e-300, 0.0, 1e-300, -1e-8, 1e-8, 38.6]])


def test_oracle_against_high_precision():
    got = MO.mes_term(GAMMA)
    ref = np.array([_exact_term(g) for g in GAMMA])
    assert np.all(np.isfinite(got)) and np.all(got >= 0.0)
    rel = np.abs(got - ref) / np.maximum(np.abs(ref), 1e-280)  # below 1e-280 the terms are subnormal or zero
    # measured 4.6e-11 at g = -39.8: exp(logpdf - log_ndtr) subtracts two numbers near -800; 3.5e-12 above g = -20
    assert rel[GAMMA < -20].max() < 5e-10
    assert rel[GAMMA >= -20].max() < 5e-11
    # the naive form the tail rules exist for: log(ndtr(g)) is -inf below g ~ -38
    from scipy.special import ndtr

    with np.errstate(divide="ignore"):
        assert np.isinf(np.log(ndtr(-39.0)))


def test_oracle_sigma_zero_and_average_in_k_order():
    mu = np.array([0.0, 1.0, -2.0, 0.5])
    sd = np.array([1.0, 0.0, 2.0, 0.0])
    ys = np.array([1.5, -0.25, 3.0])
    a = MO.mes_alpha(mu, sd, ys)
    assert a[1] == 0.0 and a[3] == 0.0  # sigma = 0: a point mass, nothing to learn
    for i in (0, 2):
        s = 0.0
        for y in ys:
            s = s + MO.mes_term((y - mu[i]) / sd[i])
        assert a[i] == s / 3
    prod = np.array([0.5, 1.0, 0.25, 1.0])
    assert np.array_equal(MO.mes_closure(mu, sd, ys, prod), -1 * a * prod)


def test_abi_constants_and_argument_checks(bo):
    from bayesianoptimization_b200 import _lib as B

    assert B.ACQ_MES == 4 and "b200bo_gp_set_max_values" in B.EXPORTS
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "b200bo.h")).read()
    assert "#define B200BO_ACQ_MES 4" in hdr
    v = np.zeros(3)
    assert B.lib().b200bo_gp_set_max_values(None, B.as_dp(v), 3) == B.ERR_ARG  # host-side check, no device needed


class _FakePaths:
    """Stands in for a PosteriorPaths: records the candidate rows / Philox seed it ranks and returns chosen maxima."""

    def __init__(self, q, cand_max, train_vals, log):
        self.n_paths, self.devices = q, [0]
        self.cand_max, self.train_vals, self.log = np.asarray(cand_max, float), train_vals, log

    def argmin_topk(self, X, k):
        self.log.append(("rows", np.array(X), k))
        return np.zeros(self.n_paths, np.int64), -self.cand_max, [np.zeros(0, np.int64)] * self.n_paths

    def argmin_topk_philox(self, seed, bounds, m, k, index_base=0):
        self.log.append(("philox", seed, np.array(bounds), m, k))
        q = self.n_paths
        return np.zeros(q, np.int64), -self.cand_max, np.zeros((q, 2)), [], []

    def __call__(self, X):
        self.log.append(("train", np.array(X)))
        return np.asarray(self.train_vals, float)


def _recording_gp(bo, log, nu, n, noise, d=2, cand_max=None, train_vals=None, y=None):
    from bayesianoptimization_b200.paths import draw_path_inputs

    class Recording(bo.B200GaussianProcessRegressor):
        def sample_paths(self, n_paths=1, n_features=4096, random_state=None):
            log.append(("paths", n_paths, n_features,
                        draw_path_inputs(random_state, n_paths, n_features, d, nu, n, noise)))
            cm = np.zeros(n_paths) if cand_max is None else cand_max
            tv = np.full((n, n_paths), -1.0) if train_vals is None else train_vals
            return _FakePaths(n_paths, cm, tv, log)

    gp = Recording(kernel=Matern(nu=nu), optimizer=None)
    gp.X_train_ = np.random.RandomState(0).uniform(size=(n, d))
    gp._y_raw = np.full(n, -5.0) if y is None else np.asarray(y, float)
    return gp


def _space(ref):
    from bayes_opt.target_space import TargetSpace

    return TargetSpace(None, {"a": (0.0, 1.0), "b": (-2.0, 3.0)})


def test_draw_order_paths_then_candidates(bo, ref):
    log = []
    gp = _recording_gp(bo, log, 2.5, 7, 1e-6)
    mes = bo.MaxValueEntropySearch(n_samples=4, n_features=33, n_max_candidates=50)
    space = _space(ref)
    mes._path_rng, mes._suggest_space = np.random.RandomState(42), space
    acq = mes._get_acq(gp)
    assert [e[0] for e in log] == ["paths", "rows", "train"]
    assert log[0][1:3] == (4, 33) and log[1][2] == 0
    want = np.random.RandomState(42)
    for a, b in zip(log[0][3], T.draws(want, 4, 33, 2, 2.5, 7, 1e-6)):
        assert np.array_equal(a, b)
    assert np.array_equal(log[1][1], space.random_sample(50, random_state=want))  # step 2: the y* candidate set
    assert np.array_equal(log[2][1], gp.X_train_)
    sa, sb = mes._path_rng.get_state(), want.get_state()
    assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]  # step 3 (random stage) continues from here
    assert type(acq).__name__ == "FusedAcquisition" and acq.kind == bo._lib.ACQ_MES
    assert np.array_equal(acq._ystar, mes.max_values) and acq._ystar.shape == (4,)


def test_draw_order_device_philox(bo, ref):
    log = []
    gp = _recording_gp(bo, log, 1.5, 5, 1e-4)
    mes = bo.MaxValueEntropySearch(n_samples=2, n_features=16, n_max_candidates=1000)
    mes.b200_candidate_source = "device_philox"
    space = _space(ref)
    mes._path_rng, mes._suggest_space = np.random.RandomState(7), space
    mes._get_acq(gp)
    assert [e[0] for e in log] == ["paths", "philox", "train"]
    want = np.random.RandomState(7)
    T.draws(want, 2, 16, 2, 1.5, 5, 1e-4)
    hi = int(want.randint(0, 2**32, dtype=np.uint64))  # the seed of DeviceHooks._random_sample_minimize
    seed = hi << 32 | int(want.randint(0, 2**32, dtype=np.uint64))
    assert log[1][1] == seed and log[1][3] == 1000 and log[1][4] == 0
    assert np.array_equal(log[1][2], space.bounds)
    assert np.array_equal(mes._path_rng.get_state()[1], want.get_state()[1])


def test_max_value_floor(bo, ref):
    from bayesianoptimization_b200.acquisition import mes_max_values

    log = []
    n = 4
    train = np.array([[0.0, 9.0, -3.0], [1.0, 2.0, -3.0], [0.5, 2.0, -4.0], [0.0, 0.0, -3.5]])  # (n, q)
    gp = _recording_gp(bo, log, 2.5, n, 1e-6, cand_max=[3.0, 1.0, -10.0], train_vals=train,
                       y=[0.5, 2.5, -1.0, 0.0])
    paths = gp.sample_paths(3, 8, random_state=np.random.RandomState(0))
    ys = mes_max_values(gp, paths, _space(ref), np.random.RandomState(1), 20)
    # path 0: candidates (3.0) beat the training rows (1.0); path 1: the training rows (9.0) win;
    # path 2: both lie below the largest registered target 2.5, which floors it
    assert np.array_equal(ys, [3.0, 9.0, 2.5])


def test_argument_checks(bo, ref):
    for bad in (0, 17, 1.5, True, "3"):
        with pytest.raises(ValueError, match="n_samples"):
            bo.MaxValueEntropySearch(n_samples=bad)
    for bad in (0, 2.0):
        with pytest.raises(ValueError, match="n_features"):
            bo.MaxValueEntropySearch(n_features=bad)
        with pytest.raises(ValueError, match="n_max_candidates"):
            bo.MaxValueEntropySearch(n_max_candidates=bad)
    bo.MaxValueEntropySearch(n_samples=1)
    bo.MaxValueEntropySearch(n_samples=16)
    with pytest.raises(NotImplementedError, match="base_acq"):
        bo.MaxValueEntropySearch().base_acq(np.zeros(1), np.ones(1))
    gp = _recording_gp(bo, [], 2.5, 3, 1e-6)
    with pytest.raises(RuntimeError, match="suggest"):
        bo.MaxValueEntropySearch()._get_acq(gp)
    FA, B = bo.FusedAcquisition, bo._lib
    FA(B.ACQ_MES, gp, max_values=np.arange(16.0))
    for bad in (None, [], np.arange(17.0), [1.0, np.nan], [np.inf]):
        with pytest.raises(ValueError, match="max_values"):
            FA(B.ACQ_MES, gp, max_values=bad)
    with pytest.raises(ValueError, match="ACQ_MES only"):
        FA(B.ACQ_EI, gp, max_values=[1.0])


def test_constraint_checks_consume_no_random_numbers(bo, ref):
    from sklearn.gaussian_process import GaussianProcessRegressor

    log = []
    gp = _recording_gp(bo, log, 2.5, 5, 1e-6)
    mes = bo.MaxValueEntropySearch(n_samples=2)
    rs = np.random.RandomState(9)
    mes._path_rng, mes._suggest_space = rs, _space(ref)
    host_gp = SimpleNamespace(model=[GaussianProcessRegressor()], lb=np.zeros(1), ub=np.ones(1))
    with pytest.raises(TypeError, match="B200GaussianProcessRegressor"):
        mes._get_acq(gp, constraint=host_gp)
    too_many = SimpleNamespace(model=[_recording_gp(bo, log, 2.5, 5, 1e-6) for _ in range(8)],
                               lb=np.zeros(8), ub=np.ones(8))
    with pytest.raises(NotImplementedError, match="at most 7"):
        mes._get_acq(gp, constraint=too_many)
    assert log == []
    assert np.array_equal(rs.get_state()[1], np.random.RandomState(9).get_state()[1])


def test_class_registration_and_parameter_round_trip(bo, ref):
    mes = bo.MaxValueEntropySearch(n_samples=7, n_features=512, n_max_candidates=1234)
    assert "MaxValueEntropySearch" in bo.__all__
    assert isinstance(mes, bo.AcquisitionFunction) and isinstance(mes, bo.DeviceHooks)
    assert isinstance(mes, ref.acquisition.AcquisitionFunction)
    params = mes.get_acquisition_params()
    assert params == {"n_samples": 7, "n_features": 512, "n_max_candidates": 1234}
    other = bo.MaxValueEntropySearch()
    assert other.get_acquisition_params()["n_max_candidates"] == bo.acquisition.MES_MAX_CANDIDATES
    other.set_acquisition_params(params)
    assert other.get_acquisition_params() == params
    with pytest.raises(ValueError, match="n_samples"):
        other.set_acquisition_params({**params, "n_samples": 17})
    opt = ref.BayesianOptimization(f=None, pbounds={"x": (0, 1)}, acquisition_function=mes, verbose=0)
    bo.enable(opt)
    assert opt._acquisition_function is mes
    # ThompsonSampling shares the suggest-stream code
    from bayesianoptimization_b200.acquisition import _SuggestStream

    assert isinstance(bo.ThompsonSampling(), _SuggestStream) and isinstance(mes, _SuggestStream)

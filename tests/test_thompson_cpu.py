"""Thompson sampling without a GPU: the path formulas restated in tests/thompson_oracle.py ARE samples of the GP
posterior (checked against sklearn's predict(return_cov=True)), the product's draw helper consumes the RandomState
in the documented order, and the host logic of ThompsonSampling / sample_paths."""
import numpy as np
import pytest
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, WhiteKernel

import thompson_oracle as T


@pytest.fixture(scope="module")
def bo():
    import __graft_entry__ as g

    g.build()
    import bayesianoptimization_b200 as bo

    return bo


# (kind, nu, length scale ("aniso": one per dimension), ConstantKernel value, WhiteKernel noise_level)
CASES = {
    "matern05": (T.KIND_MATERN, 0.5, 0.4, 1.0, 0.0),
    "matern15": (T.KIND_MATERN, 1.5, 0.4, 1.0, 0.0),
    "matern25": (T.KIND_MATERN, 2.5, 0.4, 1.0, 0.0),
    "rbf": (T.KIND_RBF, np.inf, 0.3, 1.0, 0.0),
    "aniso": (T.KIND_MATERN, 2.5, "aniso", 1.0, 0.0),
    "const": (T.KIND_RBF, np.inf, 0.3, 2.5, 0.0),
    "white": (T.KIND_MATERN, 1.5, 0.4, 1.0, 0.05),
}


@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_paths_are_posterior_samples(case, d):
    """Empirical mean / covariance of q = 2000 paths (L = 4096) at 16 points == sklearn's predictive mean and
    covariance with the WhiteKernel noise taken off the diagonal (a path samples the latent function).  Tolerance:
    5 Monte-Carlo standard errors + 2 c s_y^2 / sqrt(L), the size of the random-Fourier-feature error of the prior
    covariance (one set of features is shared by all paths, so that error does not average out).  A wrong spectral
    density (e.g. the RBF's for a Matern kernel) misses by 10x that allowance."""
    kind, nu, ls, c, noise = CASES[case]
    rs = np.random.RandomState(7)
    n, q, L, alpha = 60, 2000, 4096, 1e-4
    X = rs.uniform(size=(n, d))
    y = np.sin(3 * X.sum(1)) + 0.1 * rs.randn(n)
    Xq = rs.uniform(-0.1, 1.1, size=(16, d))
    lsv = np.linspace(0.3, 0.6, d) if ls == "aniso" else ls
    k = RBF(lsv) if kind == T.KIND_RBF else Matern(lsv, nu=nu)
    if c != 1.0:
        k = ConstantKernel(c) * k
    if noise:
        k = k + WhiteKernel(noise)
    gp = GaussianProcessRegressor(k, alpha=alpha, optimizer=None, normalize_y=True).fit(X, y)
    mu, cov = gp.predict(Xq, return_cov=True)
    s_y = float(np.std(y))
    cov = cov - np.eye(len(Xq)) * noise * s_y**2
    dr = T.draws(np.random.RandomState(11), q, L, d, nu, n, alpha + noise)
    f = T.path_values(X, y, Xq, dr, kind=kind, nu=nu, length_scale=lsv, const=c, alpha=alpha, noise_level=noise)
    var = np.maximum(np.diag(cov), 0.0)
    rff = 2.0 * c * s_y**2 / np.sqrt(L)
    assert np.all(np.abs(f.mean(1) - mu) <= 5 * np.sqrt(var / q) + rff)
    se = np.sqrt((np.outer(var, var) + cov**2) / q)
    assert np.all(np.abs(np.cov(f) - cov) <= 5 * se + rff)


@pytest.mark.parametrize("nu", [0.5, 1.5, 2.5, np.inf])
def test_draw_helper_consumes_the_random_state_in_order(nu):
    from bayesianoptimization_b200.paths import draw_path_inputs

    q, L, d, n, nv = 3, 17, 4, 9, 0.25
    a, b = np.random.RandomState(5), np.random.RandomState(5)
    got = draw_path_inputs(a, q, L, d, nu, n, nv)
    z = b.standard_normal((L, d))
    omega = z if nu == np.inf else z * np.sqrt(2 * nu / b.chisquare(2 * nu, L))[:, None]
    want = (omega, b.uniform(0, 2 * np.pi, L), b.standard_normal((L, q)), b.standard_normal((n, q)) * np.sqrt(nv))
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    sa, sb = a.get_state(), b.get_state()
    assert sa[0] == sb[0] and np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]
    # and the restatement used by the tests draws the same arrays
    for g, w in zip(got, T.draws(np.random.RandomState(5), q, L, d, nu, n, nv)):
        assert np.array_equal(g, w)


def test_sample_paths_validation(bo):
    from bayesianoptimization_b200._lib import B200Error

    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), optimizer=None)
    for bad in (0, 17, -1, 1.5, True):
        with pytest.raises(ValueError, match="n_paths"):
            gp.sample_paths(n_paths=bad)
    with pytest.raises(ValueError, match="n_features"):
        gp.sample_paths(n_paths=1, n_features=0)
    with pytest.raises(B200Error, match="GP is not fitted"):
        gp.sample_paths(n_paths=16)


def test_thompson_sampling_host_logic(bo, ref):
    from bayes_opt.exception import ConstraintNotSupportedError

    ts = bo.ThompsonSampling(n_features=512)
    assert isinstance(ts, ref.acquisition.AcquisitionFunction) and isinstance(ts, bo.DeviceHooks)
    assert isinstance(ts, bo.AcquisitionFunction)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), optimizer=None)
    with pytest.raises(ConstraintNotSupportedError):
        ts._get_acq(gp, constraint=object())
    with pytest.raises(NotImplementedError, match="no base_acq"):
        ts.base_acq(np.zeros(2), np.ones(2))
    with pytest.raises(ValueError, match="n_features"):
        bo.ThompsonSampling(n_features=0)
    # parameters round-trip (what save_state / load_state carry)
    params = ts.get_acquisition_params()
    assert params == {"n_features": 512}
    other = bo.ThompsonSampling()
    other.set_acquisition_params(params)
    assert other.n_features == 512 and other.get_acquisition_params() == params
    # enable() keeps an object that already has the device hooks
    opt = ref.BayesianOptimization(f=None, pbounds={"x": (0, 1)}, acquisition_function=ts, verbose=0)
    bo.enable(opt)
    assert opt._acquisition_function is ts


def test_device_closure_protocol(bo, ref):
    """The hooks recognise device closures by protocol; the host closures of user formulas are not ones."""
    from bayesianoptimization_b200.acquisition import _device_closure
    from bayesianoptimization_b200.paths import PathAcquisition

    from types import SimpleNamespace

    assert _device_closure(PathAcquisition(SimpleNamespace(devices=[0])))
    assert not _device_closure(lambda x: x)
    assert callable(getattr(bo.FusedAcquisition, "argmin_topk")) and callable(bo.FusedAcquisition.argmin_topk_philox)

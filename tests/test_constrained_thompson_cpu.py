"""Constrained Thompson sampling without a GPU: the order in which ConstrainedThompsonSampling draws its paths from
the suggest RandomState, its delegation to ThompsonSampling without a constraint, the argument checks of
ConstrainedPaths, and the parameter round trip of save_state / load_state."""
from types import SimpleNamespace

import ctypes as C
import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

import thompson_oracle as T


@pytest.fixture(scope="module")
def bo():
    import __graft_entry__ as g

    g.build()
    import bayesianoptimization_b200 as bo

    return bo


def _fake_set(q=1, d=2, device=0, xform=("device", None)):
    """Stands in for a PosteriorPaths: the attributes ConstrainedPaths checks, and a NULL handle."""
    return SimpleNamespace(n_paths=q, dim=d, device=device, devices=[device], _xform=xform,
                           _handle=SimpleNamespace(ptr=C.c_void_p()))


def _recording_gp(bo, name, log, nu, n, noise, d=2):
    """A device GP whose sample_paths records the draws PosteriorPaths would make (paths.draw_path_inputs with the
    GP's own nu, n and noise variance) instead of uploading them."""
    from bayesianoptimization_b200.paths import draw_path_inputs

    class Recording(bo.B200GaussianProcessRegressor):
        def sample_paths(self, n_paths=1, n_features=4096, random_state=None):
            log.append((name, n_paths, n_features, draw_path_inputs(random_state, n_paths, n_features, d, nu, n, noise)))
            return _fake_set(n_paths, d)

    return Recording(kernel=Matern(nu=nu), optimizer=None)


def test_draw_order_target_then_constraints(bo, ref):
    log = []
    gp = _recording_gp(bo, "target", log, 2.5, 7, 1e-6)
    models = [_recording_gp(bo, "c0", log, 1.5, 7, 1e-6), _recording_gp(bo, "c1", log, np.inf, 7, 1e-4)]
    constraint = SimpleNamespace(model=models, lb=np.array([-np.inf, 0.0]), ub=np.array([0.5, np.inf]))
    ts = bo.ConstrainedThompsonSampling(n_features=33)
    ts._path_rng = np.random.RandomState(42)
    acq = ts._get_acq(gp, constraint=constraint)
    assert [e[0] for e in log] == ["target", "c0", "c1"]
    assert all(e[1] == 1 and e[2] == 33 for e in log)
    want = np.random.RandomState(42)
    for (_, _, _, got), (nu, nv) in zip(log, [(2.5, 1e-6), (1.5, 1e-6), (np.inf, 1e-4)]):
        for a, b in zip(got, T.draws(want, 1, 33, 2, nu, 7, nv)):
            assert np.array_equal(a, b)
    sa, sb = ts._path_rng.get_state(), want.get_state()
    assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]
    cp = acq.paths
    assert type(cp).__name__ == "ConstrainedPaths" and cp.n_sets == 3 and cp.n_paths == 1
    assert np.array_equal(cp._lb, [-np.inf, 0.0]) and np.array_equal(cp._ub, [0.5, np.inf])


def test_without_constraint_it_is_thompson_sampling(bo, ref):
    from bayesianoptimization_b200.paths import PathAcquisition

    logs = {}
    for cls in (bo.ThompsonSampling, bo.ConstrainedThompsonSampling):
        log = logs[cls] = []
        ts = cls(n_features=64)
        ts._path_rng = np.random.RandomState(3)
        acq = ts._get_acq(_recording_gp(bo, "target", log, 2.5, 5, 1e-6), constraint=None)
        assert type(acq) is PathAcquisition and type(acq.paths) is SimpleNamespace
    (a,), (b,) = logs.values()
    assert a[:3] == b[:3] and all(np.array_equal(x, y) for x, y in zip(a[3], b[3]))


def test_constrained_paths_argument_checks(bo):
    from bayesianoptimization_b200.paths import ConstrainedPaths

    t = _fake_set(q=3, d=4)
    ConstrainedPaths(t, [_fake_set(3, 4), _fake_set(3, 4)], [0.0, -np.inf], [0.0, 1.0])  # lb == ub is allowed
    with pytest.raises(ValueError, match="paths"):
        ConstrainedPaths(t, [_fake_set(2, 4)], [0.0], [1.0])
    with pytest.raises(ValueError, match="d="):
        ConstrainedPaths(t, [_fake_set(3, 5)], [0.0], [1.0])
    with pytest.raises(ValueError, match="device"):
        ConstrainedPaths(t, [_fake_set(3, 4, device=1)], [0.0], [1.0])
    with pytest.raises(ValueError, match="lb > ub"):
        ConstrainedPaths(t, [_fake_set(3, 4), _fake_set(3, 4)], [0.0, 2.0], [1.0, 1.0])
    with pytest.raises(ValueError, match="lb > ub"):
        ConstrainedPaths(t, [_fake_set(3, 4)], [np.nan], [1.0])
    with pytest.raises(ValueError, match="one entry per constraint"):
        ConstrainedPaths(t, [_fake_set(3, 4)], [0.0, 0.0], [1.0, 1.0])
    ConstrainedPaths(t, [_fake_set(3, 4) for _ in range(7)], np.zeros(7), np.ones(7))  # G = 8
    with pytest.raises(ValueError, match="at most 7"):
        ConstrainedPaths(t, [_fake_set(3, 4) for _ in range(8)], np.zeros(8), np.ones(8))  # G = 9
    with pytest.raises(ValueError, match="at least one"):
        ConstrainedPaths(t, [], [], [])
    one_hot, other = (lambda X: X), (lambda X: X)
    host = lambda f: _fake_set(3, 4, xform=("host", f))  # noqa: E731
    ConstrainedPaths(host(one_hot), [host(one_hot)], [0.0], [1.0])
    with pytest.raises(NotImplementedError, match="host-side"):
        ConstrainedPaths(host(one_hot), [host(other)], [0.0], [1.0])
    with pytest.raises(NotImplementedError, match="host-side"):
        ConstrainedPaths(host(one_hot), [_fake_set(3, 4)], [0.0], [1.0])


def test_constraint_model_checks_consume_no_random_numbers(bo, ref):
    from sklearn.gaussian_process import GaussianProcessRegressor

    log = []
    gp = _recording_gp(bo, "target", log, 2.5, 5, 1e-6)
    ts = bo.ConstrainedThompsonSampling(n_features=16)
    rs = np.random.RandomState(9)
    ts._path_rng = rs
    host_gp = SimpleNamespace(model=[_recording_gp(bo, "c0", log, 2.5, 5, 1e-6), GaussianProcessRegressor()],
                              lb=np.zeros(2), ub=np.ones(2))
    with pytest.raises(TypeError, match="B200GaussianProcessRegressor"):
        ts._get_acq(gp, constraint=host_gp)
    too_many = SimpleNamespace(model=[_recording_gp(bo, f"c{j}", log, 2.5, 5, 1e-6) for j in range(8)],
                               lb=np.zeros(8), ub=np.ones(8))
    with pytest.raises(NotImplementedError, match="at most 7"):
        ts._get_acq(gp, constraint=too_many)
    assert log == []
    assert np.array_equal(rs.get_state()[1], np.random.RandomState(9).get_state()[1])


def test_class_registration_and_parameter_round_trip(bo, ref):
    cts = bo.ConstrainedThompsonSampling(n_features=512)
    assert "ConstrainedThompsonSampling" in bo.__all__ and "ConstrainedPaths" in bo.__all__
    assert isinstance(cts, bo.ThompsonSampling) and isinstance(cts, bo.AcquisitionFunction)
    assert isinstance(cts, ref.acquisition.AcquisitionFunction) and isinstance(cts, bo.DeviceHooks)
    params = cts.get_acquisition_params()
    assert params == {"n_features": 512}
    other = bo.ConstrainedThompsonSampling()
    other.set_acquisition_params(params)
    assert other.n_features == 512 and other.get_acquisition_params() == params
    with pytest.raises(ValueError, match="n_features"):
        bo.ConstrainedThompsonSampling(n_features=0)
    opt = ref.BayesianOptimization(f=None, pbounds={"x": (0, 1)}, acquisition_function=cts, verbose=0)
    bo.enable(opt)
    assert opt._acquisition_function is cts

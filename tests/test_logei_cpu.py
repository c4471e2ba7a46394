"""LogEI / LogPoI without a GPU: the numpy restatement of the device epilogue (tests/logei_oracle.py) against a 60-digit
evaluation of log h, its derivative ratios, log Phi and the log constraint factor over z in [-1e9, 40], the sigma = 0
rules, the host base_acq and log-space closure against the restatement, and the class wiring: device kinds, parameter
round trip, error types, and KrigingBeliever / GPHedge / ConstantLiar construction."""
import os
from types import SimpleNamespace

import numpy as np
import pytest

import logei_oracle as LO

pytest.importorskip("mpmath")

# z grid: uniform over [-40, 40], logarithmic down to -1e9, dense around -1 (branch), -38.6 (Phi, phi underflow in the
# naive form) and -1/sqrt(eps) = -2^26 (the asymptote)
_T = -(2.0**26)
Z = np.unique(np.concatenate([
    np.linspace(-40.0, 40.0, 401),
    -np.logspace(np.log10(40.0), 9.0, 300),
    -1.0 + np.linspace(-1e-3, 1e-3, 41), [np.nextafter(-1.0, 0.0), -1.0, np.nextafter(-1.0, -2.0)],
    -38.6 + np.linspace(-0.5, 0.5, 41),
    _T * (1.0 + np.linspace(-1e-2, 1e-2, 41)), [np.nextafter(_T, 0.0), _T, np.nextafter(_T, -np.inf)],
    [0.0, -1e-300, 1e-300, 1e-8, -1e-8],
]))

# Bars, pinned at about 10x the measured error (numpy 2 / scipy on x86-64).  Value: |d| / (1 + |log h|).  Ratios:
# relative, split where the log1mexp argument loses digits (its absolute error ~ eps against a size of 1/z^2).
BAR_LOG_H = 1e-14
BAR_RATIO = 64          # in units of eps max(1, z^2): below z = -1 w ~ 1/z^2 comes from a log1mexp argument whose
                        # absolute error is a few eps, so the relative error grows as eps z^2 (about 1 near -2^26)
BAR_LOG_NDTR = 2e-12     # measured 1.9e-13 (ndtr in the upper tail)
BAR_CFACTOR = 1e-12
BAR_CFACTOR_D = 1e-10


@pytest.fixture(scope="module")
def exact():
    return SimpleNamespace(
        log_h=np.array([LO.mp_log_h(z) for z in Z]),
        ratios=np.array([LO.mp_log_h_ratios(z) for z in Z]),
        log_ndtr=np.array([LO.mp_log_ndtr(z) for z in Z]),
    )


def test_log_h_against_60_digits(exact):
    got = LO.log_h(Z)
    assert np.all(np.isfinite(got))
    err = np.abs(got - exact.log_h) / (1.0 + np.abs(exact.log_h))
    print(f"log_h: max {err.max():.2e} at z = {Z[np.argmax(err)]:.6g}")
    assert err.max() < BAR_LOG_H
    # the problem it solves: log EI through EI itself is -inf from z ~ -38.6 down
    with np.errstate(divide="ignore"):
        naive = np.log(LO.norm_pdf(Z) + Z * LO.ndtr(Z))
    assert np.isinf(naive[Z < -40.0]).all()


def test_log_h_ratios_against_60_digits(exact):
    r, q = LO.log_h_ratios(Z)
    assert np.all(np.isfinite(r)) and np.all(np.isfinite(q)) and np.all(q >= 0) and np.all(r > 0)
    er = np.abs(r - exact.ratios[:, 0]) / np.abs(exact.ratios[:, 0])
    eq = np.abs(q - exact.ratios[:, 1]) / np.maximum(np.abs(exact.ratios[:, 1]), 1e-290)  # phi underflows above z ~ 38
    unit = np.finfo(float).eps * np.maximum(1.0, Z * Z)
    far = Z <= _T
    print(f"ratios: r {np.max(er / unit):.1f}, q {np.max(eq / unit):.1f} (eps z^2); |z| <= 40: r {er[np.abs(Z) <= 40].max():.1e}"
          f" q {eq[np.abs(Z) <= 40].max():.1e}; below -2^26 r {er[far].max():.1e} q {eq[far].max():.1e}")
    assert np.max(er / unit) < BAR_RATIO and np.max(eq / unit) < BAR_RATIO
    assert er[far].max() < 1e-14 and eq[far].max() < 1e-14  # the asymptote is exact to 1/z^2 < eps there


def test_log_ndtr_against_60_digits(exact):
    got = LO.log_ndtr(Z)
    err = np.abs(got - exact.log_ndtr) / np.maximum(np.abs(exact.log_ndtr), 1e-280)
    small = np.abs(exact.log_ndtr) < 1e-280  # log Phi = -Phi(-z) is subnormal above z ~ 37.5: compare absolutely
    print(f"log_ndtr: max rel {err[~small].max():.2e}")
    assert err[~small].max() < BAR_LOG_NDTR and np.all(np.abs(got[small]) < 1e-280)


PAIRS = [(-np.inf, 0.3), (-np.inf, -45.0), (-np.inf, 12.0), (0.2, np.inf), (45.0, np.inf), (-12.0, np.inf),
         (-0.5, 0.7), (-1e-3, 1e-3), (-8.0, 9.0),                                         # straddling
         (-50.0, -49.0), (-40.0, -38.0), (-3.0, -2.9), (-1.0, 0.0), (-1e3, -999.9),      # lower tail
         (38.0, 40.0), (49.0, 50.0), (2.9, 3.0), (0.0, 1.0), (999.9, 1e3), (5.0, 5.0 + 1e-9)]  # upper tail


@pytest.mark.parametrize("l,u", PAIRS)
def test_log_constraint_factor_against_60_digits(l, u):
    v = LO.cfactor_std(np.array([l]), np.array([u]))[0]
    fl, fu = (x[0] for x in LO.cfactor_partials(np.array([l]), np.array([u])))
    ev, efl, efu = LO.mp_cfactor(l, u)
    assert np.isfinite(v) and np.isfinite(fl) and np.isfinite(fu)
    ev_err = abs(v - ev) / (1.0 + abs(ev))
    d_err = max(abs(fl - efl), abs(fu - efu)) / (abs(efl) + abs(efu))
    print(f"cfactor ({l}, {u}): value {ev_err:.1e}, partials {d_err:.1e}")
    # a pair of width w in one tail: log Phi(a) - log Phi(b) ~ w |b| is formed from two values with absolute errors
    # of a few eps |log Phi|, so both errors grow as eps / w
    narrow = 1.0 + 1e-5 / (u - l)
    assert ev_err < BAR_CFACTOR * narrow and d_err < BAR_CFACTOR_D * narrow


def test_constraint_factor_in_data_units_and_frozen_norm_rule():
    mean = np.array([0.0, 1.0, -3.0, 2.0, np.nan, 0.5])
    sd = np.array([1.0, 0.5, 0.1, 0.0, 1.0, 2.0])
    v = LO.log_cfactor(-1.0, 2.0, mean, sd)
    ref = LO.cfactor_std((-1.0 - mean) / np.where(sd > 0, sd, 1.0), (2.0 - mean) / np.where(sd > 0, sd, 1.0))
    ok = (sd > 0) & ~np.isnan(mean)
    assert np.array_equal(v[ok], ref[ok]) and np.all(np.isnan(v[~ok]))
    assert np.array_equal(LO.log_cfactor(-np.inf, np.inf, mean, sd), np.zeros(6))
    # far from feasibility the factor is finite: the closure still ranks there (p underflows to 0)
    far = LO.log_cfactor(-np.inf, 0.0, np.array([50.0, 60.0]), np.array([1.0, 1.0]))
    assert np.all(np.isfinite(far)) and far[1] < far[0]


def test_sigma_zero_limits_and_logpoi():
    a = np.array([0.5, -0.5, 0.0, 0.5, -0.5, np.nan])
    sd = np.array([0.0, 0.0, 0.0, 1e-320, 1e-320, 1.0])
    v = LO.log_acq_term(LO.LOGEI, a, sd)
    assert v[0] == np.log(0.5) and v[1] == -np.inf and np.isnan(v[2]) and v[3] == np.log(0.5)
    assert v[4] == -np.inf and np.isnan(v[5])
    p = LO.log_acq_term(LO.LOGPOI, a, sd)
    assert p[0] == 0.0 and p[1] == -np.inf and np.isnan(p[2]) and np.isnan(p[5])
    # the closure is +inf / NaN there, so np.argmin semantics carry over
    c = LO.closure(LO.LOGEI, a, sd, 0.0, 0.0)
    assert c[1] == np.inf and np.isnan(c[2])
    # gradients stay finite for every finite z
    z = Z[np.isfinite(Z)]
    for kind in (LO.LOGEI, LO.LOGPOI):
        _, cm, cs = LO.log_acq_term_grad(kind, z, np.ones_like(z))
        assert np.all(np.isfinite(cm)) and np.all(np.isfinite(cs))


def test_closure_sums_constraints_in_order():
    rs = np.random.RandomState(3)
    mean, sd = rs.randn(50), rs.uniform(0.1, 2.0, 50)
    cons = [(rs.randn(50), rs.uniform(0.1, 1.0, 50), -0.5, 0.5), (rs.randn(50), rs.uniform(0.1, 1.0, 50), 1.0, np.inf)]
    c = LO.closure(LO.LOGEI, mean, sd, 0.3, 0.01, cons)
    s = LO.log_acq_term(LO.LOGEI, mean - 0.3 - 0.01, sd)
    s = s + LO.log_cfactor(-0.5, 0.5, cons[0][0], cons[0][1])
    s = s + LO.log_cfactor(1.0, np.inf, cons[1][0], cons[1][1])
    assert np.array_equal(c, -s)
    # exp(log EI) is EI where EI is representable
    from scipy.stats import norm

    a = mean - 0.3 - 0.01
    ei = a * norm.cdf(a / sd) + sd * norm.pdf(a / sd)
    np.testing.assert_allclose(np.exp(-LO.closure(LO.LOGEI, mean, sd, 0.3, 0.01)), ei, rtol=1e-12)


def _central(f, x, h):
    return (f(x + h) - f(x - h)) / (2 * h)


def test_gradient_coefficients_against_central_differences():
    mean = np.array([0.2, -1.5, -30.0, -500.0, 2.0])
    sd = np.array([0.7, 0.3, 1.1, 2.0, 0.05])
    for kind in (LO.LOGEI, LO.LOGPOI):
        _, cm, cs = LO.log_acq_term_grad(kind, mean, sd)
        h = 1e-6 * np.maximum(1.0, np.abs(mean))
        dm = _central(lambda m: LO.log_acq_term(kind, m, sd), mean, h)
        ds = _central(lambda s: LO.log_acq_term(kind, mean, s), sd, 1e-6 * sd)
        np.testing.assert_allclose(cm, dm, rtol=1e-6)
        np.testing.assert_allclose(cs, ds, rtol=1e-6)
    for lo, hi in ((-0.5, 0.5), (3.0, 4.0), (-np.inf, -2.0), (1.0, np.inf), (-40.0, -39.0)):
        cm, cs = LO.log_cfactor_grad(lo, hi, mean[:3], sd[:3])
        dm = _central(lambda m: LO.log_cfactor(lo, hi, m, sd[:3]), mean[:3], 1e-6)
        ds = _central(lambda s: LO.log_cfactor(lo, hi, mean[:3], s), sd[:3], 1e-7)
        np.testing.assert_allclose(cm, dm, rtol=1e-5, atol=1e-8)
        np.testing.assert_allclose(cs, ds, rtol=1e-5, atol=1e-8)


# ---------------------------------------------------------------------------------------------------------------
# the acquisition classes
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bo():
    import __graft_entry__ as g

    g.build()
    import bayesianoptimization_b200 as bo

    return bo


def test_abi_constants(bo):
    from bayesianoptimization_b200 import _lib as B

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "b200bo.h")).read()
    assert "#define B200BO_ACQ_LOGEI 6" in hdr and "#define B200BO_ACQ_LOGPOI 7" in hdr
    assert (B.ACQ_LOGEI, B.ACQ_LOGPOI) == (LO.LOGEI, LO.LOGPOI) == (6, 7)
    assert (B.ACQ_UCB, B.ACQ_EI, B.ACQ_POI, B.ACQ_NONE, B.ACQ_MES) == (0, 1, 2, 3, 4)


def test_host_base_acq_matches_the_oracle(bo, ref):
    rs = np.random.RandomState(0)
    mean = np.concatenate([rs.randn(200), [-1e3, -1e5, 0.0, 0.0, 1.0]])
    std = np.concatenate([rs.uniform(1e-3, 2.0, 200), [1.0, 1e-3, 0.0, 1e-3, 0.0]])
    ei = bo.LogExpectedImprovement(xi=0.01)
    poi = bo.LogProbabilityOfImprovement(xi=0.02)
    ei.y_max = poi.y_max = 0.5
    with np.errstate(all="ignore"):
        np.testing.assert_allclose(ei.base_acq(mean, std), LO.log_acq_term(LO.LOGEI, mean - 0.5 - 0.01, std),
                                   rtol=1e-13, atol=0)
        got = poi.base_acq(mean, std)
    want = LO.log_acq_term(LO.LOGPOI, mean - 0.5 - 0.02, std)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = np.isfinite(want)
    np.testing.assert_allclose(got[ok], want[ok], rtol=1e-13, atol=1e-300)
    assert np.array_equal(got[~ok & ~np.isnan(want)], want[~ok & ~np.isnan(want)])
    from bayesianoptimization_b200 import acquisition as A

    for lo, hi in ((-0.5, 0.5), (3.0, 4.0), (-np.inf, -2.0), (1.0, np.inf)):
        np.testing.assert_allclose(A.log_constraint_factor(mean[:200], std[:200], lo, hi),
                                   LO.log_cfactor(lo, hi, mean[:200], std[:200]), rtol=1e-13, atol=1e-15)


class _FakeGP:
    def __init__(self, f, dim=2):
        self.f, self.X_train_ = f, np.zeros((1, dim))

    def predict(self, x, return_std=True):
        return self.f(x)


def test_host_closure_combines_constraints_in_log_space(bo, ref):
    from bayesianoptimization_b200 import acquisition as A

    rs = np.random.RandomState(1)
    x = rs.uniform(size=(40, 2))
    gp = _FakeGP(lambda x: (x[:, 0] - 1.0, 0.1 + x[:, 1]))
    c1 = _FakeGP(lambda x: (x.sum(1), 0.2 + 0.0 * x[:, 0]))
    c2 = _FakeGP(lambda x: (x[:, 0] * 3.0, 0.05 + x[:, 1]))
    con = SimpleNamespace(model=[c1, c2], lb=np.array([-np.inf, 2.5]), ub=np.array([0.1, np.inf]))
    ei = bo.LogExpectedImprovement(xi=0.01)
    ei.y_max = 0.3
    vals = A._LogSpace._get_acq(ei, gp, con)(x)
    m, s = gp.f(x)
    cons = [(*c1.f(x), -np.inf, 0.1), (*c2.f(x), 2.5, np.inf)]
    want = LO.closure(LO.LOGEI, m, s, 0.3, 0.01, cons)
    np.testing.assert_allclose(vals, want, rtol=1e-13)
    assert np.all(np.isfinite(vals))  # the product form underflows to 0 here: every row would tie at -0.0
    p = np.ones(40)
    from scipy.stats import norm

    p = p * norm(loc=cons[0][0], scale=cons[0][1]).cdf(0.1) * (1 - norm(loc=cons[1][0], scale=cons[1][1]).cdf(2.5))
    assert (p == 0.0).sum() > 0


def test_class_wiring_and_device_kind(bo, ref):
    from bayesianoptimization_b200 import _lib as B
    from bayesianoptimization_b200 import acquisition as A

    ei, poi = bo.LogExpectedImprovement(xi=0.01), bo.LogProbabilityOfImprovement(xi=0.0)
    assert isinstance(ei, ref.acquisition.ExpectedImprovement) and isinstance(ei, bo.AcquisitionFunction)
    assert isinstance(poi, ref.acquisition.ProbabilityOfImprovement) and isinstance(poi, bo.AcquisitionFunction)
    assert A._device_kind(ei) == B.ACQ_LOGEI and A._device_kind(poi) == B.ACQ_LOGPOI
    assert A._device_kind(bo.ExpectedImprovement(xi=0.0)) == B.ACQ_EI  # the stock classes keep their kinds
    assert A._device_kind(bo.ProbabilityOfImprovement(xi=0.0)) == B.ACQ_POI

    class Mine(bo.LogExpectedImprovement):
        def base_acq(self, mean, std):
            return -np.abs(mean - 1.0) + np.log(std)

    assert A._device_kind(Mine(xi=0.0)) is None  # a user formula runs where the user wrote it (host, log space)
    for name in ("LogExpectedImprovement", "LogProbabilityOfImprovement"):
        assert name in bo.__all__ and getattr(bo, name) is getattr(A, name)


def test_parameters_round_trip_and_errors(bo, ref):
    from bayes_opt.exception import NoValidPointRegisteredError
    from bayes_opt.target_space import TargetSpace

    a = bo.LogExpectedImprovement(xi=0.05, exploration_decay=0.9, exploration_decay_delay=2)
    b = bo.LogExpectedImprovement(xi=1.0)
    b.set_acquisition_params(a.get_acquisition_params())
    assert b.get_acquisition_params() == a.get_acquisition_params()
    p = bo.LogProbabilityOfImprovement(xi=0.1, exploration_decay=0.5)
    q = bo.LogProbabilityOfImprovement(xi=0.0)
    q.set_acquisition_params(p.get_acquisition_params())
    assert q.get_acquisition_params() == p.get_acquisition_params()
    with pytest.raises(ValueError):
        bo.LogExpectedImprovement(xi=-1.0)
    with pytest.raises(ValueError):
        bo.LogProbabilityOfImprovement(xi=0.1, exploration_decay=2.0)
    for acq in (bo.LogExpectedImprovement(xi=0.0), bo.LogProbabilityOfImprovement(xi=0.0)):
        with pytest.raises(ValueError, match="y_max is not set"):
            acq.base_acq(np.zeros(2), np.ones(2))
    # constraints without a feasible registered point: the reference's error, from the inherited suggest
    from bayesianoptimization_b200.constraint import ConstraintModel

    space = TargetSpace(None, {"x": (0.0, 1.0)}, constraint=ConstraintModel(lambda x: x, -np.inf, -1.0))
    space.register(np.array([0.5]), 1.0, constraint_value=0.5)
    for acq in (bo.LogExpectedImprovement(xi=0.0), bo.LogProbabilityOfImprovement(xi=0.0)):
        with pytest.raises(NoValidPointRegisteredError):
            acq.suggest(gp=None, target_space=space)


def test_wrappers_take_the_log_classes(bo, ref):
    kb = bo.KrigingBeliever(bo.LogExpectedImprovement(xi=0.01))
    assert isinstance(kb.base_acquisition, bo.LogExpectedImprovement)
    kb2 = bo.KrigingBeliever(bo.LogProbabilityOfImprovement(xi=0.01))
    assert isinstance(kb2.base_acquisition, bo.LogProbabilityOfImprovement)
    cl = bo.ConstantLiar(bo.LogExpectedImprovement(xi=0.01))
    assert isinstance(cl.base_acquisition, bo.LogExpectedImprovement)
    h = bo.GPHedge([bo.LogExpectedImprovement(xi=0.01), bo.LogProbabilityOfImprovement(xi=0.01),
                    bo.UpperConfidenceBound(kappa=2.0)])
    assert [type(a).__name__ for a in h.base_acquisitions] == ["LogExpectedImprovement",
                                                               "LogProbabilityOfImprovement", "UpperConfidenceBound"]
    state = kb.get_acquisition_params()
    kb3 = bo.KrigingBeliever(bo.LogExpectedImprovement(xi=0.5))
    kb3.set_acquisition_params(state)
    assert kb3.get_acquisition_params() == state

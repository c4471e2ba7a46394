"""Trust-region Thompson sampling (TuRBO / SCBO, DESIGN.md 4.18) without a GPU: the state machine of
bayesianoptimization_b200.trust_region, the centre and the box, the host candidate sampler and its RandomState order,
the numpy restatement of the device source (tests/trust_region_oracle.py), the get/set round trip and the refusals."""
import math
import warnings

import numpy as np
import pytest

from bayesianoptimization_b200 import trust_region as T


def cfg(**kw):
    return T.TrustRegionConfig(**kw)


def fold(state, y, d, viol=None, config=None):
    return state.update(np.asarray(y, dtype=np.float64), viol, d, config or cfg())


# ---------------------------------------------------------------------------------------------- state machine


def test_first_batch_of_a_run_only_starts_it():
    s = fold(T.TrustRegionState(), [1.0, 2.0, 0.5], d=4)
    assert (s.length, s.n_success, s.n_failure, s.run_start, s.n_seen) == (0.8, 0, 0, 0, 3)
    assert not s.run_empty
    assert fold(s, [1.0, 2.0, 0.5], d=4) == s  # nothing new: unchanged


def test_success_and_failure_counters():
    y = [1.0]
    s = fold(T.TrustRegionState(), y, d=4)
    y = y + [1.0 + 1e-3 * 1.0 + 1e-9]  # beats 1 by more than 1e-3 |1|
    s = fold(s, y, d=4)
    assert (s.n_success, s.n_failure) == (1, 0)
    y = y + [1.002]  # the run's best is 1.001 + 1e-9: not 1e-3 better
    s = fold(s, y, d=4)
    assert (s.n_success, s.n_failure) == (0, 1)
    y = y + [-5.0]
    s = fold(s, y, d=4)
    assert (s.n_success, s.n_failure) == (0, 2)
    # a negative best: the margin is relative to |best|
    s2 = fold(T.TrustRegionState(), [-10.0], d=4)
    assert fold(s2, [-10.0, -9.99], d=4).n_failure == 1
    assert fold(s2, [-10.0, -9.98], d=4).n_success == 1


def test_doubling_is_capped_at_length_max():
    c = cfg(success_tolerance=3)
    s, y = fold(T.TrustRegionState(), [0.0], 4, config=c), [0.0]
    lengths = []
    for i in range(1, 13):
        y = y + [float(i)]
        s = fold(s, y, 4, config=c)
        lengths.append(s.length)
    assert lengths[:3] == [0.8, 0.8, 1.6]  # doubled after the third success, counter reset
    assert s.n_success == 0 and max(lengths) == 1.6 and lengths[-1] == 1.6


def test_halving_after_tau_fail_failures():
    d, q = 8, 1
    tau = T.failure_tolerance(d, q)
    assert tau == 8
    s, y = fold(T.TrustRegionState(), [1.0], d), [1.0]
    for i in range(tau - 1):
        y = y + [0.0]
        s = fold(s, y, d)
        assert s.length == 0.8 and s.n_failure == i + 1
    y = y + [0.0]
    s = fold(s, y, d)
    assert s.length == 0.4 and s.n_failure == 0


@pytest.mark.parametrize("d,q,tau", [(2, 1, 4), (4, 1, 4), (5, 1, 5), (16, 1, 16), (16, 8, 2), (32, 8, 4),
                                     (32, 5, 7), (3, 8, 1), (64, 16, 4)])
def test_failure_tolerance_of_d_and_q(d, q, tau):
    assert T.failure_tolerance(d, q) == tau == math.ceil(max(4, d) / q)
    # the state machine takes q from the size of the batch just folded in
    s, y = fold(T.TrustRegionState(), [1.0], d), [1.0]
    for _ in range(tau):
        y = y + [0.0] * q
        s = fold(s, y, d)
    assert s.length == 0.4


def test_fixed_failure_tolerance_overrides_the_rule():
    c = cfg(failure_tolerance=2)
    s, y = fold(T.TrustRegionState(), [1.0], 32, config=c), [1.0]
    for _ in range(2):
        y = y + [0.0]
        s = fold(s, y, 32, config=c)
    assert s.length == 0.4


def test_restart_below_length_min():
    c = cfg(length_init=0.8, length_min=0.3, failure_tolerance=1)
    s, y = fold(T.TrustRegionState(), [1.0, 0.5], 3, config=c), [1.0, 0.5]
    y = y + [0.0]
    s = fold(s, y, 3, config=c)
    assert s.length == 0.4 and s.n_restarts == 0
    y = y + [0.0, -1.0]
    s = fold(s, y, 3, config=c)  # 0.2 < 0.3: restart, the run begins at the next registered row
    assert (s.length, s.n_success, s.n_failure, s.run_start, s.n_seen, s.n_restarts) == (0.8, 0, 0, 5, 5, 1)
    assert s.run_empty
    y = y + [-3.0, -2.0]  # the random rows of the restart call start the new run
    s = fold(s, y, 3, config=c)
    assert not s.run_empty and s.run_start == 5 and s.center_index(y, None) == 6  # the old rows are forgotten


# ---------------------------------------------------------------------------------------------- centre, SCBO ranking


def test_center_without_constraints_is_the_best_row_of_the_run():
    y = np.array([5.0, 1.0, 3.0, 3.0])
    s = T.TrustRegionState(run_start=1, n_seen=4)
    assert s.center_index(y, None) == 2  # first of equal rows, the older row 0 is outside the run


def test_total_violation_matches_the_constrained_paths_rule():
    c = np.array([[0.5, 2.0], [-1.0, 0.0], [np.nan, 0.0]])
    v = T.total_violation(c, [0.0, -np.inf], [1.0, 1.0])
    assert v[0] == 1.0 and v[1] == 1.0 and np.isnan(v[2])
    assert np.array_equal(T.total_violation(np.array([0.2, 3.0]), 0.0, 1.0), [0.0, 2.0])


def test_center_with_constraints():
    y = np.array([10.0, 1.0, 2.0, 7.0])
    viol = np.array([0.5, 0.0, 0.0, 0.1])
    s = T.TrustRegionState(n_seen=4)
    assert s.center_index(y, viol) == 2  # feasible rows first, by target
    viol = np.array([0.5, 0.3, 0.3, 0.4])
    assert s.center_index(y, viol) == 1  # no feasible row: smallest violation, first of equal


def test_scbo_success_rule():
    assert T.improves(-100.0, 0.0, 50.0, 0.2)  # a feasible row beats an infeasible best
    assert not T.improves(100.0, 0.1, -50.0, 0.0)  # an infeasible row never beats a feasible best
    assert T.improves(0.0, 0.19, 0.0, 0.2) and not T.improves(0.0, 0.2, 0.0, 0.2)
    assert T.improves(2.0, 0.0, 1.0, 0.0) and not T.improves(1.0005, 0.0, 1.0, 0.0)
    s = fold(T.TrustRegionState(), [3.0], 4, viol=np.array([1.0]))
    s = fold(s, [3.0, -9.0], 4, viol=np.array([1.0, 0.0]))
    assert s.n_success == 1


# ---------------------------------------------------------------------------------------------- box


def test_box_from_isotropic_length_scale_has_equal_widths_in_data_units():
    bounds = np.array([[0.0, 1.0], [-2.0, 2.0], [10.0, 20.0]])
    lo, hi, _ = T.box([0.5, 0.0, 15.0], 0.2, 1.3, bounds)
    span = bounds[:, 1] - bounds[:, 0]
    lt = 1.3 / span
    w = lt / np.exp(np.mean(np.log(lt)))
    np.testing.assert_allclose(hi - lo, 0.2 * w * span, rtol=1e-14)
    np.testing.assert_allclose(hi - lo, (hi - lo)[0], rtol=1e-14)  # the same length scale in every column
    assert np.all(lo < [0.5, 0.0, 15.0]) and np.all(hi > [0.5, 0.0, 15.0])


def test_box_from_ard_length_scales():
    bounds = np.array([[0.0, 1.0]] * 4)
    ls = np.array([0.1, 0.2, 0.4, 0.8])
    lo, hi, _ = T.box(np.full(4, 0.5), 0.2, ls, bounds)
    w = ls / np.exp(np.mean(np.log(ls)))
    np.testing.assert_allclose(hi - lo, 0.2 * w, rtol=1e-14)
    assert math.isclose(np.prod((hi - lo) / 0.2), 1.0, rel_tol=1e-12)  # volume of the cube of side L


def test_box_is_intersected_with_shrunken_bounds():
    bounds = np.array([[0.2, 0.6], [0.0, 0.1]])  # e.g. after a bounds transformer
    lo, hi, _ = T.box([0.55, 0.05], 1.6, [0.5, 0.5], bounds)
    assert np.all(lo >= bounds[:, 0]) and np.all(hi <= bounds[:, 1])
    assert hi[0] == 0.6 and lo[1] == 0.0 and hi[1] == 0.1


def test_centre_outside_shrunken_bounds_is_clipped_and_the_box_stays_valid():
    bounds = np.array([[0.0, 1.0], [0.0, 1.0]])
    lo, hi, c = T.box([2.0, 0.5], 0.2, [0.3, 0.3], bounds)
    assert np.array_equal(c, [1.0, 0.5])
    assert np.all(lo <= c) and np.all(c <= hi) and np.all(bounds[:, 0] <= lo) and np.all(hi <= bounds[:, 1])
    assert hi[0] == 1.0 and lo[0] < 1.0  # a box of positive width at the clipped edge
    lo, hi, c = T.box([-3.0, 7.0], 1.6, [0.3, 0.3], bounds)
    assert np.array_equal(c, [0.0, 1.0]) and np.all(lo <= c) and np.all(c <= hi)


def test_centre_is_chosen_among_rows_inside_the_current_bounds():
    X = np.array([[0.5, 0.5], [2.0, 0.5], [0.9, 0.1], [0.2, 0.3]])
    y = np.array([1.0, 9.0, 3.0, 2.0])
    s = T.TrustRegionState(run_start=0, n_seen=4)
    b = np.array([[0.0, 1.0], [0.0, 1.0]])
    assert s.center_index(y, None) == 1  # without bounds: the best row, outside them
    assert s.center_index(y, None, X, b) == 2  # with bounds: as TargetSpace.mask counts rows
    assert s.center_index(y, np.array([0.0, 0.0, 0.5, 0.0]), X, b) == 3  # feasible rows inside first
    shrunk = np.array([[0.0, 0.3], [0.0, 0.2]])  # e.g. set_bounds / a bounds transformer past the whole run
    assert s.center_index(y, None, X, shrunk) is None
    assert T.TrustRegionState(run_start=3, n_seen=4).center_index(y, None, X, np.array([[0.0, 0.1], [0.0, 1.0]])) \
        is None


# ---------------------------------------------------------------------------------------------- sources


def test_perturb_probability():
    assert T.perturb_probability(1) == T.perturb_probability(20) == 1.0
    assert T.perturb_probability(32) == 19 / 31 and T.perturb_probability(64) == 19 / 63
    for d in (21, 32, 64):
        assert math.isclose(1 + T.perturb_probability(d) * (d - 1), 20.0)


def restated_host(rs, n, lo, hi, center, p):
    d = len(lo)
    U = rs.random_sample((n, d))
    V = rs.random_sample((n, d))
    f = rs.randint(0, d, n)
    out = np.empty((n, d))
    for i in range(n):
        for j in range(d):
            out[i, j] = lo[j] + (hi[j] - lo[j]) * U[i, j] if (j == f[i] or V[i, j] < p) else center[j]
    return out


@pytest.mark.parametrize("d", [1, 6, 32])
def test_host_sampler_order_and_rows(d):
    rs0 = np.random.RandomState(3)
    lo = rs0.uniform(-1, 0, d)
    hi = lo + rs0.uniform(0.1, 2, d)
    center = lo + 0.5 * (hi - lo)
    p = T.perturb_probability(d)
    n = 257
    a, b = np.random.RandomState(7), np.random.RandomState(7)
    X = T.host_candidates(a, n, lo, hi, center, p)
    R = restated_host(b, n, lo, hi, center, p)
    assert X.tobytes() == R.tobytes()
    assert a.random_sample() == b.random_sample()  # the same amount consumed
    # RNG consumption depends on n and d only
    e, f = np.random.RandomState(7), np.random.RandomState(7)
    T.host_candidates(e, n, lo, hi, center, p)
    T.host_candidates(f, n, lo * 0, hi * 0 + 5, lo * 0 + 1, 0.0)
    assert e.random_sample() == f.random_sample()
    assert np.all((X >= lo) & (X <= hi))
    assert np.all((X != center).sum(1) >= 1)  # every row perturbs its forced column


def test_host_sampler_at_p_one_is_the_box():
    d, n = 5, 100
    lo, hi = np.zeros(d), np.arange(1, d + 1, dtype=float)
    X = T.host_candidates(np.random.RandomState(1), n, lo, hi, lo, 1.0)
    U = np.random.RandomState(1).random_sample((n, d))
    assert X.tobytes() == (lo + (hi - lo) * U).tobytes()


@pytest.mark.parametrize("d", [6, 20])
def test_oracle_tr_source_equals_philox_uniform_at_d_le_20(d):
    from oracle.gp_oracle import philox_uniform
    from trust_region_oracle import philox_tr

    rows = np.arange(1000, 1300)
    lo, hi = -np.ones(d), np.linspace(0.5, 2.0, d)
    X = philox_tr(0xDEADBEEF12345, rows, d, lo, hi, np.zeros(d), T.perturb_probability(d))
    assert X.tobytes() == philox_uniform(0xDEADBEEF12345, rows, d, lo, hi).tobytes()


def _scalar_tr(seed, row, j, d, lo, hi, center, p):
    """One coordinate of the trust-region source from Philox4x32-10 calls on scalars: lanes 0, 1 and 2 restated
    without the oracle's vectorised helpers."""
    from oracle.gp_oracle import philox4x32_10

    s0, s1, r0, r1 = seed & 0xFFFFFFFF, seed >> 32, row & 0xFFFFFFFF, row >> 32

    def word(lane, c2, col):
        o = [int(v) for v in philox4x32_10(np.uint64(r0), np.uint64(r1), np.uint64(c2), np.uint64(lane), s0, s1)]
        return o[0] | (o[1] << 32) if col % 2 == 0 else o[2] | (o[3] << 32)

    u = (word(0, j // 2, j) >> 11) * 2.0**-53
    x = lo + (hi - lo) * u
    if p >= 1.0:
        return x
    o0 = int(philox4x32_10(np.uint64(r0), np.uint64(r1), np.uint64(0), np.uint64(2), s0, s1)[0])
    f = (o0 * d) >> 32
    v = (word(1, j // 2, j) >> 11) * 2.0**-53
    return x if (j == f or v < p) else center


@pytest.mark.parametrize("d", [7, 32, 64])
def test_oracle_tr_source_against_a_scalar_restatement(d):
    from trust_region_oracle import philox_tr

    seed = 0xA5A5F00D12345678
    rows = [0, 1, 2, 12345, (1 << 32) + 7, 2**40 + 3]
    lo, hi = np.linspace(-2.0, -1.0, d), np.linspace(0.5, 3.0, d)
    center = 0.5 * (lo + hi)
    for p in (T.perturb_probability(d), 0.0, 0.5):
        X = philox_tr(seed, rows, d, lo, hi, center, p)
        for i, r in enumerate(rows):
            for j in range(d):
                assert X[i, j] == _scalar_tr(seed, r, j, d, lo[j], hi[j], center[j], p)


@pytest.mark.parametrize("d", [32, 64])
def test_oracle_tr_source_follows_the_rule(d):
    from oracle.gp_oracle import philox_uniform
    from trust_region_oracle import _lane_uniform, forced_column, philox_tr

    seed, n = 987654321, 4000
    rows = np.arange(n) + (1 << 33)  # high word of the row counter in use
    lo, hi = np.full(d, -2.0), np.full(d, 3.0)
    center = np.linspace(-1.0, 2.0, d)
    p = T.perturb_probability(d)
    X = philox_tr(seed, rows, d, lo, hi, center, p)
    U = philox_uniform(seed, rows, d, lo, hi)
    V = _lane_uniform(seed, rows, d, 1)
    f = forced_column(seed, rows, d)
    assert f.min() >= 0 and f.max() < d
    for i in (0, 1, 777, n - 1):
        for j in range(d):
            want = U[i, j] if (j == f[i] or V[i, j] < p) else center[j]
            assert X[i, j] == want
    pert = (X != center).sum(1)
    assert pert.min() >= 1
    # E[count] = 1 + p (d - 1) = 20; var = p (1 - p) (d - 1)
    sd = math.sqrt(p * (1 - p) * (d - 1) / n)
    assert abs(pert.mean() - 20.0) < 5 * sd + 1e-9
    # f is close to uniform over the columns
    counts = np.bincount(f, minlength=d)
    assert counts.min() > 0.5 * n / d and counts.max() < 1.5 * n / d


# ---------------------------------------------------------------------------------------------- acquisition object


@pytest.fixture(scope="module")
def bo():
    import __graft_entry__ as g

    g.build()
    import bayesianoptimization_b200 as bo

    return bo


def test_params_round_trip(bo):
    import json

    a = bo.TrustRegionThompsonSampling(n_features=512, length_init=0.5, length_min=0.01, length_max=1.0,
                                       success_tolerance=2, failure_tolerance=3)
    a.tr_state = T.TrustRegionState(length=0.125, n_success=1, n_failure=2, run_start=7, n_seen=19, n_restarts=3)
    params = json.loads(json.dumps(a.get_acquisition_params()))
    b = bo.TrustRegionThompsonSampling()
    b.set_acquisition_params(params)
    assert b.n_features == 512 and b.tr_state == a.tr_state and b.tr_config == a.tr_config


def test_constructor_validation(bo):
    with pytest.raises(ValueError):
        bo.TrustRegionThompsonSampling(length_min=1.0, length_init=0.8)
    with pytest.raises(ValueError):
        bo.TrustRegionThompsonSampling(success_tolerance=0)
    with pytest.raises(ValueError):
        bo.TrustRegionThompsonSampling(failure_tolerance=1.5)
    with pytest.raises(ValueError):
        bo.TrustRegionThompsonSampling(length_max=float("inf"))


def test_refusals_consume_no_random_numbers(bo):
    from bayes_opt import BayesianOptimization
    from bayes_opt import acquisition as ref

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt = BayesianOptimization(f=None, pbounds={"x": (0.0, 1.0), "n": (0, 5, int)}, random_state=1,
                                   acquisition_function=bo.TrustRegionThompsonSampling(), verbose=0)
    for x, n in ((0.1, 1), (0.7, 3)):
        opt.register(params={"x": x, "n": n}, target=x + n)
    rs = np.random.RandomState(5)
    before = rs.get_state()[1].copy(), rs.get_state()[2]
    with pytest.raises(NotImplementedError):
        opt._acquisition_function.suggest(opt._gp, opt._space, random_state=rs)
    assert np.array_equal(rs.get_state()[1], before[0]) and rs.get_state()[2] == before[1]
    tr = bo.TrustRegionThompsonSampling()
    for wrap in (lambda a: bo.ConstantLiar(a), lambda a: bo.GPHedge([a]), lambda a: bo.KrigingBeliever(a),
                 lambda a: bo.acquisition.accelerate(ref.ConstantLiar(a))):
        with pytest.raises(TypeError, match="TrustRegionThompsonSampling"):
            wrap(tr)

"""Trust-region Thompson sampling on the device (DESIGN.md 4.18): the trust-region candidate source against its numpy
restatement (tests/trust_region_oracle.py), selection over device candidates against the same rows uploaded from the
host, and TrustRegionThompsonSampling through the reference's BayesianOptimization driver (both candidate sources,
both refine modes, SCBO without a feasible point, save/load resume)."""
import ctypes as C
import warnings

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import RBF, Matern

from bayesianoptimization_b200 import trust_region as T
from trust_region_oracle import _lane_uniform, forced_column, philox_tr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _box(d, seed=0):
    rs = np.random.RandomState(seed)
    lo = rs.uniform(-2.0, 0.0, d)
    hi = lo + rs.uniform(0.05, 3.0, d)
    center = lo + rs.uniform(0.0, 1.0, d) * (hi - lo)
    return lo, hi, center


def _tr_rows(bo, seed, lo, hi, center, p, idx):
    B = bo._lib
    d = len(lo)
    idx = np.ascontiguousarray(idx, dtype=np.int64)
    out = np.empty((len(idx), d))
    B.check(B.lib().b200bo_philox_tr_rows(0, seed, B.as_dp(B.c_f64(lo)), B.as_dp(B.c_f64(hi)),
                                          B.as_dp(B.c_f64(center)), float(p), d,
                                          idx.ctypes.data_as(C.POINTER(C.c_int64)), len(idx), B.as_dp(out)))
    return out


@pytest.mark.parametrize("d", [6, 20, 32, 64])
def test_tr_rows_bit_equal_to_the_oracle(bo, d):
    lo, hi, center = _box(d, d)
    p = T.perturb_probability(d)
    seed = 0x0123456789ABCDEF + d
    idx = np.concatenate([np.arange(0, 700), (1 << 32) + np.arange(-50, 50), [2**40 + 3]])
    got = _tr_rows(bo, seed, lo, hi, center, p, idx)
    want = philox_tr(seed, idx, d, lo, hi, center, p)
    assert got.tobytes() == want.tobytes()
    # in the box, and equal to the centre outside the perturbed columns
    assert np.all((got >= lo) & (got <= hi))
    if p < 1.0:
        mask = (_lane_uniform(seed, idx, d, 1) < p) | (np.arange(d)[None, :] == forced_column(seed, idx, d)[:, None])
        assert np.array_equal(got[~mask], np.broadcast_to(center, got.shape)[~mask])
        assert np.all(mask.sum(1) >= 1)
    else:  # d <= 20: the plain Philox source over the box
        from oracle.gp_oracle import philox_uniform

        assert got.tobytes() == philox_uniform(seed, idx, d, lo, hi).tobytes()
    # other values of p, 0 included (only the forced column moves)
    for pp in (0.0, 0.37):
        got = _tr_rows(bo, seed, lo, hi, center, pp, idx[:200])
        assert got.tobytes() == philox_tr(seed, idx[:200], d, lo, hi, center, pp).tobytes()
        if pp == 0.0:
            assert np.all((got != center).sum(1) <= 1)


def test_tr_arguments_are_validated(bo):
    lo, hi, center = _box(4)
    for args in ((lo, hi, hi + 1.0, 0.5), (lo, hi, center, 1.5), (lo, hi, center, -0.1), (lo, hi, center, np.nan),
                 (lo, hi * np.inf, center, 0.5), (hi, lo - 1.0, center, 0.5)):
        with pytest.raises(ValueError):
            _tr_rows(bo, 1, *args, np.arange(4))


def _gp(bo, n, d, seed, nu=2.5, ls=None):
    rs = np.random.RandomState(seed)
    X = rs.uniform(-2.0, 1.0, size=(n, d))
    y = np.sin(X @ rs.uniform(0.5, 1.5, d)) + 0.1 * rs.randn(n)
    k = RBF(ls or 0.8 * np.sqrt(d)) if nu == np.inf else Matern(ls or 0.8 * np.sqrt(d), nu=nu)
    return bo.B200GaussianProcessRegressor(kernel=k, alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)


def _compare_selection(paths, d, q, m, k, base, seed, lo, hi, center, p):
    bi, bv, bx, ti, tx = paths.argmin_topk_philox_tr(seed, lo, hi, center, p, m, k, index_base=base)
    X = philox_tr(seed, np.arange(base, base + m), d, lo, hi, center, p)
    hi_, hv, hti = paths.argmin_topk(X, k)
    assert np.array_equal(bi, hi_ + base)
    assert bv.tobytes() == hv.tobytes()
    assert bx.tobytes() == X[hi_].tobytes()
    for p_ in range(q):
        assert np.array_equal(ti[p_], hti[p_] + base)
        assert tx[p_].tobytes() == X[hti[p_]].tobytes()


@pytest.mark.parametrize("q", [1, 4, 16])
@pytest.mark.parametrize("d", [6, 24])
def test_selection_over_device_tr_candidates_equals_host_rows(bo, q, d):
    gp = _gp(bo, 300, d, seed=q + d)
    paths = gp.sample_paths(q, 512, random_state=3)
    lo, hi, center = _box(d, 7)
    p = T.perturb_probability(d)
    _compare_selection(paths, d, q, m=128 * 23 + 37, k=10, base=5_000_017, seed=99 + q, lo=lo, hi=hi, center=center,
                       p=p)


def test_selection_over_several_tiles_per_cta(bo):
    d, q = 24, 4
    paths = _gp(bo, 300, d, seed=9).sample_paths(q, 512, random_state=5)
    lo, hi, center = _box(d, 3)
    # 128 * 132 * 2 + ragged: every CTA of the persistent grid strides over several tiles
    _compare_selection(paths, d, q, m=70_001, k=10, base=17, seed=4, lo=lo, hi=hi, center=center,
                       p=T.perturb_probability(d))


@pytest.mark.parametrize("m", [128 * 40 + 101, 2 * 8 * 128 * 132 + 1001])
def test_constrained_selection_over_device_tr_candidates_equals_host_rows(bo, m):
    from bayesianoptimization_b200.paths import ConstrainedPaths

    d, q = 24, 4
    gps = [_gp(bo, 250, d, seed=s, nu=nu) for s, nu in ((1, 2.5), (2, 1.5), (3, np.inf))]
    sets = [g.sample_paths(q, 512, random_state=10 + i) for i, g in enumerate(gps)]
    lo, hi, center = _box(d, 11)
    # bounds that split the box's candidates into feasible and infeasible ones
    Xb = philox_tr(5, np.arange(2000), d, lo, hi, center, T.perturb_probability(d))
    c1, c2 = sets[1](Xb).ravel(), sets[2](Xb).ravel()
    cp = ConstrainedPaths(sets[0], sets[1:], [np.quantile(c1, 0.3), -np.inf], [np.inf, np.quantile(c2, 0.7)])
    # the larger m spans three chunks of the constrained selection on a 132-SM H100 (index_base + c0 per chunk)
    _compare_selection(cp, d, q, m=m, k=12, base=123_456, seed=5, lo=lo, hi=hi, center=center,
                       p=T.perturb_probability(d))


def test_plain_and_tr_sources_agree_at_d_le_20(bo):
    d, q = 16, 4
    paths = _gp(bo, 200, d, seed=4).sample_paths(q, 256, random_state=1)
    lo, hi, center = _box(d, 2)
    a = paths.argmin_topk_philox_tr(77, lo, hi, center, 1.0, 10_000, 8, index_base=31)
    b = paths.argmin_topk_philox(77, np.stack([lo, hi], 1), 10_000, 8, index_base=31)
    for u, v in zip(a[:3], b[:3]):
        assert np.asarray(u).tobytes() == np.asarray(v).tobytes()


# ---------------------------------------------------------------------------------------------- live optimiser

D_LIVE = 24


def _levy(**kw):
    x = np.array([kw[f"x{i:02d}"] for i in range(D_LIVE)])
    w = 1 + (x - 1) / 4
    t = np.sin(np.pi * w[0]) ** 2 + ((w[-1] - 1) ** 2) * (1 + np.sin(2 * np.pi * w[-1]) ** 2)
    t += np.sum((w[:-1] - 1) ** 2 * (1 + 10 * np.sin(np.pi * w[:-1] + 1) ** 2))
    return -float(t)


PB = {f"x{i:02d}": (-5.0, 10.0) for i in range(D_LIVE)}


def _optimizer(bo, ref, source, refine, seed=3, **tr):
    opt = ref.BayesianOptimization(f=None, pbounds=PB, random_state=seed, verbose=0,
                                   acquisition_function=bo.TrustRegionThompsonSampling(n_features=1024, **tr))
    return bo.enable(opt, candidate_source=source, refine=refine)


def _in_box(x, box):
    return box is not None and np.all(x >= box[0]) and np.all(x <= box[1])


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
@pytest.mark.parametrize("refine", ["stencil", "analytic"])
def test_live_run_stays_in_its_boxes_and_replays_on_the_cpu(bo, ref, source, refine):
    # a short failure tolerance and a high length_min, so that the run halves and restarts within 30 steps
    cfg = dict(length_min=0.2, failure_tolerance=2)
    opt = _optimizer(bo, ref, source, refine, **cfg)
    acq = opt._acquisition_function
    rs = np.random.RandomState(0)
    for _ in range(4):
        p = opt.space.array_to_params(opt.space.random_sample(1, rs)[0])
        opt.register(params=p, target=_levy(**p))
    seen, states = [], []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for _ in range(30):
            n_before = len(opt.space)
            p = opt.suggest()
            x = opt.space.params_to_array(p)
            seen.append(n_before)
            states.append(acq.tr_state)
            if acq.last_box is not None:
                assert _in_box(x, acq.last_box)
            else:
                assert acq.tr_state.run_empty  # a restart call: a random point of the space
            opt.register(params=p, target=_levy(**p))
        # replay the state machine on the registered rows
        s = T.TrustRegionState(length=acq.tr_config.length_init)
        for n, st in zip(seen, states):
            s = s.update(opt.space.target[:n], None, D_LIVE, acq.tr_config)
            assert s == st
        print(f"{source}/{refine}: restarts {s.n_restarts}, final length {s.length}, best {opt.max['target']:.3f}")
        assert s.n_restarts >= 1 or s.length < 0.8
        batch = bo.suggest_batch(opt, 8)
    X = np.array([opt.space.params_to_array(p) for p in batch])
    assert len({x.tobytes() for x in X}) == 8
    if acq.last_box is not None:
        assert all(_in_box(x, acq.last_box) for x in X)


def test_scbo_suggests_before_any_feasible_point(bo, ref):
    from scipy.optimize import NonlinearConstraint

    d = 8
    pb = {f"x{i}": (0.0, 1.0) for i in range(d)}

    def f(**kw):
        return float(-np.sum((np.array(list(kw.values())) - 0.3) ** 2))

    def c(**kw):
        return float(np.sum(np.array(list(kw.values()))))

    opt = ref.BayesianOptimization(f=f, pbounds=pb, constraint=NonlinearConstraint(c, -np.inf, 1.0), random_state=2,
                                   verbose=0, acquisition_function=bo.TrustRegionThompsonSampling(n_features=1024))
    opt = bo.enable(opt, candidate_source="device_philox")
    for v in (0.6, 0.7, 0.8):  # sum = 8 v > 1: infeasible
        opt.probe({k: v for k in pb}, lazy=False)
    assert not opt.space.mask.any()
    acq = opt._acquisition_function
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for _ in range(12):
            p = opt.suggest()
            x = opt.space.params_to_array(p)
            assert acq.last_box is None or _in_box(x, acq.last_box)
            opt.probe(p, lazy=False)
    print(f"feasible points after 12 SCBO steps: {int(opt.space.mask.sum())}")
    assert opt.space.mask.any()


def test_save_and_load_resume_the_run(bo, ref, tmp_path):
    a = _optimizer(bo, ref, "device_philox", "stencil", seed=8)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        rs = np.random.RandomState(1)
        for _ in range(3):
            p = a.space.array_to_params(a.space.random_sample(1, rs)[0])
            a.register(params=p, target=_levy(**p))
        for _ in range(6):
            p = a.suggest()
            a.register(params=p, target=_levy(**p))
        path = tmp_path / "state.json"
        a.save_state(path)
        b = _optimizer(bo, ref, "device_philox", "stencil", seed=8)
        b.load_state(path)
        assert b._acquisition_function.tr_state == a._acquisition_function.tr_state
        assert a.suggest() == b.suggest()
        assert b._acquisition_function.tr_state == a._acquisition_function.tr_state


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
def test_centre_outside_shrunken_bounds(bo, ref, source):
    """set_bounds past the run's best, and a point registered outside the bounds: the centre is taken among the rows
    inside the current bounds (or clipped into them), so the box stays valid and inside the bounds."""
    opt = _optimizer(bo, ref, source, "stencil", seed=4)
    acq = opt._acquisition_function
    rs = np.random.RandomState(2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for _ in range(5):
            p = opt.space.array_to_params(opt.space.random_sample(1, rs)[0])
            opt.register(params=p, target=_levy(**p))
        for _ in range(3):
            p = opt.suggest()
            opt.register(params=p, target=_levy(**p))
        best = opt.space.params[int(np.argmax(opt.space.target))]
        # bounds that exclude the best row in every column
        new = {k: ((-5.0, b - 0.5) if b > 0.0 else (b + 0.5, 10.0)) for k, b in zip(opt.space.keys, best)}
        opt.set_bounds(new)
        outside = {k: (v[1] + 1.0 if v[1] < 10.0 else v[0] - 1.0) for k, v in new.items()}
        opt.register(params=outside, target=1e6)  # better than anything, outside the bounds
        bnd = opt.space.bounds
        for _ in range(6):
            p = opt.suggest()
            x = opt.space.params_to_array(p)
            assert np.all(x >= bnd[:, 0]) and np.all(x <= bnd[:, 1])
            if acq.last_box is not None:
                lo, hi = acq.last_box
                assert np.all(lo <= hi) and np.all(lo >= bnd[:, 0]) and np.all(hi <= bnd[:, 1])
                assert _in_box(x, acq.last_box)
            opt.register(params=p, target=_levy(**p))


def test_sequential_domain_reduction_with_restarts(bo, ref):
    """A bounds transformer shrinks the bounds around the global best after every step while the trust region
    restarts often: every suggestion stays inside the bounds of its step."""
    from bayes_opt import SequentialDomainReductionTransformer

    pb = {f"x{i:02d}": (-5.0, 10.0) for i in range(D_LIVE)}
    opt = ref.BayesianOptimization(
        f=_levy, pbounds=pb, random_state=6, verbose=0,
        bounds_transformer=SequentialDomainReductionTransformer(minimum_window=0.5),
        acquisition_function=bo.TrustRegionThompsonSampling(n_features=512, length_min=0.3, failure_tolerance=1))
    opt = bo.enable(opt, candidate_source="device_philox")
    acq = opt._acquisition_function
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt.maximize(init_points=4, n_iter=0)
        for _ in range(20):
            bnd = opt.space.bounds.copy()
            p = opt.suggest()
            x = opt.space.params_to_array(p)
            assert np.all(x >= bnd[:, 0]) and np.all(x <= bnd[:, 1])
            opt.probe(p, lazy=False)
            opt.set_bounds(opt._bounds_transformer.transform(opt.space))  # as maximize() does after each step
    print(f"restarts {acq.tr_state.n_restarts}")
    assert acq.tr_state.n_restarts >= 1

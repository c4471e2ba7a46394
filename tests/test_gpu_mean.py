"""The posterior-mean merit on the device (B200BO_ACQ_MEAN, DESIGN.md 4.17): the mean-only tile kernel against
b200bo_gp_predict (bit for bit) and sklearn on every covariance variant, host / device / Philox candidates, the merit
and selection against the restatement (tests/mean_oracle.py), the gradient, PosteriorMean inside the reference's
optimizer, and recommend() leaving a live run untouched."""
import copy
import ctypes as C
import types
import warnings

import numpy as np
import pytest
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import ConstantKernel, Matern, WhiteKernel

import kernel_matrix_cases as KM
import mean_oracle as MO
from grad_oracle import GradGP

pytestmark = pytest.mark.gpu

ALPHA = 1e-6
TILE = {"B200BO_SMALL_PATH": "0"}


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


def _mean_acq(bo, gp, con=None):
    return bo.FusedAcquisition(bo._lib.ACQ_MEAN, gp, con)


def _alpha(gp):
    return np.asarray(gp.alpha_, dtype=float)


def _T(gp):
    from bayesianoptimization_b200.gpr import parse_kernel

    const = parse_kernel(gp.kernel_).const_value
    return MO.bound_T(float(np.ravel(gp._y_train_mean)[0]), float(np.ravel(gp._y_train_std)[0]), const, _alpha(gp))


# ---------------------------------------------------------------------------------------------------------------
# the tile kernel's mu: bit-equal to b200bo_gp_predict, within 1e-10 of sklearn, the same bits on an fp32 handle
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", sorted(KM.PREDICT))
def test_tile_mu_matches_predict_and_sklearn(bo, monkeypatch, cid):
    for k, v in TILE.items():
        monkeypatch.setenv(k, v)
    c = KM.PREDICT[cid]
    n, d = c["n"], c["d"]
    X, y, rs = KM.problem(c, n, d, 300 + sorted(KM.PREDICT).index(cid))
    xt = np.vstack([KM.inputs(c, 3000, d, rs), X[:16]])  # 24 tiles, training rows included
    k = KM.kernel(c, d)
    gp = bo.B200GaussianProcessRegressor(kernel=k, alpha=ALPHA, normalize_y=True, optimizer=None).fit(X, y)
    mu_pred, _ = _quiet(gp.predict, xt, return_std=True)
    mu = -_mean_acq(bo, gp)(xt)
    assert np.array_equal(mu, mu_pred)
    sk = GaussianProcessRegressor(kernel=k, alpha=ALPHA, normalize_y=True, optimizer=None).fit(X, y)
    mu_sk = _quiet(sk.predict, xt)
    err = float(np.max(np.abs(mu - mu_sk) / (np.abs(mu_sk) + sk._y_train_std)))
    print(f"\n{cid} mu vs sklearn {err:.1e}")
    assert err <= 1e-10
    gp32 = bo.B200GaussianProcessRegressor(kernel=k, alpha=ALPHA, normalize_y=True, optimizer=None,
                                           precision="fp32").fit(X, y)
    assert np.array_equal(-_mean_acq(bo, gp32)(xt), mu)


# ---------------------------------------------------------------------------------------------------------------
# constrained merit, selection, candidate sources
# ---------------------------------------------------------------------------------------------------------------
def _fit(bo, X, y, c, ls, noise=0.0, devices=None):
    k = ConstantKernel(c, "fixed") * Matern(length_scale=ls, nu=2.5, length_scale_bounds="fixed")
    if noise:
        k = k + WhiteKernel(noise, "fixed")
    return bo.B200GaussianProcessRegressor(kernel=k, alpha=ALPHA, normalize_y=True, optimizer=None,
                                           devices=devices).fit(X, y)


def _constrained(bo, J, d=5, n=300, seed=0, lb=None, ub=None, devices=None):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    s = X.sum(1)
    tgt = _fit(bo, X, np.sin(3 * s) + 0.05 * rs.randn(n), 1.5, 0.4, 1e-3, devices)
    gps = [_fit(bo, X, np.cos((j + 1) * s + X[:, j % d]) + 0.02 * rs.randn(n), 1.0, 0.5, devices=devices)
           for j in range(J)]
    lb = [-0.5, -np.inf, -0.8, -0.2, -np.inf, -1.0, -0.3][:J] if lb is None else lb
    ub = [0.5, 0.3, np.inf, 0.9, 0.4, 0.0, np.inf][:J] if ub is None else ub
    con = types.SimpleNamespace(model=gps, lb=np.array(lb, float), ub=np.array(ub, float))
    return X, tgt, con, rs


def _oracle_values(bo, tgt, con, xt):
    """The restatement on the device's own means (b200bo_gp_predict, tile path) and T."""
    mu0 = _quiet(tgt.predict, xt)
    cm = [_quiet(g.predict, xt) for g in con.model]
    return MO.value(mu0, cm, con.lb, con.ub, _T(tgt)), MO.violation(cm, con.lb, con.ub, len(xt))


@pytest.mark.parametrize("J", [1, 2, 7])
def test_merit_and_selection_match_the_restatement(bo, monkeypatch, J):
    for k, v in TILE.items():
        monkeypatch.setenv(k, v)
    X, tgt, con, rs = _constrained(bo, J, seed=J)
    xt = rs.uniform(size=(20000, X.shape[1]))
    acq = _mean_acq(bo, tgt, con)
    v = acq(xt)
    ref, viol = _oracle_values(bo, tgt, con, xt)
    feas = viol == 0
    print(f"\nJ={J}: {feas.sum()} of {len(xt)} mean-feasible")
    assert 0 < feas.sum() < len(xt)
    assert np.array_equal(v[feas], ref[feas])  # -mu_0, bit for bit
    np.testing.assert_allclose(v[~feas], ref[~feas], rtol=1e-14)  # T from A1 summed in another order
    assert v[feas].max() < v[~feas].min()
    idx, val, top = acq.argmin_topk(xt, 10)
    order = np.argsort(v, kind="stable")
    assert idx == int(np.argmin(v)) and val == v[idx] and list(top) == list(order[:10])


def test_no_feasible_candidate_and_infinite_bounds(bo, monkeypatch):
    for k, v in TILE.items():
        monkeypatch.setenv(k, v)
    X, tgt, con, rs = _constrained(bo, 2, lb=[5.0, -np.inf], ub=[6.0, np.inf])
    xt = rs.uniform(size=(5000, X.shape[1]))
    v = _mean_acq(bo, tgt, con)(xt)
    ref, viol = _oracle_values(bo, tgt, con, xt)
    assert np.all(viol > 0)
    np.testing.assert_allclose(v, ref, rtol=1e-14)
    idx, _, top = _mean_acq(bo, tgt, con).argmin_topk(xt, 5)
    assert idx == int(np.argmin(viol)) or viol[idx] == viol.min()


def test_host_device_and_philox_candidates_agree(bo):
    import torch

    X, tgt, con, rs = _constrained(bo, 2)
    d = X.shape[1]
    acq = _mean_acq(bo, tgt, con)
    lo, hi = np.full(d, -0.2), np.full(d, 1.2)
    m, k, seed = 300_000, 16, 1234
    bi, bv, bx, ti, tx = acq.argmin_topk_philox(seed, np.column_stack([lo, hi]), m, k)
    rows = np.empty((m, d))
    idx = np.arange(m, dtype=np.int64)
    bo._lib.check(bo._lib.lib().b200bo_philox_rows(0, seed, bo._lib.as_dp(lo), bo._lib.as_dp(hi), d,
                                                   idx.ctypes.data_as(C.POINTER(C.c_int64)), m, bo._lib.as_dp(rows)))
    hi_i, hi_v, hi_top = acq.argmin_topk(rows, k)
    assert (bi, bv, list(ti)) == (hi_i, hi_v, list(hi_top))
    assert np.array_equal(bx, rows[bi]) and np.array_equal(tx, rows[ti])
    # device-resident candidates: values and records of the host path
    v = acq(rows)
    Xd = torch.from_numpy(rows).cuda()
    out = torch.empty(m, dtype=torch.float64, device="cuda")
    mu = torch.empty(m, dtype=torch.float64, device="cuda")
    sel = torch.empty(2 * (k + 1), dtype=torch.float64, device="cuda")
    spec = acq.spec
    bo._lib.check(bo._lib.lib().b200bo_acq_eval_dev(C.byref(spec), Xd.data_ptr(), m, out.data_ptr(), mu.data_ptr(),
                                                    None, k, sel.data_ptr(), 0, None))
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), v)
    assert np.array_equal(mu.cpu().numpy(), _quiet(tgt.predict, rows))
    rec = sel.cpu().numpy().view(np.int64).reshape(-1, 2)[:, 1]
    assert rec[0] == hi_i and list(rec[1:]) == list(hi_top)
    # sd is refused
    sd = torch.empty(m, dtype=torch.float64, device="cuda")
    assert bo._lib.lib().b200bo_acq_eval_dev(C.byref(spec), Xd.data_ptr(), m, out.data_ptr(), None, sd.data_ptr(), 0,
                                             None, 0, None) == bo._lib.ERR_ARG


def test_illbig_mu_against_truth(bo, monkeypatch):
    from oracle import make_illcond as MI
    from oracle import make_illcond_big as MB
    from test_gpu_illcond import C_SK, FLOOR
    from test_gpu_illcond_big import PREDICT_BAR

    for k, v in TILE.items():
        monkeypatch.setenv(k, v)
    for name in sorted(MB.CASES):
        c, r = MB.CASES[name], MB.load(name)
        gp = bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True,
                                             optimizer=None).fit(r["X"], r["y"])
        mu = -_mean_acq(bo, gp)(r["xt"])
        e = float(np.max(np.abs(mu - r["mu"]) / (np.abs(r["mu"]) + r["y_std"])))
        e_sk = float(np.max(np.abs(r["sk_mu"] - r["mu"]) / (np.abs(r["mu"]) + r["y_std"])))
        print(f"\n{name} mu {e:.1e} sklearn {e_sk:.1e}")
        assert e <= max(C_SK["mu"] * e_sk, FLOOR["mu"]) and e <= PREDICT_BAR[name]


# ---------------------------------------------------------------------------------------------------------------
# gradient
# ---------------------------------------------------------------------------------------------------------------
def test_value_and_grad_match_the_oracle(bo):
    rs = np.random.RandomState(4)
    d, n = 4, 200
    X = rs.uniform(size=(n, d))
    s = X.sum(1)
    ys = [np.sin(3 * s), np.cos(2 * s), X[:, 0] - X[:, 1]]
    pars = [(1.4, 0.5), (1.0, 0.6), (0.8, 0.7)]
    gps = [_fit(bo, X, yy, c, ls) for yy, (c, ls) in zip(ys, pars)]
    ggs = [GradGP(X, yy, 2.5, ls, const=c, alpha=ALPHA) for yy, (c, ls) in zip(ys, pars)]
    lb, ub = [-0.3, -np.inf], [0.4, 0.2]
    con = types.SimpleNamespace(model=gps[1:], lb=np.array(lb), ub=np.array(ub))
    xt = rs.uniform(size=(150, d))
    for cc in (None, con):
        acq = _mean_acq(bo, gps[0], cc)
        val, grad = acq.value_and_grad(xt)
        cons = [] if cc is None else [(g, lo, hi) for g, lo, hi in zip(ggs[1:], lb, ub)]
        rv, rg = MO.value_grad(ggs[0], xt, cons)
        np.testing.assert_allclose(val, acq(xt), rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(val, rv, rtol=1e-9, atol=1e-10)
        np.testing.assert_allclose(grad, rg, rtol=1e-7, atol=1e-8 * np.max(np.abs(rg)))


# ---------------------------------------------------------------------------------------------------------------
# PosteriorMean and recommend() in the reference's optimizer
# ---------------------------------------------------------------------------------------------------------------
def _opt(bo, ref, acq, seed=1, constraint=None, noise=0.05, **enable):
    rs = np.random.RandomState(seed + 100)

    def f(x, y):
        return -(x - 0.3) ** 2 - (y + 0.2) ** 2 + noise * rs.randn()

    opt = ref.BayesianOptimization(f=f, pbounds={"x": (-1, 1), "y": (-1, 1)}, acquisition_function=acq,
                                   constraint=constraint, random_state=seed, verbose=0)
    opt.set_gp_params(kernel=Matern(nu=2.5) + WhiteKernel(1e-3), alpha=1e-6)
    bo.enable(opt, **enable)
    if constraint is not None:
        for m in opt.constraint.model:
            m.set_params(kernel=Matern(nu=2.5) + WhiteKernel(1e-3))
    return opt


def test_posterior_mean_suggestions_match_a_host_closure(bo, ref):
    acq = bo.PosteriorMean()
    opt = _opt(bo, ref, acq, noise=0.0)
    opt.set_gp_params(kernel=Matern(nu=2.5, length_scale=0.5, length_scale_bounds="fixed"), optimizer=None)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt.maximize(init_points=5, n_iter=0)
        for _ in range(3):
            rs_host = copy.deepcopy(opt._random_state)
            X, y = opt.space.params, opt.space.target
            sk = GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.5, length_scale_bounds="fixed"),
                                          alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)

            def host(x):
                return -sk.predict(x.reshape(-1, 2))

            want = ref.acquisition.AcquisitionFunction._acq_min(acq, host, opt.space, random_state=rs_host)
            got = opt.suggest()
            np.testing.assert_allclose(opt.space.params_to_array(got), want, atol=1e-4)
            a, b = opt._random_state.get_state(legacy=False), rs_host.get_state(legacy=False)
            assert np.array_equal(a["state"]["key"], b["state"]["key"]) and a["state"]["pos"] == b["state"]["pos"]
            opt.probe(params=got, lazy=False)


def test_posterior_mean_modes_and_refusals(bo, ref):
    for kw in ({"refine": "analytic"}, {"candidate_source": "device_philox"}):
        opt = _opt(bo, ref, bo.PosteriorMean(), **kw)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            opt.maximize(init_points=4, n_iter=2)
        assert len(opt.space) == 6
    for wrap in (lambda a: bo.ConstantLiar(a), lambda a: bo.GPHedge([a]), lambda a: bo.KrigingBeliever(a),
                 lambda a: bo.PendingNEI(a)):
        with pytest.raises(TypeError):
            wrap(bo.PosteriorMean())
    opt = ref.BayesianOptimization(f=None, pbounds={"x": (-1, 1)}, acquisition_function=ref.acquisition.ConstantLiar(
        bo.PosteriorMean()), verbose=0)
    with pytest.raises(TypeError):
        bo.enable(opt)


def _same_gp(a, b):
    assert np.array_equal(a.X_train_, b.X_train_) and np.array_equal(a._y_raw, b._y_raw)
    assert np.array_equal(a.kernel_.theta, b.kernel_.theta) and np.array_equal(a.alpha_, b.alpha_)


def test_recommend_leaves_a_live_noisy_run_untouched(bo, ref):
    from scipy.optimize import NonlinearConstraint

    def run(with_recommend):
        rs = np.random.RandomState(9)
        con = NonlinearConstraint(lambda x, y: x + y + 0.05 * rs.randn(), -np.inf, 0.5)
        acq = bo.ConstrainedNoisyExpectedImprovement(xi=0.0, n_samples=4)
        opt = _opt(bo, ref, acq, seed=2, constraint=con)
        trace, recs = [], []
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for p in range(4):
                opt.probe(params={"x": -0.8 + 0.4 * p, "y": 0.5 - 0.3 * p}, lazy=False)
            for step in range(4):
                if with_recommend:
                    recs.append((bo.recommend(opt, in_sample=True),
                                 bo.recommend(opt, in_sample=False, n_random=2000, n_smart=3, random_state=step)))
                x = opt.suggest()
                trace.append((opt.space.params_to_array(x), opt._random_state.get_state(legacy=False)))
                opt.probe(params=x, lazy=False)
        return opt, trace, recs

    a, ta, _ = run(False)
    b, tb, recs = run(True)
    for (xa, sa), (xb, sb) in zip(ta, tb):
        assert np.array_equal(xa, xb)
        assert np.array_equal(sa["state"]["key"], sb["state"]["key"]) and sa["state"]["pos"] == sb["state"]["pos"]
    _same_gp(a._gp, b._gp)
    for ga, gb in zip(a.constraint.model, b.constraint.model):
        _same_gp(ga, gb)
    # the in-sample pick is the registered row with the best restated merit on GPs fitted to the registered rows
    ins, outs = recs[-1]
    X = b.space.params[:-1]
    assert ins["params"] in [b.space.array_to_params(x) for x in X]
    assert set(ins) == {"target", "params", "std", "constraint", "allowed"}
    assert outs["allowed"] in (True, False) and np.isfinite(outs["std"])


def test_recommend_in_sample_is_the_best_oracle_merit(bo, ref):
    from scipy.optimize import NonlinearConstraint

    con = NonlinearConstraint(lambda x, y: x - y, -0.5, 0.5)
    opt = _opt(bo, ref, bo.UpperConfidenceBound(kappa=1.0), constraint=con, noise=0.1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for p in range(12):
            opt.probe(params={"x": np.sin(p), "y": np.cos(3 * p)}, lazy=False)
        gp_before = opt._gp
        r = bo.recommend(opt, random_state=0)
    assert opt._gp is gp_before and not hasattr(gp_before, "X_train_")  # never fitted by recommend
    X = opt.space.params
    # the clones recommend fits draw their restarts from random_state=0: fit the same ones here
    from bayes_opt.util import ensure_rng
    from sklearn.base import clone

    rng = ensure_rng(0)
    tg = clone(opt._gp).set_params(random_state=rng).fit(X, opt.space.target)
    cg = clone(opt.constraint.model[0]).set_params(random_state=rng).fit(X, opt.space.constraint_values.reshape(-1))
    v = MO.value(_quiet(tg.predict, X), [_quiet(cg.predict, X)], [-0.5], [0.5], _T(tg))
    best = int(np.argsort(v, kind="stable")[0])
    assert r["params"] == opt.space.array_to_params(X[best])
    assert r["allowed"] == (MO.violation([_quiet(cg.predict, X[best:best + 1])], [-0.5], [0.5], 1)[0] == 0)


def test_two_devices_are_bit_identical(bo):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    X, tgt, con, rs = _constrained(bo, 2, seed=5)
    _, tgt2, con2, _ = _constrained(bo, 2, seed=5, devices=[0, 1])
    xt = rs.uniform(size=(200_000, X.shape[1]))
    a, b = _mean_acq(bo, tgt, con), _mean_acq(bo, tgt2, con2)
    assert a.argmin_topk(xt, 10)[0] == b.argmin_topk(xt, 10)[0]
    ia, va, ta = a.argmin_topk(xt, 10)
    ib, vb, tb = b.argmin_topk(xt, 10)
    assert (ia, va, list(ta)) == (ib, vb, list(tb))
    pa, pb = a.argmin_topk_philox(7, [(0, 1)] * X.shape[1], 300_000, 8), b.argmin_topk_philox(
        7, [(0, 1)] * X.shape[1], 300_000, 8)
    assert pa[0] == pb[0] and pa[1] == pb[1] and list(pa[3]) == list(pb[3])
    assert np.array_equal(a(xt[:5000]), b(xt[:5000]))

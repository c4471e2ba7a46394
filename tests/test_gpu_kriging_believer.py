"""Kriging believer on the device (DESIGN.md 4.11): b200bo_gp_fork / b200bo_gp_condition through
B200GaussianProcessRegressor.condition_on_pending, and KrigingBeliever.suggest / suggest_batch.

Over the predict cases of tests/kernel_matrix_cases.py (every covariance code, iso and ARD, WhiteKernel, the round
transform, ragged N) and N = 4096 (no slack: every conditioning forks):
  * a fork is bit-equal to its source at the same capacity and equal to round-off across a re-pitch;
  * the conditioned mean and standard deviation for p = 1, 7, 64 pending points against the closed form from sklearn on
    the ORIGINAL GP (tests/believer_oracle.py): mu_f = mu, sigma_f^2 = sigma^2 - S(x,P) (S(P,P) + s_n^2 I)^-1 S(P,x);
  * p single-row conditions equal one p-row call bit for bit;
  * pruning on / off gives bit-equal selection records on a conditioned handle;
  * analytic gradients on a conditioned handle against the numpy restatement (tests/grad_oracle.py).
Then the acquisition: q = 1 equals the base suggest() bit for bit (UCB, EI, PoI, MES; host and Philox candidates),
q = 4 / 16 reach the optimum of a restated pipeline, a live BayesianOptimization runs the asynchronous pattern and a
save_state / load_state round trip, and a non-PD conditioning raises LinAlgError.
"""
import warnings

import numpy as np
import pytest
from sklearn.gaussian_process import GaussianProcessRegressor

import believer_oracle as BO
import grad_oracle as G
import kernel_matrix_cases as KM

pytestmark = pytest.mark.gpu

ALPHA = 1e-6
RTOL = 1e-5  # the fp64 parity bar
CASES = dict(KM.PREDICT)
CASES["n4096"] = dict(kern="m25", ard=True, const=1.3, n=4096, d=16)
# conditioned mu / variance metrics (|d mu| / (|mu| + s_y), |d var| / prior var) against the closed form, pinned at
# about 10x the error measured on an H100 80GB HBM3 at a 700 W power limit (largest over p = 1, 7, 64) and never below
# 1e-13, as in kernel_matrix_cases.  Comments: measured mu, var.
BAR = {
    "p1": 2.2e-13,  # 2.2e-14 4.7e-15
    "p2": 1e-13,  # 5.8e-15 3.7e-15
    "p3": 5e-13,  # 1.0e-14 4.9e-14
    "p4": 1e-13,  # 5.2e-15 1.9e-15
    "p5": 1.2e-12,  # 7.7e-15 1.2e-13
    "p6": 1e-13,  # 4.9e-15 1.3e-15
    "p7": 7e-12,  # 6.7e-13 7.6e-14
    "p8": 1e-13,  # 3.5e-15 1.8e-15
    "p9": 3e-11,  # 2.8e-12 5.5e-13
    "p10": 1e-13,  # 7.1e-15 3.5e-15
    "p11": 7e-12,  # 1.1e-13 7.0e-13
    "p12": 3e-13,  # 3.0e-14 3.5e-15
    "p13": 6.4e-11,  # 3.8e-13 6.4e-12
    "n4096": 2.8e-12,  # 2.1e-14 2.7e-13
}


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


_PROBLEMS = {}


def _problem(bo, name):
    """(device GP, sklearn GP, X, query rows, rs) of a case, built once per module."""
    if name not in _PROBLEMS:
        case = CASES[name]
        n, d = case["n"], case["d"]
        X, y, rs = KM.problem(case, n, d, seed=7)
        sk = GaussianProcessRegressor(kernel=KM.kernel(case, d), alpha=ALPHA, normalize_y=True, optimizer=None).fit(X, y)
        gp = bo.B200GaussianProcessRegressor(kernel=KM.kernel(case, d), alpha=ALPHA, normalize_y=True, optimizer=None)
        gp.fit(X, y)
        Xq = np.vstack([KM.inputs(case, 600, d, rs), X[:8], X[8:16] + 1e-4])
        _PROBLEMS[name] = (gp, sk, X, Xq, rs)
    return _PROBLEMS[name]


def _pending(case, X, p, rs):
    """p pending rows: uniform, with a quarter of them 1e-3 from training rows."""
    d = X.shape[1]
    P = KM.inputs(case, p, d, rs)
    k = p // 4
    P[:k] = X[rs.choice(len(X), k, replace=False)] + 1e-3 * rs.choice([-1.0, 1.0], size=(k, d))
    return P


def _metrics(case, sk, mu, sd, mu_r, sd_r):
    s_y = float(np.ravel(sk._y_train_std)[0])
    prior = ((case.get("const") or 1.0) + (case.get("white") or 0.0)) * s_y * s_y
    return float(np.max(np.abs(mu - mu_r) / (np.abs(mu_r) + s_y))), float(np.max(np.abs(sd**2 - sd_r**2)) / prior)


def _ei(bo, gp, y_max):
    return bo.FusedAcquisition(1, gp, xi=0.01, y_max=y_max)


@pytest.mark.parametrize("name", list(CASES))
def test_fork_is_bit_equal_at_the_same_capacity_and_close_across_a_repitch(bo, name):
    gp, sk, X, Xq, rs = _problem(bo, name)
    mu0, sd0 = _quiet(gp.predict, Xq, return_std=True)
    same = gp.condition_on_pending(np.empty((0, X.shape[1])))  # a fork with no extra row: np' == np
    assert same is not gp and same._handle().ptr.value != gp._handle().ptr.value
    mu1, sd1 = _quiet(same.predict, Xq, return_std=True)
    assert np.array_equal(mu0, mu1) and np.array_equal(sd0, sd1)
    y_max = float(np.max(sk.y_train_))
    cand = KM.inputs(CASES[name], 20000, X.shape[1], rs)
    r0, r1 = _ei(bo, gp, y_max).argmin_topk(cand, 10), _ei(bo, same, y_max).argmin_topk(cand, 10)
    assert r0[0] == r1[0] and r0[1] == r1[1] and np.array_equal(r0[2], r1[2])
    wide = gp.condition_on_pending(np.empty((0, X.shape[1])), extra_rows=300)  # np' > np
    mu2, sd2 = _quiet(wide.predict, Xq, return_std=True)
    dm, dv = _metrics(CASES[name], sk, mu2, sd2, mu0, sd0)
    tol = max(1e-12, CASES[name].get("bar", 0.0))
    assert dm < tol and dv < tol, (dm, dv)
    assert np.array_equal(gp.alpha_, wide.alpha_) and np.array_equal(gp.L_, wide.L_)


@pytest.mark.parametrize("name", list(CASES))
def test_conditioned_posterior_matches_the_closed_form(bo, name):
    case = CASES[name]
    gp, sk, X, Xq, rs = _problem(bo, name)
    n = X.shape[0]
    worst = [0.0, 0.0]
    for p in (1, 7, 64):
        P = _pending(case, X, p, rs)
        cg = gp.condition_on_pending(P)
        assert cg.X_train_.shape == (n + p, X.shape[1]) and gp.X_train_.shape == (n, X.shape[1])
        mu_p = _quiet(sk.predict, P)
        assert np.max(np.abs(cg._y_raw[n:] - mu_p) / (np.abs(mu_p) + sk._y_train_std)) < RTOL  # believer values
        assert np.array_equal(cg.alpha_[n:], np.zeros(p)) and np.array_equal(cg.alpha_[:n], gp.alpha_)
        mu, sd = _quiet(cg.predict, Xq, return_std=True)
        mu_r, sd_r = _quiet(BO.closed_form, sk, P, Xq)
        dm, dv = _metrics(case, sk, mu, sd, mu_r, sd_r)
        worst = [max(worst[0], dm), max(worst[1], dv)]
        print(f"BELIEVER_ERR {name} p={p} mu={dm:.2e} var={dv:.2e}")
    assert worst[0] < min(RTOL, BAR[name]) and worst[1] < min(RTOL, BAR[name]), worst


@pytest.mark.parametrize("name", ["p2", "p3", "p9", "n4096"])
def test_single_row_conditions_equal_one_call(bo, name):
    gp, sk, X, Xq, rs = _problem(bo, name)
    P = _pending(CASES[name], X, 7, rs)
    one = gp.condition_on_pending(P)
    step = gp.condition_on_pending(P[:1], extra_rows=6)
    for i in range(1, 7):
        assert step.condition_on_pending(P[i:i + 1]) is step  # in place: the fork reserved the rows
    assert np.array_equal(one.X_train_, step.X_train_) and np.array_equal(one._y_raw, step._y_raw)
    a, b = _quiet(one.predict, Xq, return_std=True), _quiet(step.predict, Xq, return_std=True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert np.array_equal(one.L_, step.L_)
    cap = -(-(X.shape[0] + 7) // 128) * 128  # the fork's padded capacity
    more = step.condition_on_pending(_pending(CASES[name], X, cap - X.shape[0] - 7 + 1, rs))
    assert more is not step and step.X_train_.shape[0] == X.shape[0] + 7  # beyond it: a new fork, step untouched
    assert more.X_train_.shape[0] == cap + 1


@pytest.mark.parametrize("name", ["p1", "p5", "p8", "n4096"])
def test_pruning_records_are_bit_equal_on_a_conditioned_handle(bo, name, monkeypatch):
    gp, sk, X, Xq, rs = _problem(bo, name)
    cg = gp.condition_on_pending(_pending(CASES[name], X, 7, rs))
    cand = KM.inputs(CASES[name], 1 << 16, X.shape[1], rs)
    y_max = float(np.max(sk.y_train_))
    for kind, kw in ((0, dict(kappa=2.576)), (1, dict(xi=0.01, y_max=y_max)), (2, dict(xi=0.01, y_max=y_max))):
        acq = bo.FusedAcquisition(kind, cg, **kw)
        monkeypatch.delenv("B200BO_PRUNE", raising=False)
        on = acq.argmin_topk(cand, 10)
        monkeypatch.setenv("B200BO_PRUNE", "0")
        off = acq.argmin_topk(cand, 10)
        monkeypatch.delenv("B200BO_PRUNE")
        assert on[0] == off[0] and on[1] == off[1] and np.array_equal(on[2], off[2]), kind


@pytest.mark.parametrize("name", ["p4", "p6", "p10", "p11", "p13"])
def test_analytic_gradients_on_a_conditioned_handle(bo, name):
    case = CASES[name]
    gp, sk, X, Xq, rs = _problem(bo, name)
    d = X.shape[1]
    P = _pending(case, X, 7, rs)
    cg = gp.condition_on_pending(P)
    nu = KM.NU[case["kern"]]
    ls, const, noise = KM.length_scale(case, d), case.get("const") or 1.0, case.get("white") or 0.0
    base = G.GradGP(X, sk._y_train_mean + sk._y_train_std * sk.y_train_, nu, ls, const, noise, ALPHA,
                    rnd=case.get("rnd", 0))
    mu_p = base.predict_grad(P)[0]
    aug = G.GradGP(np.vstack([X, P]), np.concatenate([base.y_norm, (mu_p - base.y_mean) / base.y_std]), nu, ls, const,
                   noise, ALPHA, normalize=False, rnd=case.get("rnd", 0))
    aug.y_mean, aug.y_std = base.y_mean, base.y_std  # the statistics of the fit stay
    rows = np.vstack([KM.inputs(case, 40, d, rs), P[:4] + 1e-2])
    y_max = float(np.max(sk._y_train_mean + sk._y_train_std * sk.y_train_))
    for kind, kw in ((G.UCB, dict(kappa=2.576)), (G.EI, dict(xi=0.01, y_max=y_max)), (G.POI, dict(xi=0.01, y_max=y_max))):
        val, grad = bo.FusedAcquisition(kind, cg, **kw).value_and_grad(rows)
        val_r, grad_r = G.acq_value_grad(kind, aug, rows, **kw)
        scale = np.max(np.abs(grad_r), axis=1) + np.abs(val_r) / np.min(ls) + 1e-6
        err = float(np.max(np.max(np.abs(grad - grad_r), axis=1) / scale))
        assert np.max(np.abs(val - val_r) / (np.abs(val_r) + 1e-3)) < RTOL and err < RTOL, (kind, err)


# ---- the acquisition ------------------------------------------------------------------------------------------
PB = {f"x{j}": (0.0, 1.0) for j in range(4)}


def _space(n=60, seed=3):
    from bayes_opt.target_space import TargetSpace

    space = TargetSpace(None, PB)
    rs = np.random.RandomState(seed)
    for _ in range(n):
        x = space.random_sample(random_state=rs)
        space.register(x, float(np.sin(5 * x.sum()) + np.cos(3 * x[0])))
    return space


def _gp(bo):
    from sklearn.gaussian_process.kernels import Matern

    return bo.B200GaussianProcessRegressor(kernel=Matern(length_scale=0.4, nu=2.5), alpha=1e-6, normalize_y=True,
                                           optimizer=None)


def _base(bo, kind):
    return {"ucb": lambda: bo.UpperConfidenceBound(kappa=2.576, exploration_decay=0.9),
            "ei": lambda: bo.ExpectedImprovement(xi=0.01), "poi": lambda: bo.ProbabilityOfImprovement(xi=0.01),
            "mes": lambda: bo.MaxValueEntropySearch(n_samples=4, n_features=512, n_max_candidates=4096)}[kind]()


@pytest.mark.parametrize("source", ["host_rng", "device_philox"])
@pytest.mark.parametrize("kind", ["ucb", "ei", "poi", "mes"])
def test_q1_equals_suggest(bo, ref, kind, source):
    space, out = _space(), []
    for batch in (True, False):
        base = _base(bo, kind)
        base.b200_candidate_source = source
        rs = np.random.RandomState(11)
        if batch:
            x = _quiet(bo.KrigingBeliever(base).suggest_batch, _gp(bo), space, 1, n_random=5000, n_smart=3,
                       random_state=rs)[0]
        else:
            x = _quiet(base.suggest, _gp(bo), space, n_random=5000, n_smart=3, random_state=rs)
        out.append((x, rs.get_state()))
    assert np.array_equal(out[0][0], out[1][0])
    assert np.array_equal(out[0][1][1], out[1][1][1]) and out[0][1][2:] == out[1][1][2:]


@pytest.mark.parametrize("q", [4, 16])
@pytest.mark.parametrize("kind", ["ucb", "ei"])
def test_batch_reaches_the_optimum_of_a_restated_pipeline(bo, ref, kind, q):
    """Round j of the restatement: the numpy-conditioned posterior on the device's picks 0..j-1, the same candidates,
    the same random stage, SciPy L-BFGS-B from its top-n_smart.  The device's pick j is at least as good (to optimiser
    tolerance) as the restated round's best, and the picks are distinct."""
    from scipy.optimize import minimize
    from scipy.stats import norm

    space = _space()
    base = _base(bo, kind)
    kb = bo.KrigingBeliever(base)
    rs = np.random.RandomState(5)
    picks = _quiet(kb.suggest_batch, _gp(bo), space, q, n_random=3000, n_smart=3, random_state=rs)
    assert picks.shape == (q, 4) and len({p.tobytes() for p in picks}) == q
    rs = np.random.RandomState(5)
    cand = space.random_sample(3000, random_state=rs)
    sk = GaussianProcessRegressor(kernel=_gp(bo).kernel, alpha=1e-6, normalize_y=True, optimizer=None)
    sk.fit(space.params, space.target)
    ym, ys = float(np.ravel(sk._y_train_mean)[0]), float(np.ravel(sk._y_train_std)[0])
    y_max, kappa = float(space.target.max()), 2.576
    for j in range(q):
        P = picks[:j]
        aug = GaussianProcessRegressor(kernel=sk.kernel_, alpha=1e-6, optimizer=None).fit(
            np.vstack([sk.X_train_, P]), np.concatenate([sk.y_train_, BO.believer_targets(sk, P)]) if j else sk.y_train_)

        def neg_acq(x, aug=aug):
            mu, sd = aug.predict(np.atleast_2d(x), return_std=True)
            mu, sd = mu * ys + ym, sd * ys
            if kind == "ucb":
                return -(mu + kappa * sd)
            a = mu - y_max - 0.01
            z = a / sd
            return -(a * norm.cdf(z) + sd * norm.pdf(z))

        vals = neg_acq(cand)
        best = float(vals.min())
        for s in cand[np.argsort(vals)[:3]]:
            r = minimize(lambda x: float(neg_acq(x)[0]), s, bounds=space.bounds, method="L-BFGS-B")
            best = min(best, float(r.fun))
        got = float(neg_acq(picks[j])[0])
        assert got <= best + 1e-4 * (abs(best) + 1e-3), (j, got, best)


def test_live_optimizer_async_pattern_and_state_round_trip(bo, ref, tmp_path):
    def make():
        opt = ref.BayesianOptimization(f=None, pbounds=PB, random_state=4, verbose=0,
                                       acquisition_function=bo.KrigingBeliever(bo.ExpectedImprovement(xi=0.01)))
        bo.enable(opt)
        opt._gp.set_params(optimizer=None)
        return opt

    opt = make()
    rs = np.random.RandomState(0)
    for _ in range(20):
        x = rs.uniform(size=4)
        opt.register(params=x, target=float(np.sin(5 * x.sum())))
    xs = [_quiet(opt.suggest) for _ in range(3)]  # three workers, nothing registered in between
    arr = [opt._space.params_to_array(x) for x in xs]
    assert len({a.tobytes() for a in arr}) == 3 and len(opt._acquisition_function.dummies) == 3
    opt.register(params=xs[0], target=0.3)  # worker 0 reports: its dummy expires at the next suggest
    _quiet(opt.suggest)
    dummies = opt._acquisition_function.dummies
    assert len(dummies) == 3 and not any(np.allclose(d, arr[0]) for d in dummies)
    path = tmp_path / "state.json"
    opt.save_state(path)
    other = make()
    other.load_state(path)
    assert [d.tolist() for d in other._acquisition_function.dummies] == [d.tolist() for d in dummies]
    X = bo.suggest_batch(other, 5)
    assert len(X) == 5 and len(other._acquisition_function.dummies) == 8


def test_non_pd_conditioning_raises_linalg_error(bo):
    """One training point, no jitter, unit variance: conditioning on that point again gives the pivot 1 - 1 = 0."""
    from sklearn.gaussian_process.kernels import RBF

    gp = bo.B200GaussianProcessRegressor(kernel=RBF(1.0), alpha=0.0, optimizer=None).fit(np.array([[0.25, 0.5]]), [1.0])
    with pytest.raises(np.linalg.LinAlgError):
        gp.condition_on_pending(np.array([[0.25, 0.5]]))
    mu0 = gp.predict(np.array([[0.9, 0.1]]))  # the source is untouched and still usable
    ok = gp.condition_on_pending(np.array([[0.9, 0.1]]))
    mu, sd = ok.predict(np.array([[0.9, 0.1], [0.3, 0.3]]), return_std=True)
    assert abs(mu[0] - mu0[0]) < 1e-12 and sd[0] < 1e-6 and ok.X_train_.shape[0] == 2

"""Noisy expected improvement on the device (DESIGN.md 4.13) against the numpy restatement tests/nei_oracle.py: the
fantasies of b200bo_gp_set_fantasies, the NEI / LogNEI values of the 16-warp kernel on every phase-B pipe and of the
small-batch kernels, selection order, the sigma_n^2 = tau reduction to EI, the refusals, and the reference's
BayesianOptimization driven through enable()."""
from __future__ import annotations

import warnings

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import ConstantKernel, Matern, WhiteKernel

import nei_oracle as NO

pytestmark = pytest.mark.gpu

C0, LS, NOISE = 1.7, 0.35, 0.04


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _fit(bo, n, d, noise=NOISE, alpha=1e-10, seed=0):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    y = np.sin(3.0 * X.sum(1)) + np.sqrt(noise) * rs.randn(n)
    k = ConstantKernel(C0) * Matern(length_scale=LS, nu=2.5)
    if noise > 0:
        k = k + WhiteKernel(noise)
    gp = bo.B200GaussianProcessRegressor(kernel=k, alpha=alpha, normalize_y=True, optimizer=None)
    gp.fit(X, y)
    return gp, X, y


def _oracle(gp, X, S, seed, jitter=1e-6, mask=None, noise=NOISE):
    kc = ConstantKernel(C0) * Matern(length_scale=LS, nu=2.5)
    Kc = kc(X)
    s2 = gp.alpha + noise
    tau = min(gp.alpha, jitter)
    ym, ys = float(gp._y_train_mean), float(gp._y_train_std)
    y_n = (gp._y_raw - ym) / ys
    Z, E = NO.draws(np.random.RandomState(seed), len(y_n), S)
    mask = np.ones(len(y_n), bool) if mask is None else mask
    F, A, best = NO.fantasies(Kc, y_n, s2, tau, Z, E, mask, ym, ys)
    return kc, Kc, tau, ym, ys, F, A, best


@pytest.mark.parametrize("n,d", [(300, 3), (300, 20)])
def test_fantasies_match_the_restatement(bo, n, d):
    gp, X, y = _fit(bo, n, d)
    fant = gp.noiseless_fantasies(4, random_state=11)
    _, _, _, ym, ys, F, A, best = _oracle(gp, X, 4, 11)
    tol = 1e-8 * (np.abs(ys * F + ym) + ys)
    assert np.all(np.abs(fant.F - (ys * F + ym)) <= tol)
    assert np.all(np.abs(fant.best - best) <= 1e-8 * (np.abs(best) + ys))
    assert fant.gp is not gp


@pytest.mark.parametrize("kind", ["nei", "lognei"])
@pytest.mark.parametrize("pipe", ["bulk", "bulk_nomc"])
@pytest.mark.parametrize("S", [1, 4, 16])
@pytest.mark.parametrize("d", [3, 20])  # candidate coordinates in registers (d <= 16) and in shared memory
def test_values_match_the_restatement(bo, monkeypatch, kind, pipe, S, d):
    import ctypes as C

    import torch

    monkeypatch.setenv("B200BO_PREDICT_PIPE", pipe)
    gp, X, y = _fit(bo, 300, d)
    fant = gp.noiseless_fantasies(S, random_state=3)
    kc, Kc, tau, ym, ys, F, A, best = _oracle(gp, X, S, 3)
    rs = np.random.RandomState(5)
    xi = 0.01
    code = bo._lib.ACQ_NEI if kind == "nei" else bo._lib.ACQ_LOGNEI
    acq = bo.FusedAcquisition(code, gp, xi=xi, fantasies=fant)
    for m in (1000, 20):  # tiled kernel, small-batch kernels
        Xc = rs.uniform(size=(m, d))
        Ks = kc(Xc, X)
        sd = NO.noiseless_sd(Kc, tau, Ks, C0, ys)
        want = -NO.nei(Ks, A, best, sd, xi, ym, ys, log=(kind == "lognei"))
        got = acq(Xc)
        np.testing.assert_allclose(got, want, rtol=1e-7, atol=1e-10)
        # selection in the restatement's order (ties to the lower index; the values here are distinct well beyond
        # the tolerance above)
        idx, val, top = acq.argmin_topk(Xc, 5)
        order = np.lexsort((np.arange(m), want))
        assert idx == order[0] and np.array_equal(top, order[:5])
    # device-resident candidates (b200bo_acq_eval_dev) give the host path's values bit for bit
    Xd = torch.from_numpy(Xc).cuda()
    out = torch.empty(Xc.shape[0], dtype=torch.float64, device="cuda")
    spec = acq.spec
    bo._lib.check(bo._lib.lib().b200bo_acq_eval_dev(C.byref(spec), Xd.data_ptr(), Xc.shape[0], out.data_ptr(), None,
                                                    None, 0, None, 0, None))
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), acq(Xc))


@pytest.mark.parametrize("kind", ["nei", "lognei"])
def test_philox_candidates_match_the_restatement(bo, kind):
    gp, X, y = _fit(bo, 300, 3)
    fant = gp.noiseless_fantasies(4, random_state=2)
    kc, Kc, tau, ym, ys, F, A, best = _oracle(gp, X, 4, 2)
    code = bo._lib.ACQ_NEI if kind == "nei" else bo._lib.ACQ_LOGNEI
    acq = bo.FusedAcquisition(code, gp, xi=0.01, fantasies=fant)
    i, v, xb, ti, tx = acq.argmin_topk_philox(77, np.array([[0.0, 1.0]] * 3), 4000, 4)
    Ks = kc(tx, X)
    want = -NO.nei(Ks, A, best, NO.noiseless_sd(Kc, tau, Ks, C0, ys), 0.01, ym, ys, log=(kind == "lognei"))
    np.testing.assert_allclose(v, want[0], rtol=1e-7, atol=1e-10)
    assert np.all(np.diff(want) >= -1e-9 * (np.abs(want[:-1]) + 1e-12))
    assert np.array_equal(xb, tx[0])


def _cd5(f, rows, h):
    """Fourth-order central differences: near a training point sigma0 is small and LogNEI's curvature large, where the
    two-point rule's h^2 term shows."""
    cols = []
    for e in np.eye(rows.shape[1]):
        cols.append((8 * (f(rows + h * e) - f(rows - h * e)) - (f(rows + 2 * h * e) - f(rows - 2 * h * e))) / (12 * h))
    return np.stack(cols, axis=1)


@pytest.mark.parametrize("kind", ["nei", "lognei"])
@pytest.mark.parametrize("S", [1, 4, 16])
def test_gradient_matches_central_differences_of_the_restatement(bo, kind, S):
    gp, X, y = _fit(bo, 300, 3)
    fant = gp.noiseless_fantasies(S, random_state=4)
    kc, Kc, tau, ym, ys, F, A, best = _oracle(gp, X, S, 4)
    code = bo._lib.ACQ_NEI if kind == "nei" else bo._lib.ACQ_LOGNEI
    acq = bo.FusedAcquisition(code, gp, xi=0.01, fantasies=fant)

    def f(rows):
        Ks = kc(rows, X)
        return -NO.nei(Ks, A, best, NO.noiseless_sd(Kc, tau, Ks, C0, ys), 0.01, ym, ys, log=(kind == "lognei"))

    rows = np.random.RandomState(6).uniform(0.05, 0.95, size=(12, 3))
    val, grad = acq.value_and_grad(rows)
    np.testing.assert_allclose(val, f(rows), rtol=1e-7, atol=1e-10)
    h = 1e-6
    cd = _cd5(f, rows, h)
    np.testing.assert_allclose(grad, cd, rtol=2e-5, atol=1e-6 * (1.0 + np.abs(cd).max()))


def test_gradient_with_constraints_matches_central_differences(bo):
    gp, X, y = _fit(bo, 300, 3)
    c1, _, _ = _fit(bo, 300, 3, seed=1)
    fant = gp.noiseless_fantasies(4, random_state=5)

    class Con:
        model = [c1]
        lb = np.array([-0.5])
        ub = np.array([0.8])

    rows = np.random.RandomState(7).uniform(0.05, 0.95, size=(10, 3))
    h = 1e-6
    for code in (bo._lib.ACQ_NEI, bo._lib.ACQ_LOGNEI):
        acq = bo.FusedAcquisition(code, gp, Con, xi=0.0, fantasies=fant)
        val, grad = acq.value_and_grad(rows)
        with acq.refine_mode():  # one kernel choice for every batch: the values difference cleanly
            np.testing.assert_array_equal(val, acq(rows))
            cd = _cd5(acq, rows, h)
        np.testing.assert_allclose(grad, cd, rtol=2e-5, atol=1e-6 * (1.0 + np.abs(cd).max()))


def test_constraints_and_philox(bo):
    gp, X, y = _fit(bo, 300, 3)
    c1, _, _ = _fit(bo, 300, 3, seed=1)
    c2, _, _ = _fit(bo, 300, 3, seed=2)
    fant = gp.noiseless_fantasies(4, random_state=9)

    class Con:
        model = [c1, c2]
        lb = np.array([-0.5, -np.inf])
        ub = np.array([0.8, 0.3])

    for code in (bo._lib.ACQ_NEI, bo._lib.ACQ_LOGNEI):
        acq = bo.FusedAcquisition(code, gp, Con, xi=0.0, fantasies=fant)
        plain = bo.FusedAcquisition(code, gp, xi=0.0, fantasies=fant)
        Xc = np.random.RandomState(4).uniform(size=(700, 3))
        got, base = acq(Xc), plain(Xc)
        probs = []
        for j, c in enumerate(Con.model):
            mu, sd = c.predict(Xc, return_std=True)
            from scipy.stats import norm

            probs.append(norm(mu, sd).cdf(Con.ub[j]) - norm(mu, sd).cdf(Con.lb[j]))
        if code == bo._lib.ACQ_NEI:
            np.testing.assert_allclose(got, base * probs[0] * probs[1], rtol=1e-7, atol=1e-12)
        else:
            np.testing.assert_allclose(got, base - np.log(probs[0]) - np.log(probs[1]), rtol=1e-7, atol=1e-9)
        # the small-batch kernels with the two constraint GPs
        np.testing.assert_allclose(acq(Xc[:25]), got[:25], rtol=1e-12, atol=1e-14)


def test_noise_equal_tau_is_ei(bo):
    gp, X, y = _fit(bo, 300, 3, noise=0.0, alpha=1e-6)
    fant = gp.noiseless_fantasies(4, jitter=1e-6, random_state=0)
    assert fant.gp is gp
    ym, ys = float(gp._y_train_mean), float(gp._y_train_std)
    assert np.array_equal(fant.F, np.repeat((ys * ((gp._y_raw - ym) / ys) + ym)[:, None], 4, axis=1)) or \
        np.allclose(fant.F, gp._y_raw[:, None], rtol=0, atol=1e-12 * ys)
    y_max = float(np.max(fant.best))
    nei = bo.FusedAcquisition(bo._lib.ACQ_NEI, gp, xi=0.01, fantasies=fant)
    ei = bo.FusedAcquisition(bo._lib.ACQ_EI, gp, xi=0.01, y_max=y_max)
    Xc = np.random.RandomState(8).uniform(size=(2000, 3))
    a, b = nei(Xc), ei(Xc)
    np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-13)
    ia, _, ta = nei.argmin_topk(Xc, 10)
    ib, _, tb = ei.argmin_topk(Xc, 10)
    assert ia == ib and np.array_equal(ta, tb)


def test_refusals(bo, monkeypatch):
    gp, X, y = _fit(bo, 300, 3)
    fant = gp.noiseless_fantasies(2, random_state=0)
    acq = bo.FusedAcquisition(bo._lib.ACQ_NEI, gp, fantasies=fant)
    Xc = np.random.RandomState(1).uniform(size=(5000, 3))  # the tiled kernel
    for env, val in (("B200BO_PREDICT_WARPS", "8"), ("B200BO_PREDICT_IMPL", "dfma"), ("B200BO_PREDICT_IMPL", "tf32"),
                     ("B200BO_PREDICT_PIPE", "cpasync"), ("B200BO_PREDICT_MMA", "884")):
        with monkeypatch.context() as mp:
            mp.setenv(env, val)
            with pytest.raises(NotImplementedError):
                acq(Xc)
    assert np.all(np.isfinite(acq(Xc)))
    # a later fit drops the fantasies of the noiseless handle
    fant.gp._device_fit(__import__("bayesianoptimization_b200.gpr", fromlist=["x"]).parse_kernel(gp.kernel_))
    with pytest.raises(bo._lib.B200Error):
        acq(Xc)
    with pytest.raises(ValueError):
        gp.noiseless_fantasies(2, incumbent=np.zeros(300, bool))


def _noisy_opt(bo, ref, acq, constraint=None, seed=1):
    rs = np.random.RandomState(seed)

    def f(x, y):
        return -(x - 0.3) ** 2 - (y + 0.2) ** 2 + 0.05 * rs.randn()

    kw = {}
    if constraint is not None:
        kw["constraint"] = constraint
    opt = ref.BayesianOptimization(f=f, pbounds={"x": (-1, 1), "y": (-1, 1)}, acquisition_function=acq,
                                   random_state=seed, verbose=0, **kw)
    opt.set_gp_params(alpha=2e-3)  # noise through alpha: the noiseless GP is a second handle (tau = 1e-6)
    bo.enable(opt)
    return opt


@pytest.mark.parametrize("cls", ["NoisyExpectedImprovement", "LogNoisyExpectedImprovement"])
def test_bayesian_optimization_through_enable(bo, ref, cls, tmp_path):
    acq = getattr(bo, cls)(xi=0.0, n_samples=4)
    opt = _noisy_opt(bo, ref, acq)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt.maximize(init_points=5, n_iter=3)
    assert len(opt.space) == 8 and acq.fantasies is not None and acq.fantasies.n_samples == 4
    path = tmp_path / "state.json"
    opt.save_state(str(path))
    acq2 = getattr(bo, cls)(xi=0.5, n_samples=2, jitter=1e-3)
    opt2 = _noisy_opt(bo, ref, acq2)
    opt2.load_state(str(path))
    assert (acq2.n_samples, acq2.jitter, acq2.xi) == (4, 1e-6, 0.0)


def test_int_and_categorical_space(bo, ref):
    acq = bo.NoisyExpectedImprovement(xi=0.0, n_samples=3)

    def f(x, k, c):
        return -(x - 0.2) ** 2 - 0.1 * (k - 2) ** 2 + (0.3 if c == "b" else 0.0)

    opt = ref.BayesianOptimization(f=f, pbounds={"x": (-1.0, 1.0), "k": (0, 5, int), "c": ("a", "b", "c")},
                                   acquisition_function=acq, random_state=3, verbose=0)
    opt.set_gp_params(alpha=1e-3)
    bo.enable(opt)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt.maximize(init_points=4, n_iter=2)
    assert len(opt.space) == 6


def test_constrained_and_infeasible(bo, ref):
    from bayes_opt.exception import NoValidPointRegisteredError
    from scipy.optimize import NonlinearConstraint

    con = NonlinearConstraint(lambda x, y: x + y, -np.inf, 0.5)
    opt = _noisy_opt(bo, ref, bo.LogNoisyExpectedImprovement(xi=0.0, n_samples=4), constraint=con)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt.maximize(init_points=5, n_iter=2)
    assert len(opt.space) == 7
    never = NonlinearConstraint(lambda x, y: x + y, 5.0, 6.0)
    opt = _noisy_opt(bo, ref, bo.NoisyExpectedImprovement(xi=0.0, n_samples=2), constraint=never)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(NoValidPointRegisteredError):
            opt.maximize(init_points=3, n_iter=1)


@pytest.mark.parametrize("name", ["c_m25_d3", "l_m25_d4"])
def test_illcond_gives_finite_values_or_names_jitter(bo, name):
    """An ill-conditioned fixture set of tests/golden (oracle/make_illcond.py), with observation noise 1e-4 added as a
    WhiteKernel term: the noiseless GP's K0 has tau = min(alpha, jitter) on its diagonal and either factors, giving
    finite NEI values, or raises the LinAlgError that names jitter."""
    from oracle import make_illcond as MI

    c = MI.CASES[name]
    with np.load(MI.fixture_path(name)) as z:
        X, y, xt = z["X"], z["y"], z["xt"]
    gp = bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(c) + WhiteKernel(1e-4), alpha=c["alpha"],
                                         normalize_y=True, optimizer=None)
    gp.fit(X, y)
    for jitter in (c["alpha"], 1e-6):
        try:
            fant = gp.noiseless_fantasies(4, jitter=jitter, random_state=0)
        except np.linalg.LinAlgError as e:
            assert "jitter" in str(e)
            continue
        assert np.all(np.isfinite(fant.F)) and np.all(np.isfinite(fant.best))
        for code in (bo._lib.ACQ_NEI, bo._lib.ACQ_LOGNEI):
            v = bo.FusedAcquisition(code, gp, fantasies=fant)(xt)
            assert np.all(np.isfinite(v))


@pytest.mark.parametrize("name", ["p1", "p2", "p4", "p6", "p8", "p10", "p13"])
def test_fantasies_on_the_kernel_matrix_cases(bo, name):
    """The fantasies of every covariance family of tests/kernel_matrix_cases.py (iso / ARD, ConstantKernel, int columns,
    d on both sides of 16) with a WhiteKernel noise term, against the restatement."""
    import kernel_matrix_cases as KM

    case = dict(KM.PREDICT[name])
    case["white"] = case.get("white") or 1e-2
    n, d = min(case["n"], 400), case["d"]
    rs = np.random.RandomState(11)
    X = rs.uniform(size=(n, d)) * (3.0 if case.get("rnd") else 1.0)
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    gp = bo.B200GaussianProcessRegressor(kernel=KM.kernel(case, d), alpha=1e-6, normalize_y=True, optimizer=None)
    gp.fit(X, y)
    fant = gp.noiseless_fantasies(4, random_state=1)
    noiseless = dict(case, white=None)
    Xt = KM.round_transform(d, case["rnd"])(X) if case.get("rnd") else X
    Kc = KM.base_kernel(noiseless, d)(Xt)
    ym, ys = float(gp._y_train_mean), float(gp._y_train_std)
    Z, E = NO.draws(np.random.RandomState(1), n, 4)
    F, A, best = NO.fantasies(Kc, (y - ym) / ys, 1e-6 + case["white"], 1e-6, Z, E, np.ones(n, bool), ym, ys)
    assert np.all(np.abs(fant.F - (ys * F + ym)) <= 1e-8 * (np.abs(ys * F + ym) + ys))
    assert np.all(np.abs(fant.best - best) <= 1e-8 * (np.abs(best) + ys))


def test_noiseless_handle_is_reused(bo):
    gp, X, y = _fit(bo, 300, 3)
    a = gp.noiseless_fantasies(2, random_state=0)
    b = gp.noiseless_fantasies(2, random_state=0)
    assert a.handle is b.handle  # one noiseless handle per GP, refitted in place
    np.testing.assert_array_equal(a.F, b.F)

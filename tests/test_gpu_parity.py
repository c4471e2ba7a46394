"""Parity of the CUDA path (through the C ABI) against the oracle and the committed golden
fixtures.  fp64 bar: 1e-5 relative (north_star); in practice the kernels sit near 1e-10."""
import ctypes as C
import pickle
import warnings

import numpy as np
import pytest
from numpy.testing import assert_allclose
from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern

pytestmark = pytest.mark.gpu

RTOL = 1e-5  # the north_star bar for fp64


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(scope="module")
def TS(ref):
    """The reference's TargetSpace (the hooks consume its RNG stream and bounds)."""
    return ref.target_space.TargetSpace


@pytest.fixture(scope="module")
def O():
    from oracle import gp_oracle

    return gp_oracle


@pytest.fixture(params=["dmma", "dmma8", "dfma"])
def impl(request, monkeypatch):
    """The variants of the fused fp64 kernel (read per launch): DMMA with 16 warps (default), DMMA with 8 warps,
    DFMA register tiles."""
    monkeypatch.setenv("B200BO_PREDICT_IMPL", "dfma" if request.param == "dfma" else "dmma")
    monkeypatch.setenv("B200BO_PREDICT_WARPS", "8" if request.param == "dmma8" else "16")
    return request.param


def make_gp(bo, kernel, **kw):
    kw.setdefault("alpha", 1e-6)
    kw.setdefault("normalize_y", True)
    kw.setdefault("optimizer", None)
    return bo.B200GaussianProcessRegressor(kernel=kernel, **kw)


def rel_err(a, b, floor=1e-300):
    return np.max(np.abs(a - b) / np.maximum(np.abs(b), floor))


# ------------------------------------------------------------------------------------------
# fit: K, L, alpha_, L^-1
# ------------------------------------------------------------------------------------------
def test_fit_state_vs_golden(bo, golden):
    g = golden("c2s_ei")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=float(g["length_scale"]))).fit(g["X"], g["y"])
    n = g["X"].shape[0]
    from bayesianoptimization_b200 import _lib as B

    K = np.empty((n, n))
    B.check(B.lib().b200bo_gp_get(gp._handle().ptr, B.GET_K, B.as_dp(K), n * n))
    Kref = g["K"].copy()
    Kref[np.diag_indices(n)] += 1e-6
    assert_allclose(K, Kref, rtol=1e-12, atol=1e-15)
    assert_allclose(gp.L_, g["L"], rtol=1e-8, atol=1e-12)
    assert np.all(np.triu(gp.L_, 1) == 0)
    assert_allclose(gp.alpha_, g["alpha_"], rtol=1e-6)
    W = np.empty((n, n))
    B.check(B.lib().b200bo_gp_get(gp._handle().ptr, B.GET_LINV, B.as_dp(W), n * n))
    assert_allclose(W @ g["L"], np.eye(n), atol=1e-9)
    assert float(gp._y_train_mean) == pytest.approx(float(g["y_mean"]), rel=1e-14)
    assert float(gp._y_train_std) == pytest.approx(float(g["y_std"]), rel=1e-14)


@pytest.mark.parametrize("n,d,aniso", [(300, 3, False), (900, 4, True)])
def test_concurrent_restarts_equal_sequential(bo, monkeypatch, n, d, aniso):
    """The 1 + n_restarts L-BFGS-B runs of fit() (SK/gaussian_process/_gpr.py:321-340) run concurrently
    (one thread + CUDA stream + factor buffers each).  Every LML evaluation is deterministic and
    independent of what else is in flight, so theta and the LML must be BIT-identical to the sequential
    loop (B200BO_PARALLEL_RESTARTS=0), and the RandomState must end in the same state."""
    X, y = _synth(n, d)
    ls = np.full(d, 0.7) if aniso else 0.7
    out = {}
    for mode in ("concurrent", "sequential", "concurrent")[:2 if aniso else 3]:
        monkeypatch.setenv("B200BO_PARALLEL_RESTARTS", "0" if mode == "sequential" else "1")
        rs = np.random.RandomState(5)
        gp = bo.B200GaussianProcessRegressor(kernel=ConstantKernel(1.0) * Matern(nu=2.5, length_scale=ls), alpha=1e-6,
                                             normalize_y=True, n_restarts_optimizer=4, random_state=rs)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            gp.fit(X, y)
        res = (gp.kernel_.theta.copy(), gp.log_marginal_likelihood_value_, rs.uniform(), gp.predict(X[:5]))
        if mode in out:
            ref = out[mode]
            assert np.array_equal(ref[0], res[0]) and ref[1] == res[1]
        out[mode] = res
    a, b = out["concurrent"], out["sequential"]
    assert np.array_equal(a[0], b[0])
    assert a[1] == b[1] and a[2] == b[2]
    assert np.array_equal(a[3], b[3])


def test_blocked_diagonal_kernel_equals_unblocked(bo, monkeypatch):
    """The 8-column-panel diagonal-block kernel (csrc/potrf_block.cuh; rsqrt pivots, inverse by
    recursive doubling) against the first, unblocked kernel (B200BO_POTRF=legacy; sqrt + divisions,
    inverse by substitution): factor, inverse and alpha_ agree to round-off."""
    from bayesianoptimization_b200 import _lib as B

    X, y = _synth(700, 5)
    n = X.shape[0]
    out = {}
    for mode in ("blocked", "legacy"):
        if mode == "legacy":
            monkeypatch.setenv("B200BO_POTRF", "legacy")
        else:
            monkeypatch.delenv("B200BO_POTRF", raising=False)
        gp = make_gp(bo, Matern(nu=2.5, length_scale=0.8)).fit(X, y)
        W = np.empty((n, n))
        B.check(B.lib().b200bo_gp_get(gp._handle().ptr, B.GET_LINV, B.as_dp(W), n * n))
        out[mode] = (gp.L_.copy(), W, gp.alpha_.copy())
    assert_allclose(out["blocked"][0][:64, :64], out["legacy"][0][:64, :64], rtol=1e-11, atol=1e-14)
    assert_allclose(out["blocked"][0], out["legacy"][0], rtol=1e-8, atol=1e-12)
    L = out["blocked"][0]
    for mode in out:
        assert np.max(np.abs(out[mode][1] @ L - np.eye(n))) < 1e-7, mode
    assert_allclose(out["blocked"][2], out["legacy"][2], rtol=1e-7)


@pytest.mark.parametrize("n", [1, 63, 64, 65, 127, 129, 200, 257, 700])
def test_factor_padding_and_ragged_sizes(bo, O, n):
    rs = np.random.RandomState(n)
    d = 3
    X = rs.uniform(size=(n, d))
    y = np.sin(3 * X.sum(1)) + 0.05 * rs.randn(n)
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.5)).fit(X, y)
    st = O.fit_fixed(X, y, length_scale=0.5)
    assert_allclose(gp.L_, st.L, rtol=1e-7, atol=1e-11)
    xt = rs.uniform(size=(300, d))
    mu, sd = gp.predict(xt, return_std=True)
    mu0, sd0 = O.predict(st, xt)
    assert_allclose(mu, mu0, rtol=RTOL, atol=1e-9)
    assert_allclose(sd, sd0, rtol=RTOL, atol=1e-8)


# ------------------------------------------------------------------------------------------
# predict + acquisition vs golden (reference outputs)
# ------------------------------------------------------------------------------------------
def test_c2s_predict_and_acq_vs_golden(bo, golden, impl):
    g = golden("c2s_ei")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=float(g["length_scale"]))).fit(g["X"], g["y"])
    mu, sd = gp.predict(g["xt"], return_std=True)
    assert_allclose(mu, g["mu"], rtol=RTOL, atol=1e-10)
    assert_allclose(sd, g["sd"], rtol=RTOL, atol=1e-10)
    assert_allclose(gp.predict(g["xt"]), g["mu"], rtol=RTOL, atol=1e-10)
    for cls, key, kw in [
        (bo.ExpectedImprovement, "acq_ei", dict(xi=float(g["xi"]))),
        (bo.ProbabilityOfImprovement, "acq_poi", dict(xi=float(g["xi"]))),
        (bo.UpperConfidenceBound, "acq_ucb", dict(kappa=float(g["kappa"]))),
    ]:
        a = cls(**kw)
        if hasattr(a, "y_max"):
            a.y_max = float(g["y_max"])
        f = a._get_acq(gp=gp)
        ys = f(g["xt"])
        assert_allclose(ys, g[key], rtol=RTOL, atol=1e-14)
        if key == "acq_ei":
            idx, val, top = f.argmin_topk(g["xt"], 10)
            assert idx == int(g["argmin"])
            assert val == ys[idx]
            assert list(top) == list(g["top10"])
            # single-row calls (what L-BFGS-B does; small-batch path) agree with the batch to
            # round-off (different, but fixed, summation order)
            for i in (0, 17, 4095):
                assert f(g["xt"][i])[0] == pytest.approx(ys[i], rel=1e-11, abs=1e-15)


def test_c1_readme_ucb_vs_golden(bo, golden):
    g = golden("c1_readme_ucb")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=float(g["length_scale"]))).fit(g["X"], g["y"])
    assert_allclose(gp.L_, g["L"], rtol=1e-8, atol=1e-12)
    mu, sd = gp.predict(g["xt"], return_std=True)
    assert_allclose(mu, g["mu"], rtol=RTOL, atol=1e-9)
    assert_allclose(sd, g["sd"], rtol=RTOL, atol=1e-8)
    f = bo.UpperConfidenceBound(kappa=float(g["kappa"]))._get_acq(gp=gp)
    ys = f(g["xt"])
    assert_allclose(ys, g["acq"], rtol=RTOL, atol=1e-8)
    assert int(np.argmin(ys)) == int(np.argmin(g["acq"]))
    assert_allclose([f(g["xt"][i])[0] for i in range(16)], g["acq_single"], rtol=RTOL, atol=1e-8)


def test_near_duplicate_candidates(bo, golden):
    g = golden("c2s_ei")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=float(g["length_scale"]))).fit(g["X"], g["y"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mu, sd = gp.predict(g["xe"], return_std=True)
    assert_allclose(mu, g["mu_e"], rtol=RTOL, atol=1e-8)
    # sigma at the jitter floor is a difference of O(1) numbers; LAPACK itself only has
    # absolute accuracy there
    assert_allclose(sd, g["sd_e"], rtol=1e-3, atol=2e-7)


KERNELS = {
    "m05": (lambda: Matern(nu=0.5, length_scale=0.6)),
    "m15": (lambda: Matern(nu=1.5, length_scale=0.6)),
    "rbf": (lambda: RBF(length_scale=0.6)),
    "m25aniso": (lambda: Matern(nu=2.5, length_scale=[0.3, 0.6, 1.2, 2.4])),
    "crbf": (lambda: ConstantKernel(2.0) * RBF(length_scale=0.8)),
    "cm25": (lambda: ConstantKernel(0.5) * Matern(nu=2.5, length_scale=0.5)),
}


@pytest.mark.parametrize("tag", sorted(KERNELS))
def test_kernel_families_vs_golden(bo, golden, tag):
    g = golden("kernels_small")
    gp = make_gp(bo, KERNELS[tag]()).fit(g["X"], g["y"])
    assert_allclose(gp.L_, g[f"{tag}_L"], rtol=1e-8, atol=1e-12)
    mu, sd = gp.predict(g["xt"], return_std=True)
    assert_allclose(mu, g[f"{tag}_mu"], rtol=RTOL, atol=1e-9)
    assert_allclose(sd, g[f"{tag}_sd"], rtol=RTOL, atol=1e-9)
    lml, grad = gp.log_marginal_likelihood(gp.kernel_.theta, eval_gradient=True)
    assert lml == pytest.approx(float(g[f"{tag}_lml"]), rel=1e-8)
    assert_allclose(grad, g[f"{tag}_lml_grad"], rtol=1e-5, atol=1e-6)
    # the factor buffers now hold another theta; predict must transparently re-factorise
    mu2 = gp.predict(g["xt"])
    assert_allclose(mu2, mu, rtol=0, atol=0)


def test_lml_and_gradient_vs_golden(bo, golden):
    g = golden("c2s_ei")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(g["X"], g["y"])
    for t, v, gr in zip(g["thetas"], g["lml"], g["lml_grad"]):
        lml, grad = gp.log_marginal_likelihood(np.array([t]), eval_gradient=True)
        assert lml == pytest.approx(float(v), rel=1e-8, abs=1e-8)
        assert grad[0] == pytest.approx(float(gr), rel=1e-5, abs=1e-5)
        assert gp.log_marginal_likelihood(np.array([t])) == pytest.approx(float(v), rel=1e-8, abs=1e-8)


def test_constrained_acquisition_vs_golden(bo, golden, impl):
    g = golden("c4s_constrained")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=float(g["ls"]))).fit(g["X"], g["y"])
    cm = bo.ConstraintModel(None, g["lb"], g["ub"])
    for m, l in zip(cm.model, g["ls_c"]):
        m.set_params(kernel=Matern(nu=2.5, length_scale=float(l)), optimizer=None)
    cm.fit(g["X"], g["c"])
    assert_allclose(cm.predict(g["xt"]), g["p"], rtol=RTOL, atol=1e-12)
    assert_allclose(cm.approx(g["xt"]), g["approx"], rtol=RTOL, atol=1e-9)
    for cls, key in [(bo.ProbabilityOfImprovement, "acq_poi"), (bo.ExpectedImprovement, "acq_ei")]:
        a = cls(xi=float(g["xi"]))
        a.y_max = float(g["y_max"])
        ys = a._get_acq(gp=gp, constraint=cm)(g["xt"])
        assert_allclose(ys, g[key], rtol=RTOL, atol=1e-13)
    cm1 = bo.ConstraintModel(None, -0.5, 0.5)
    cm1.model[0].set_params(kernel=Matern(nu=2.5, length_scale=0.5), optimizer=None)
    cm1.fit(g["X"], g["c"][:, 1])
    assert_allclose(cm1.predict(g["xt"]), g["p1"], rtol=RTOL, atol=1e-12)
    a = bo.ExpectedImprovement(xi=float(g["xi"]))
    a.y_max = float(g["y_max"])
    ys1 = a._get_acq(gp=gp, constraint=cm1)(g["xt"])
    # J=1 fused == (-EI) * p1
    ei = a._get_acq(gp=gp)(g["xt"])
    assert_allclose(ys1, ei * g["p1"], rtol=RTOL, atol=1e-13)


# ------------------------------------------------------------------------------------------
# hyper-parameter fit (device LML driven by host L-BFGS-B): two-tier parity (SURVEY section 7)
# ------------------------------------------------------------------------------------------
def test_full_fit_vs_golden(bo, golden):
    g = golden("fit_full_small")
    rs = np.random.RandomState(3)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), alpha=1e-6, normalize_y=True,
                                         n_restarts_optimizer=5, random_state=rs)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gp.fit(g["X"], g["y"])
    # the shared RandomState advanced exactly as sklearn's fit advances it
    assert_allclose(rs.uniform(size=3), g["next_uniform"], rtol=0, atol=0)
    assert gp.log_marginal_likelihood_value_ == pytest.approx(float(g["lml"]), rel=1e-7)
    assert_allclose(gp.kernel_.theta, g["theta"], rtol=1e-4, atol=1e-4)
    mu, sd = gp.predict(g["xt"], return_std=True)
    assert_allclose(mu, g["mu"], rtol=1e-3, atol=1e-4)  # theta* only matches to optimiser tolerance
    assert_allclose(sd, g["sd"], rtol=1e-3, atol=1e-4)


# ------------------------------------------------------------------------------------------
# larger sizes vs the oracle
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,d,m", [(1000, 8, 5000), (1024, 8, 4096), (2048, 16, 3000), (300, 17, 1000), (500, 33, 700)])
def test_midsize_vs_oracle(bo, O, n, d, m, impl):
    rs = np.random.RandomState(5)
    X = rs.uniform(size=(n, d))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    xt = rs.uniform(size=(m, d))
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(X, y)
    st = O.fit_fixed(X, y, length_scale=0.7)
    assert_allclose(gp.L_, st.L, rtol=1e-6, atol=1e-10)
    a = bo.ExpectedImprovement(xi=0.01)
    a.y_max = float(y.max())
    f = a._get_acq(gp=gp)
    ys = f(xt)
    ref = O.acq_closure(st, O.ACQ_EI, xi=0.01, y_max=float(y.max()))(xt)
    assert_allclose(ys, ref, rtol=RTOL, atol=1e-14)
    idx, val, top = f.argmin_topk(xt, 10)
    i0, v0, t0 = O.argmin_topk(ref, 10)
    assert idx == i0 and list(top) == list(t0)
    mu, sd = gp.predict(xt, return_std=True)
    mu0, sd0 = O.predict(st, xt)
    assert_allclose(mu, mu0, rtol=RTOL, atol=1e-10)
    assert_allclose(sd, sd0, rtol=RTOL, atol=1e-10)


def test_c3_full_size_vs_oracle_and_properties(bo, O):
    """BASELINE config 3 sizes (N=4096, d=16): direct oracle comparison on 4096 candidates plus
    size-independent properties (linearity of mu in y, variance independent of y, interpolation
    at training points, batch == single-row)."""
    n, d, m = 4096, 16, 4096
    rs = np.random.RandomState(0)
    X = rs.uniform(size=(n, d))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    xt = rs.uniform(size=(m, d))
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(X, y)
    st = O.fit_fixed(X, y, length_scale=0.7)
    a = bo.ExpectedImprovement(xi=0.01)
    a.y_max = float(y.max())
    f = a._get_acq(gp=gp)
    ys = f(xt)
    ref = O.acq_closure(st, O.ACQ_EI, xi=0.01, y_max=float(y.max()))(xt)
    assert_allclose(ys, ref, rtol=RTOL, atol=1e-14)
    assert int(np.argmin(ys)) == int(np.argmin(ref))
    mu, sd = gp.predict(xt, return_std=True)
    mu0, sd0 = O.predict(st, xt)
    assert_allclose(mu, mu0, rtol=RTOL, atol=1e-10)
    assert_allclose(sd, sd0, rtol=RTOL, atol=1e-10)
    # interpolation: at training points |mu - y| is tiny compared with the data scale
    mu_tr, sd_tr = gp.predict(X[:512], return_std=True)
    assert np.max(np.abs(mu_tr - y[:512])) < 1e-2
    assert np.max(sd_tr) < 5e-2
    # linearity in y (normalize_y=False), variance independent of y
    y2 = np.cos(2 * X.sum(1))
    g1 = make_gp(bo, Matern(nu=2.5, length_scale=0.7), normalize_y=False).fit(X, y)
    m1, s1 = g1.predict(xt[:1024], return_std=True)
    g2 = make_gp(bo, Matern(nu=2.5, length_scale=0.7), normalize_y=False).fit(X, y2)
    m2, s2 = g2.predict(xt[:1024], return_std=True)
    g3 = make_gp(bo, Matern(nu=2.5, length_scale=0.7), normalize_y=False).fit(X, y + y2)
    m3, s3 = g3.predict(xt[:1024], return_std=True)
    assert_allclose(m1 + m2, m3, rtol=1e-8, atol=1e-9)
    assert np.array_equal(s1, s2) and np.array_equal(s1, s3)
    # batch vs single row (small-batch path): round-off only; run-to-run bit reproducibility
    assert f(xt[7])[0] == pytest.approx(ys[7], rel=1e-10)
    assert f(xt[7])[0] == f(xt[7])[0]
    assert np.array_equal(f(xt), ys)


def _synth(n, d, seed=0):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    return X, y


def test_c2_full_batch_2pow20(bo, O):
    """BASELINE configs[1]: d=8, N=1024, EI, one 2^20-candidate batch, fp64.  Full batch on the
    device; a strided 2^14 subsample against the oracle; selection against numpy on the full
    vector; tile-position independence (a chunk evaluated alone gives the same bits)."""
    n, d, m = 1024, 8, 1 << 20
    X, y = _synth(n, d)
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(X, y)
    st = O.fit_fixed(X, y, length_scale=0.7)
    a = bo.ExpectedImprovement(xi=0.01)
    a.y_max = float(y.max())
    f = a._get_acq(gp=gp)
    xt = np.random.RandomState(1).uniform(size=(m, d))
    ys = f(xt)
    sub = slice(0, m, 64)
    ref = O.acq_closure(st, O.ACQ_EI, xi=0.01, y_max=float(y.max()))(xt[sub])
    assert_allclose(ys[sub], ref, rtol=RTOL, atol=1e-14)
    idx, val, top = f.argmin_topk(xt, 10)
    assert idx == int(np.argmin(ys)) and val == ys[idx]
    assert list(top) == list(np.argsort(ys, kind="stable")[:10])
    for s0 in (0, 128 * 77, 128 * 77 + 5):
        assert np.array_equal(f(xt[s0:s0 + 20_000]), ys[s0:s0 + 20_000])


def test_c4_constrained_poi_full_size(bo, O):
    """BASELINE configs[3]: d=16, N=2048, PoI x p_constraint with a 2-GP ConstraintModel
    (lb=[-inf,-0.5], ub=[0.6,0.5]); 2^18 candidates on the device, 4096-point subsample vs oracle."""
    n, d, m = 2048, 16, 1 << 18
    X, y = _synth(n, d)
    c = np.column_stack([np.cos(X.sum(1)), np.sin(2 * X.sum(1))])
    lb, ub = np.array([-np.inf, -0.5]), np.array([0.6, 0.5])
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(X, y)
    cm = bo.ConstraintModel(None, lb, ub)
    for mdl, l in zip(cm.model, (0.9, 0.5)):
        mdl.set_params(kernel=Matern(nu=2.5, length_scale=l), optimizer=None)
    cm.fit(X, c)
    allowed = cm.allowed(c)
    y_max = float(y[allowed].max())
    a = bo.ProbabilityOfImprovement(xi=0.01)
    a.y_max = y_max
    f = a._get_acq(gp=gp, constraint=cm)
    xt = np.random.RandomState(1).uniform(size=(m, d))
    ys = f(xt)
    st = O.fit_fixed(X, y, length_scale=0.7)
    cs = [O.fit_fixed(X, c[:, j], length_scale=l) for j, l in enumerate((0.9, 0.5))]
    sub = slice(0, m, 64)
    ref = O.acq_closure(st, O.ACQ_POI, xi=0.01, y_max=y_max, constraint=(cs, lb, ub))(xt[sub])
    assert_allclose(ys[sub], ref, rtol=RTOL, atol=1e-14)
    idx, val, top = f.argmin_topk(xt, 10)
    assert idx == int(np.argmin(ys)) and list(top) == list(np.argsort(ys, kind="stable")[:10])


def test_c5_n8192_d32_ucb_shard(bo, O):
    """BASELINE configs[4]: d=32, N=8192, UCB kappa=2.576 - one GPU's shard (2^19 candidates) of
    the 8-GPU job; 2048-point subsample vs oracle; shard-local selection vs numpy."""
    n, d, m = 8192, 32, 1 << 19
    X, y = _synth(n, d)
    gp = make_gp(bo, Matern(nu=2.5, length_scale=1.0)).fit(X, y)
    f = bo.UpperConfidenceBound(kappa=2.576)._get_acq(gp=gp)
    xt = np.random.RandomState(1).uniform(size=(m, d))
    ys = f(xt)
    st = O.fit_fixed(X, y, length_scale=1.0)
    assert_allclose(gp.L_[-64:], st.L[-64:], rtol=1e-6, atol=1e-10)
    sub = slice(0, m, 256)
    ref = O.acq_closure(st, O.ACQ_UCB, kappa=2.576)(xt[sub])
    assert_allclose(ys[sub], ref, rtol=RTOL, atol=1e-12)
    idx, val, top = f.argmin_topk(xt, 10)
    assert idx == int(np.argmin(ys)) and list(top) == list(np.argsort(ys, kind="stable")[:10])


@pytest.mark.parametrize("n,d", [(40, 2), (700, 5), (2048, 16)])
def test_small_batch_path_vs_tiled_and_oracle(bo, O, n, d, monkeypatch):
    """The small-batch kernels (single rows / FD stencils) against the tiled kernel and the oracle,
    incl. a constrained closure and ragged candidate counts (1, 17, 33, 70)."""
    rs = np.random.RandomState(n)
    X = rs.uniform(size=(n, d))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    cvals = np.cos(X.sum(1))
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.6)).fit(X, y)
    cm = bo.ConstraintModel(None, -0.3, 0.8)
    cm.model[0].set_params(kernel=Matern(nu=2.5, length_scale=0.9), optimizer=None)
    cm.fit(X, cvals)
    st = O.fit_fixed(X, y, length_scale=0.6)
    sc = O.fit_fixed(X, cvals, length_scale=0.9)
    a = bo.ExpectedImprovement(xi=0.01)
    a.y_max = float(y.max())
    f, fc = a._get_acq(gp=gp), a._get_acq(gp=gp, constraint=cm)
    ref = O.acq_closure(st, O.ACQ_EI, xi=0.01, y_max=float(y.max()))
    refc = O.acq_closure(st, O.ACQ_EI, xi=0.01, y_max=float(y.max()), constraint=([sc], [-0.3], [0.8]))
    for m in (1, 17, 33, 70):
        xt = rs.uniform(size=(m, d))
        out = {}
        for path in ("1", "0"):
            monkeypatch.setenv("B200BO_SMALL_PATH", path)
            out[path] = (f(xt), fc(xt), gp.predict(xt, return_std=True))
        assert_allclose(out["1"][0], ref(xt), rtol=RTOL, atol=1e-14)
        assert_allclose(out["1"][1], refc(xt), rtol=RTOL, atol=1e-14)
        assert_allclose(out["1"][0], out["0"][0], rtol=1e-8, atol=1e-15)
        assert_allclose(out["1"][1], out["0"][1], rtol=1e-8, atol=1e-15)
        mu0, sd0 = O.predict(st, xt)
        assert_allclose(out["1"][2][0], mu0, rtol=RTOL, atol=1e-10)
        assert_allclose(out["1"][2][1], sd0, rtol=RTOL, atol=1e-10)
        idx, val, top = f.argmin_topk(xt, 5)
        assert idx == int(np.argmin(out["1"][0]))


def test_batched_fd_stencil_matches_sequential_lbfgsb(bo, golden, TS):
    """_smart_minimize with the batched stencil map follows the same iterates as plain SciPy
    L-BFGS-B with one objective call per stencil point (R/bayes_opt/acquisition.py:366)."""
    from scipy.optimize import minimize

    g = golden("c2s_ei")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=float(g["length_scale"]))).fit(g["X"], g["y"])
    a = bo.ExpectedImprovement(xi=float(g["xi"]))
    a.y_max = float(g["y_max"])
    f = a._get_acq(gp=gp)
    space = TS(None, {f"x{i:02d}": (0.0, 1.0) for i in range(8)})
    seeds = g["xt"][g["top10"][:3]]
    x_b, v_b = a._smart_minimize(f, space, seeds, np.random.RandomState(0))
    best = None
    for s in seeds:
        r = minimize(f, s, bounds=space.bounds, method="L-BFGS-B")
        if r.success and (best is None or r.fun < best.fun):
            best = r
    assert_allclose(x_b, np.clip(best.x, 0, 1), rtol=1e-6, atol=1e-8)
    assert float(v_b) == pytest.approx(float(np.squeeze(best.fun)), rel=1e-8)


# ------------------------------------------------------------------------------------------
# selection semantics, edge cases, errors
# ------------------------------------------------------------------------------------------
def test_selection_semantics_ties(bo):
    """argmin / top-k selection: ties -> lowest index (np.argmin / stable argsort order)."""
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.5)).fit(np.random.RandomState(0).rand(5, 2), np.arange(5.0))
    rs = np.random.RandomState(3)
    xt = rs.rand(777, 2)
    f = bo.UpperConfidenceBound(kappa=1.0)._get_acq(gp=gp)
    ys = f(xt)
    idx, val, top = f.argmin_topk(xt, 20)
    assert idx == int(np.argmin(ys)) and val == ys.min()
    assert list(top) == list(np.argsort(ys, kind="stable")[:20])
    # duplicated candidates -> exact ties -> lowest index first
    xt2 = np.vstack([xt[:100], xt[:100]])
    ys2 = f(xt2)
    idx2, _, top2 = f.argmin_topk(xt2, 8)
    assert idx2 == int(np.argmin(ys2))
    assert list(top2) == list(np.argsort(ys2, kind="stable")[:8])
    # fewer candidates than seeds requested
    idx3, _, top3 = f.argmin_topk(xt[:3], 10)
    assert idx3 == int(np.argmin(ys[:3])) and list(top3) == list(np.argsort(ys[:3], kind="stable"))


def test_selection_nan_semantics(bo):
    """NaN acquisition values: np.argmin returns the FIRST NaN; np.argsort puts NaNs last."""
    X = np.array([[0.1], [0.5], [0.9]])
    y = np.array([0.0, 1.0, 0.5])
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.3), alpha=1e-12, normalize_y=False).fit(X, y)
    a = bo.ExpectedImprovement(xi=0.0)
    a.y_max = 1.0
    f = a._get_acq(gp=gp)
    rs = np.random.RandomState(0)
    xt = np.vstack([rs.rand(50, 1), X, rs.rand(50, 1), X])
    ys = f(xt)
    idx, val, top = f.argmin_topk(xt, 12)
    assert idx == int(np.argmin(ys))
    assert list(top) == list(np.argsort(ys, kind="stable")[:12])


def test_sigma_zero_nan_semantics(bo):
    """EI with sigma == 0: a*Phi(+-inf) + 0*phi -> a or 0; a == 0 and sigma == 0 -> NaN, and NaN is
    np.argmin's minimum (SURVEY section 7 'EI/PoI edge semantics')."""
    X = np.array([[0.1], [0.5], [0.9]])
    y = np.array([0.0, 1.0, 0.5])
    # alpha=0 -> exact interpolation -> clamped variance 0 at training points
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.3), alpha=1e-12, normalize_y=False).fit(X, y)
    a = bo.ExpectedImprovement(xi=0.0)
    a.y_max = 1.0
    f = a._get_acq(gp=gp)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mu, sd = gp.predict(X, return_std=True)
    ys = f(X)
    for i in range(3):
        if sd[i] == 0.0:
            aa = mu[i] - 1.0
            expect = np.nan if aa == 0 else (-aa if aa > 0 else 0.0)
            assert (np.isnan(ys[i]) and np.isnan(expect)) or ys[i] == pytest.approx(expect, abs=1e-12)


def test_not_positive_definite_raises_linalgerror(bo):
    X = np.vstack([np.full((1, 2), 0.5)] * 3 + [np.array([[0.1, 0.2]])])
    y = np.array([1.0, 2.0, 3.0, 4.0])
    gp = make_gp(bo, Matern(nu=2.5, length_scale=1.0), alpha=0.0)
    with pytest.raises(np.linalg.LinAlgError):
        gp.fit(X, y)


def test_unsupported_kernel_raises(bo):
    from sklearn.gaussian_process.kernels import RationalQuadratic

    gp = make_gp(bo, RationalQuadratic())
    with pytest.raises(NotImplementedError):
        gp.fit(np.random.rand(5, 2), np.random.rand(5))
    gp = make_gp(bo, Matern(nu=1.0))
    with pytest.raises(NotImplementedError):
        gp.fit(np.random.rand(5, 2), np.random.rand(5))


def test_closure_survives_lml_evaluation(bo, golden):
    """log_marginal_likelihood(theta) re-uses the device factor buffers; a closure created before must
    transparently see the fitted model again."""
    g = golden("c2s_ei")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(g["X"], g["y"])
    f = bo.UpperConfidenceBound(kappa=float(g["kappa"]))._get_acq(gp=gp)
    y0 = f(g["xt"][:300])
    gp.log_marginal_likelihood(np.log([0.3]), eval_gradient=True)
    assert np.array_equal(f(g["xt"][:300]), y0)
    assert_allclose(y0, g["acq_ucb"][:300], rtol=RTOL, atol=1e-12)


def test_prior_predict_unfitted(bo):
    gp = make_gp(bo, Matern(nu=2.5))
    mu, sd = gp.predict(np.random.rand(7, 3), return_std=True)
    assert np.all(mu == 0) and np.all(sd == 1)


def test_pickle_roundtrip_refits_on_device(bo, golden):
    g = golden("c2s_ei")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(g["X"], g["y"])
    mu = gp.predict(g["xt"][:256])
    gp2 = pickle.loads(pickle.dumps(gp))
    assert np.array_equal(gp2.predict(g["xt"][:256]), mu)


def test_round_transform_for_int_parameters(bo, O):
    """wrap_kernel with np.round on one dimension (R/bayes_opt/parameter.py:308-320, :484-487)."""
    rs = np.random.RandomState(2)
    X = np.column_stack([rs.uniform(0, 1, 80), np.round(rs.uniform(0, 10, 80))])
    y = np.sin(X[:, 0] * 3) + 0.1 * X[:, 1]

    def transform(v):
        v = np.atleast_2d(v).astype(float).copy()
        v[:, 1] = np.round(v[:, 1])
        return v

    from bayes_opt.parameter import wrap_kernel

    gp = make_gp(bo, wrap_kernel(Matern(nu=2.5, length_scale=0.8), transform)).fit(X, y)
    xt = np.column_stack([rs.uniform(0, 1, 500), rs.uniform(0, 10, 500)])
    mu, sd = gp.predict(xt, return_std=True)
    st = O.fit_fixed(transform(X), y, length_scale=0.8)
    mu0, sd0 = O.predict(st, transform(xt))
    assert_allclose(mu, mu0, rtol=RTOL, atol=1e-10)
    assert_allclose(sd, sd0, rtol=RTOL, atol=1e-9)


def test_c_abi_direct_calls(bo, golden):
    """Raw ctypes calls against include/b200bo.h (no Python classes in between)."""
    from bayesianoptimization_b200 import _lib as B

    L = B.lib()
    g = golden("c2s_ei")
    h = C.c_void_p()
    assert L.b200bo_gp_create(C.byref(h), 0) == 0
    ls = np.array([float(g["length_scale"])])
    spec = B.KernelSpec(B.KERNEL_MATERN, B.NU_25, 1, 0, 1.0, B.as_dp(ls))
    X, y, xt = B.c_f64(g["X"]), B.c_f64(g["y"]), B.c_f64(g["xt"])
    info = C.c_int64()
    assert L.b200bo_gp_fit(h, B.as_dp(X), B.as_dp(y), X.shape[0], X.shape[1], C.byref(spec), 1e-6, 1,
                           C.byref(info)) == 0
    assert L.b200bo_gp_n(h) == X.shape[0] and L.b200bo_gp_dim(h) == X.shape[1]
    mu, sd = np.empty(len(xt)), np.empty(len(xt))
    ncl = C.c_int64()
    assert L.b200bo_gp_predict(h, B.as_dp(xt), len(xt), B.as_dp(mu), B.as_dp(sd), C.byref(ncl)) == 0
    assert_allclose(mu, g["mu"], rtol=RTOL, atol=1e-10)
    assert_allclose(sd, g["sd"], rtol=RTOL, atol=1e-10)
    acq = B.AcqSpec()
    acq.kind, acq.n_gps, acq.xi, acq.y_max = B.ACQ_EI, 1, float(g["xi"]), float(g["y_max"])
    acq.gps[0] = h.value
    out = np.empty(len(xt))
    bv, bi = C.c_double(), C.c_int64()
    tv, ti = np.empty(10), np.empty(10, dtype=np.int64)
    assert L.b200bo_acq_argmin_topk(C.byref(acq), B.as_dp(xt), len(xt), 10, C.byref(bv), C.byref(bi),
                                    B.as_dp(tv), ti.ctypes.data_as(C.POINTER(C.c_int64)), B.as_dp(out)) == 0
    assert_allclose(out, g["acq_ei"], rtol=RTOL, atol=1e-14)
    assert bi.value == int(g["argmin"]) and list(ti) == list(g["top10"])
    ms = C.c_float()
    assert L.b200bo_last_kernel_ms(C.byref(ms)) == 0 and ms.value > 0
    # argument errors come back as codes + message, never a crash
    assert L.b200bo_gp_predict(h, None, 5, B.as_dp(mu), None, None) == B.ERR_ARG
    assert b"candidates" in L.b200bo_last_error()
    L.b200bo_gp_destroy(h)


def test_device_resident_entry_point(bo, golden):
    """b200bo_acq_eval_dev with torch-owned device buffers on a non-default stream."""
    import torch

    from bayesianoptimization_b200 import _lib as B

    g = golden("c2s_ei")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(g["X"], g["y"])
    a = bo.ExpectedImprovement(xi=float(g["xi"]))
    a.y_max = float(g["y_max"])
    f = a._get_acq(gp=gp)
    xt = torch.from_numpy(g["xt"]).cuda()
    out = torch.empty(xt.shape[0], dtype=torch.float64, device="cuda")
    sel = torch.zeros((11, 2), dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        B.check(B.lib().b200bo_acq_eval_dev(C.byref(f.spec), xt.data_ptr(), xt.shape[0], out.data_ptr(),
                                            None, None, 10, sel.data_ptr(), 1000, s.cuda_stream))
    s.synchronize()
    assert_allclose(out.cpu().numpy(), g["acq_ei"], rtol=RTOL, atol=1e-14)
    idx = sel[:, 1].cpu().numpy()
    assert idx[0] == int(g["argmin"]) + 1000
    assert list(idx[1:] - 1000) == list(g["top10"])
    vals = sel[:, 0].cpu().numpy().view(np.float64)
    assert vals[0] == g["acq_ei"].min() or abs(vals[0] - g["acq_ei"].min()) < 1e-12


# ------------------------------------------------------------------------------------------
# end-to-end suggest()
# ------------------------------------------------------------------------------------------
def test_suggest_end_to_end_readme(bo, golden, TS):
    """Full suggest() (fit with 5 restarts + 10k candidates + 10 L-BFGS-B refinements) from the
    reference's RNG state: end-to-end tier - same point to optimiser tolerance."""
    g = golden("c1_readme_ucb")
    space = TS(None, {"x": (2, 4), "y": (-3, 3)})
    for x, t in zip(g["X"], g["y"]):
        space.register(x, t)
    rs = np.random.RandomState()
    rs.set_state(("MT19937", g["rs_keys"], int(g["rs_pos"]), 0, 0.0))
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), alpha=1e-6, normalize_y=True,
                                         n_restarts_optimizer=5, random_state=rs)
    acq = bo.UpperConfidenceBound(kappa=float(g["kappa"]))
    x1 = acq.suggest(gp, space, random_state=rs)
    assert_allclose(x1, g["suggestion"], rtol=1e-3, atol=1e-3)
    # determinism pin of the reference's save/load tests: same state -> identical suggestion
    rs.set_state(("MT19937", g["rs_keys"], int(g["rs_pos"]), 0, 0.0))
    acq2 = bo.UpperConfidenceBound(kappa=float(g["kappa"]))
    x2 = acq2.suggest(gp, space, random_state=rs)
    assert np.array_equal(x1, x2)


def test_constant_liar_vs_golden(bo, golden, TS):
    g = golden("constant_liar_small")
    space = TS(lambda x, y: -((x - 3) ** 2) - (y - 1) ** 2, {"x": (1, 4), "y": (0, 3.0)})
    for x, t in zip(g["X"], g["y"]):
        space.register(x, t)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), alpha=1e-6, normalize_y=True,
                                         n_restarts_optimizer=5, random_state=np.random.RandomState(0))
    cl = bo.ConstantLiar(bo.UpperConfidenceBound(kappa=2.576), strategy="max")
    rng = np.random.RandomState(5)
    sug = [cl.suggest(gp=gp, target_space=space, random_state=rng) for _ in range(4)]
    assert_allclose(np.array(sug), g["suggestions"], rtol=2e-3, atol=2e-3)
    assert len(cl.dummies) == 4


def test_constrained_suggest_runs_and_respects_errors(bo, TS):
    from bayes_opt.exception import ConstraintNotSupportedError, TargetSpaceEmptyError

    from scipy.optimize import NonlinearConstraint

    space = TS(lambda x, y: -((x - 3) ** 2) - (y - 1) ** 2, {"x": (1, 4), "y": (0, 3.0)},
               constraint=NonlinearConstraint(lambda x, y: x + y, -np.inf, 4.0))
    space._constraint._model = [bo.to_b200_gp(m) for m in space._constraint._model]  # what enable() does
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), alpha=1e-6, normalize_y=True,
                                         n_restarts_optimizer=2, random_state=np.random.RandomState(0))
    ei = bo.ExpectedImprovement(xi=0.01)
    with pytest.raises(TargetSpaceEmptyError):
        ei.suggest(gp, space, random_state=np.random.RandomState(1))
    rs = np.random.RandomState(0)
    for _ in range(8):
        space.probe(space.random_sample(random_state=rs))
    x = ei.suggest(gp, space, n_random=2000, n_smart=3, random_state=rs)
    assert x.shape == (2,) and np.all(x >= space.bounds[:, 0]) and np.all(x <= space.bounds[:, 1])
    with pytest.raises(ConstraintNotSupportedError):
        bo.UpperConfidenceBound().suggest(gp, space, random_state=rs)


def test_gphedge_runs_and_updates_gains(bo, TS):
    """GPHedge (R/bayes_opt/acquisition.py:1181-1360) over device base acquisitions."""
    space = TS(lambda x, y: -((x - 3) ** 2) - (y - 1) ** 2, {"x": (1, 4), "y": (0, 3.0)})
    rs = np.random.RandomState(0)
    for _ in range(6):
        space.probe(space.random_sample(random_state=rs))
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), alpha=1e-6, normalize_y=True,
                                         n_restarts_optimizer=2, random_state=np.random.RandomState(0))
    hedge = bo.GPHedge([bo.UpperConfidenceBound(kappa=2.0), bo.ExpectedImprovement(xi=0.01),
                        bo.ProbabilityOfImprovement(xi=0.01)])
    x1 = hedge.suggest(gp, space, n_random=3000, n_smart=3, random_state=rs)
    assert x1.shape == (2,) and hedge.previous_candidates.shape == (3, 2)
    space.probe(x1)
    x2 = hedge.suggest(gp, space, n_random=3000, n_smart=3, random_state=rs)
    assert np.any(hedge.gains != 0) and x2.shape == (2,)
    p = hedge.get_acquisition_params()
    h2 = bo.GPHedge([bo.UpperConfidenceBound(kappa=2.0), bo.ExpectedImprovement(xi=0.01),
                     bo.ProbabilityOfImprovement(xi=0.01)])
    h2.set_acquisition_params(p)
    assert h2.get_acquisition_params() == p
    with pytest.raises(TypeError):
        hedge.base_acq(0, 1)


def test_mixed_int_space_round_transform_and_de_branch(bo, golden, TS):
    """Float + int parameters: device np.round transform vs the reference's values, then the
    DifferentialEvolution + polish branch of _smart_minimize from the same RNG state."""
    from bayes_opt.parameter import wrap_kernel

    g = golden("mixed_int_small")
    space = TS(None, {"x": (0.0, 5.0), "k": (0, 6, int)})
    assert np.array_equal(space.random_sample(50, np.random.RandomState(9)), g["rand_draw"])
    for x, t in zip(g["X"], g["y"]):
        space.register(x, t)
    gp = make_gp(bo, wrap_kernel(Matern(nu=2.5, length_scale=1.3), space.kernel_transform)).fit(
        space.params, space.target)
    mu, sd = gp.predict(g["xt"], return_std=True)
    assert_allclose(mu, g["mu"], rtol=RTOL, atol=1e-10)
    assert_allclose(sd, g["sd"], rtol=RTOL, atol=1e-9)
    ei = bo.ExpectedImprovement(xi=0.01)
    ei.y_max = float(g["y_max"])
    assert_allclose(ei._get_acq(gp=gp)(g["xt"]), g["acq_ei"], rtol=RTOL, atol=1e-14)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sug = ei.suggest(gp, space, n_random=2000, n_smart=4, fit_gp=False, random_state=np.random.RandomState(11))
    assert_allclose(sug, g["suggestion"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("n,d,m", [(300, 4, 1000), (1024, 8, 20_000), (4096, 16, 40_000), (500, 20, 3000),
                                   (128, 1, 500), (129, 2, 777), (640, 3, 5000), (2000, 24, 10_000),
                                   (1500, 12, 4096), (3000, 16, 30_000), (700, 17, 2500), (256, 32, 4000),
                                   (1200, 64, 1500), (2048, 10, 65_536), (900, 5, 129), (4100, 16, 20_000)])
def test_fp32_mode_wgmma_vs_oracle(bo, O, n, d, m, monkeypatch):
    """fp32 mode (precision="fp32"): the N^2 term on the wgmma tensor cores (3xTF32, fp32 accumulate
    in registers); K*, the mean and the epilogue stay fp64.  Tolerance for this mode: 1e-3
    relative, stated on the quantity the reduced precision touches - the predictive VARIANCE:
    |d var| <= 1e-3*var + 1e-4*s_y^2 (sigma^2 is a difference of O(1) numbers; SURVEY section 7)."""
    X, y = _synth(n, d)
    s_y = float(np.std(y))
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7), precision="fp32").fit(X, y)
    gp64 = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(X, y)
    st = O.fit_fixed(X, y, length_scale=0.7)
    xt = np.random.RandomState(1).uniform(size=(m, d))
    a = bo.ExpectedImprovement(xi=0.01)
    a.y_max = float(y.max())
    f = a._get_acq(gp=gp)
    monkeypatch.setenv("B200BO_SMALL_PATH", "0")
    mu, sd = gp.predict(xt, return_std=True)
    ys = f(xt)
    idx, val, top = f.argmin_topk(xt, 10)
    mu0, sd0 = O.predict_chunked(st, xt)
    ref = O.acq_closure(st, O.ACQ_EI, xi=0.01, y_max=float(y.max()))(xt)
    assert_allclose(mu, mu0, rtol=RTOL, atol=1e-10)          # the mean never leaves fp64
    assert np.all(np.abs(sd**2 - sd0**2) <= 1e-3 * sd0**2 + 1e-4 * s_y**2)
    big = sd0 > 0.1 * s_y                                    # where sigma is not a cancellation residue
    assert_allclose(sd[big], sd0[big], rtol=1e-3)
    assert_allclose(ys[big], ref[big], rtol=2e-3, atol=1e-5 * s_y)
    # the selected point is (near-)optimal under the fp64 objective
    assert ref[idx] <= ref.min() + 2e-3 * abs(ref.min()) + 1e-5 * s_y
    # the fp64 handle is untouched by the other handle's mode
    assert_allclose(gp64.predict(xt[:256], return_std=True)[1], sd0[:256], rtol=RTOL, atol=1e-10)


def test_categorical_parameter_host_transform(bo, golden):
    """Categorical parameter: the reference's one-hot kernel transform (batch-dependent as written,
    R/bayes_opt/parameter.py:434-449) is an opaque callable -> applied on the host to each batch,
    exactly where WrappedKernel.__call__ applies it; values must equal the reference's."""
    from bayes_opt.parameter import wrap_kernel

    g = golden("categorical_small")

    def transform(v):  # == TargetSpace.kernel_transform of {"x": float, "c": 3 categories}
        v = np.atleast_2d(v)
        cat = v[:, 1:]
        res = np.zeros(cat.shape)
        res[:, np.argmax(cat, axis=1)] = 1
        return np.hstack([v[:, :1], res])

    assert np.array_equal(transform(g["X"]), g["X_transformed"])
    gp = make_gp(bo, wrap_kernel(Matern(nu=2.5, length_scale=1.1), transform)).fit(g["X"], g["y"])
    mu, sd = gp.predict(g["xt"], return_std=True)
    assert_allclose(mu, g["mu"], rtol=RTOL, atol=1e-10)
    assert_allclose(sd, g["sd"], rtol=RTOL, atol=1e-9)
    f = bo.UpperConfidenceBound(kappa=2.0)._get_acq(gp=gp)
    assert_allclose(f(g["xt"]), g["acq_ucb"], rtol=RTOL, atol=1e-10)
    assert_allclose([f(g["xt"][i])[0] for i in range(12)], g["acq_single"], rtol=RTOL, atol=1e-10)


@pytest.mark.parametrize("n,d,m", [(50, 2, 7), (700, 5, 100), (1024, 8, 257)])
def test_predict_return_cov_vs_sklearn(bo, n, d, m):
    """predict(return_cov=True) (SK/gaussian_process/_gpr.py:464-475) against the live sklearn GPR."""
    from sklearn.gaussian_process import GaussianProcessRegressor

    X, y = _synth(n, d)
    xt = np.random.RandomState(2).uniform(size=(m, d))
    k = ConstantKernel(1.5) * Matern(nu=2.5, length_scale=0.6)
    ref = GaussianProcessRegressor(kernel=k, alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)
    gp = make_gp(bo, k).fit(X, y)
    mu0, c0 = ref.predict(xt, return_cov=True)
    mu, c = gp.predict(xt, return_cov=True)
    assert c.shape == (m, m)
    assert_allclose(mu, mu0, rtol=RTOL, atol=1e-10)
    assert_allclose(c, c0, rtol=RTOL, atol=1e-9 * float(np.var(y)))
    assert_allclose(np.sqrt(np.maximum(np.diag(c), 0)), gp.predict(xt, return_std=True)[1], rtol=1e-6, atol=1e-7)
    with pytest.raises(RuntimeError):
        gp.predict(xt, return_std=True, return_cov=True)


def test_sample_y_uses_device_cov(bo):
    """sample_y (SK/gaussian_process/_gpr.py:502-539) is sklearn's own code over the device
    predict(return_cov=True): same draws as drawing from the device mean/cov directly, and close to
    the live sklearn GPR's samples on a well-conditioned posterior."""
    from sklearn.gaussian_process import GaussianProcessRegressor

    X, y = _synth(60, 2)
    xt = np.random.RandomState(4).uniform(size=(6, 2))
    k = Matern(nu=2.5, length_scale=0.4)
    gp = make_gp(bo, k).fit(X, y)
    s = gp.sample_y(xt, n_samples=5, random_state=7)
    assert s.shape == (6, 5)
    mu, c = gp.predict(xt, return_cov=True)
    assert_allclose(s, np.random.RandomState(7).multivariate_normal(mu, c, 5).T, rtol=1e-12, atol=1e-12)
    ref = GaussianProcessRegressor(kernel=k, alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)
    assert_allclose(s, ref.sample_y(xt, n_samples=5, random_state=7), rtol=1e-4, atol=1e-6)


def test_incremental_append_equals_full_fit(bo, O):
    """Fixed theta: fitting on X[:n+k] after X[:n] extends the factor in O(N^2) per row
    (b200bo_gp_append) and must equal a from-scratch fit, incl. across the 128-row padding edge."""
    X, y = _synth(140, 3)
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.5))
    gp.fit(X[:120], y[:120])
    launches = bo._lib.lib().b200bo_launch_count
    for n in (121, 124, 128, 129, 131):   # 128 -> 129 crosses the capacity: falls back to a full fit
        l0 = launches()
        gp.fit(X[:n], y[:n])
        used = launches() - l0
        st = O.fit_fixed(X[:n], y[:n], length_scale=0.5)
        assert_allclose(gp.L_, st.L, rtol=1e-8, atol=1e-11)
        assert_allclose(gp.alpha_, st.alpha_, rtol=1e-6, atol=1e-9)
        xt = np.random.RandomState(n).uniform(size=(50, 3))
        mu, sd = gp.predict(xt, return_std=True)
        mu0, sd0 = O.predict(st, xt)
        assert_allclose(mu, mu0, rtol=RTOL, atol=1e-10)
        assert_allclose(sd, sd0, rtol=RTOL, atol=1e-9)
        if n in (121, 124, 128, 131):
            assert used < 60, (n, used)   # incremental path (a full fit at np=128/256 is > 20 launches/row...)
    # duplicate point with alpha=0 -> not positive definite, as a full fit would report
    gp0 = make_gp(bo, Matern(nu=2.5, length_scale=0.5), alpha=0.0, normalize_y=False).fit(X[:20], y[:20])
    with pytest.raises(np.linalg.LinAlgError):
        gp0.fit(np.vstack([X[:20], X[:1]]), np.append(y[:20], y[0]))


def test_sharded_argmin_topk_single_process_group(bo, golden):
    """The sharded selection helper (one all_gather of (k+1) records) on a 1-rank gloo group, two
    shards evaluated in turn: merged result == single-batch result."""
    import socket

    import torch.distributed as dist

    from bayesianoptimization_b200.sharding import merge_selection, shard_range, sharded_argmin_topk

    g = golden("c2s_ei")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(g["X"], g["y"])
    a = bo.ExpectedImprovement(xi=float(g["xi"]))
    a.y_max = float(g["y_max"])
    f = a._get_acq(gp=gp)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        bi, bv, top = sharded_argmin_topk(f, g["xt"], 10, 0)
        assert bi == int(g["argmin"]) and list(top) == list(g["top10"])
    finally:
        dist.destroy_process_group()
    # two shards merged by hand with the same record format
    vals, idxs = np.full((2, 11), np.nan), np.full((2, 11), -1, dtype=np.int64)
    for r in range(2):
        s0, s1 = shard_range(len(g["xt"]), r, 2)
        i, v, t = f.argmin_topk(g["xt"][s0:s1], 10)
        vals[r, 0], idxs[r, 0] = v, s0 + i
        vals[r, 1:1 + len(t)], idxs[r, 1:1 + len(t)] = f(g["xt"][s0:s1][t]), s0 + t
    bi, bv, top = merge_selection(vals, idxs, 10)
    assert bi == int(g["argmin"]) and list(top) == list(g["top10"])


def test_empty_and_single_candidate_batches(bo, golden):
    """Edge shapes: zero candidates (empty result), one candidate, (d,) vs (1,d) input, argmin on 1."""
    g = golden("c2s_ei")
    gp = make_gp(bo, Matern(nu=2.5, length_scale=0.7)).fit(g["X"], g["y"])
    f = bo.UpperConfidenceBound(kappa=2.0)._get_acq(gp=gp)
    assert f(np.empty((0, 8))).shape == (0,)
    y1 = f(g["xt"][3])
    y2 = f(g["xt"][3:4])
    assert y1.shape == (1,) and np.array_equal(y1, y2)
    idx, val, top = f.argmin_topk(g["xt"][3:4], 10)
    assert idx == 0 and val == y1[0] and list(top) == [0]
    with pytest.raises(ValueError):
        f(np.array([[np.nan] * 8]))
    with pytest.raises(ValueError):
        gp.predict(np.zeros((3, 5)))

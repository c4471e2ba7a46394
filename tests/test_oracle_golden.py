"""Pin the oracle (oracle/gp_oracle.py) to the reference: golden fixtures produced by the
unmodified reference (oracle/make_golden.py) and the live sklearn GPR (the reference's own
numerical substrate, installed in this image)."""
import numpy as np
import pytest
from numpy.testing import assert_allclose
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern

from oracle import gp_oracle as O

RT = 1e-9  # oracle vs reference: same algorithm, same libraries -> near round-off


def test_c1_readme_ucb(golden):
    g = golden("c1_readme_ucb")
    st = O.fit_fixed(g["X"], g["y"], length_scale=float(g["length_scale"]))
    assert_allclose(st.L, g["L"], rtol=1e-10, atol=1e-13)
    assert_allclose(st.alpha_, g["alpha_"], rtol=1e-7)
    mu, sd = O.predict(st, g["xt"])
    assert_allclose(mu, g["mu"], rtol=RT, atol=1e-10)
    assert_allclose(sd, g["sd"], rtol=1e-7, atol=1e-10)
    acq = O.acq_closure(st, O.ACQ_UCB, kappa=float(g["kappa"]))
    ys = acq(g["xt"])
    assert_allclose(ys, g["acq"], rtol=1e-7, atol=1e-10)
    assert int(np.argmin(ys)) == int(np.argmin(g["acq"]))
    assert_allclose([acq(g["xt"][i])[0] for i in range(16)], g["acq_single"], rtol=1e-7, atol=1e-10)


def test_c2s_ei_poi_ucb(golden):
    g = golden("c2s_ei")
    st = O.fit_fixed(g["X"], g["y"], length_scale=float(g["length_scale"]))
    K = O.kernel_train(g["X"], length_scale=float(g["length_scale"]))
    assert_allclose(K, g["K"], rtol=1e-13, atol=0)
    assert_allclose(st.L, g["L"], rtol=1e-9, atol=1e-13)
    assert_allclose(st.alpha_, g["alpha_"], rtol=1e-6)
    assert st.y_mean == pytest.approx(float(g["y_mean"]), rel=1e-14)
    assert st.y_std == pytest.approx(float(g["y_std"]), rel=1e-14)
    mu, sd = O.predict(st, g["xt"])
    assert_allclose(mu, g["mu"], rtol=RT, atol=1e-11)
    assert_allclose(sd, g["sd"], rtol=RT, atol=1e-12)
    kw = dict(kappa=float(g["kappa"]), xi=float(g["xi"]), y_max=float(g["y_max"]))
    for kind, key in [(O.ACQ_EI, "acq_ei"), (O.ACQ_POI, "acq_poi"), (O.ACQ_UCB, "acq_ucb")]:
        ys = O.acq_closure(st, kind, **kw)(g["xt"])
        assert_allclose(ys, g[key], rtol=1e-7, atol=1e-13)
    ys = O.acq_closure(st, O.ACQ_EI, **kw)(g["xt"])
    i, v, top = O.argmin_topk(ys, 10)
    assert i == int(g["argmin"])
    assert list(top) == list(g["top10"])


def test_c2s_edge_near_duplicates(golden):
    g = golden("c2s_ei")
    st = O.fit_fixed(g["X"], g["y"], length_scale=float(g["length_scale"]))
    mu, sd = O.predict(st, g["xe"])
    assert_allclose(mu, g["mu_e"], rtol=1e-8, atol=1e-9)
    # sigma near the jitter floor is a difference of O(1) numbers: absolute tolerance
    assert_allclose(sd, g["sd_e"], rtol=1e-4, atol=1e-7)


def test_c2s_lml(golden):
    g = golden("c2s_ei")
    yn, _, _ = O.normalize_y(g["y"])
    for t, v, gr in zip(g["thetas"], g["lml"], g["lml_grad"]):
        lml, grad = O.lml_and_grad(g["X"], yn, length_scale=float(np.exp(t)))
        assert lml == pytest.approx(v, rel=1e-9, abs=1e-9)
        assert grad[0] == pytest.approx(gr, rel=1e-7, abs=1e-7)


KERNELS = {
    "m05": dict(kind=O.KIND_MATERN, nu=0.5, length_scale=0.6),
    "m15": dict(kind=O.KIND_MATERN, nu=1.5, length_scale=0.6),
    "rbf": dict(kind=O.KIND_RBF, length_scale=0.6),
    "m25aniso": dict(kind=O.KIND_MATERN, nu=2.5, length_scale=np.array([0.3, 0.6, 1.2, 2.4])),
    "crbf": dict(kind=O.KIND_RBF, length_scale=0.8, const=2.0),
    "cm25": dict(kind=O.KIND_MATERN, nu=2.5, length_scale=0.5, const=0.5),
}


@pytest.mark.parametrize("tag", sorted(KERNELS))
def test_kernel_families(golden, tag):
    g = golden("kernels_small")
    kw = KERNELS[tag]
    st = O.fit_fixed(g["X"], g["y"], **kw)
    assert_allclose(st.L, g[f"{tag}_L"], rtol=1e-9, atol=1e-12)
    mu, sd = O.predict(st, g["xt"])
    assert_allclose(mu, g[f"{tag}_mu"], rtol=1e-8, atol=1e-9)
    assert_allclose(sd, g[f"{tag}_sd"], rtol=1e-7, atol=1e-9)
    lml, grad = O.lml_and_grad(g["X"], st.y_norm, **kw)
    assert lml == pytest.approx(float(g[f"{tag}_lml"]), rel=1e-9)
    assert_allclose(grad, g[f"{tag}_lml_grad"], rtol=1e-6, atol=1e-7)


def test_c4s_constrained(golden):
    g = golden("c4s_constrained")
    st = O.fit_fixed(g["X"], g["y"], length_scale=float(g["ls"]))
    cs = [O.fit_fixed(g["X"], g["c"][:, j], length_scale=float(g["ls_c"][j])) for j in range(2)]
    p = O.constraint_prob(cs, g["lb"], g["ub"], g["xt"])
    assert_allclose(p, g["p"], rtol=1e-7, atol=1e-12)
    p1 = O.constraint_prob([cs[1]], [-0.5], [0.5], g["xt"])
    assert_allclose(p1, g["p1"], rtol=1e-7, atol=1e-12)
    kw = dict(xi=float(g["xi"]), y_max=float(g["y_max"]), constraint=(cs, g["lb"], g["ub"]))
    assert_allclose(O.acq_closure(st, O.ACQ_POI, **kw)(g["xt"]), g["acq_poi"], rtol=1e-7, atol=1e-13)
    assert_allclose(O.acq_closure(st, O.ACQ_EI, **kw)(g["xt"]), g["acq_ei"], rtol=1e-7, atol=1e-13)
    approx = np.column_stack([O.predict(c, g["xt"], return_std=False) for c in cs])
    assert_allclose(approx, g["approx"], rtol=1e-8, atol=1e-10)


@pytest.mark.parametrize("kern,kw", [
    (Matern(nu=2.5, length_scale=0.4), dict(length_scale=0.4)),
    (ConstantKernel(1.7) * RBF(length_scale=1.1), dict(kind=O.KIND_RBF, length_scale=1.1, const=1.7)),
])
def test_oracle_vs_live_sklearn(kern, kw):
    """Runs anywhere sklearn is installed (this image, incl. the GPU machine)."""
    rs = np.random.RandomState(11)
    X = rs.uniform(size=(200, 6))
    y = np.cos(X.sum(1)) + 0.05 * rs.randn(200)
    xt = rs.uniform(size=(1000, 6))
    gp = GaussianProcessRegressor(kernel=kern, alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)
    st = O.fit_fixed(X, y, **kw)
    mu0, sd0 = gp.predict(xt, return_std=True)
    mu, sd = O.predict(st, xt)
    assert_allclose(mu, mu0, rtol=1e-9, atol=1e-11)
    assert_allclose(sd, sd0, rtol=1e-8, atol=1e-11)
    v0, g0 = gp.log_marginal_likelihood(gp.kernel_.theta, eval_gradient=True)
    v, g = O.lml_and_grad(X, st.y_norm, **kw)
    assert v == pytest.approx(v0, rel=1e-10)
    assert_allclose(g, g0, rtol=1e-7, atol=1e-8)


def test_mixed_int_round_transform(golden):
    g = golden("mixed_int_small")

    def tr(v):
        v = np.array(np.atleast_2d(v), dtype=float)
        v[:, 1] = np.round(v[:, 1])
        return v

    st = O.fit_fixed(tr(g["X"]), g["y"], length_scale=1.3)
    mu, sd = O.predict(st, tr(g["xt"]))
    assert_allclose(mu, g["mu"], rtol=1e-9, atol=1e-11)
    assert_allclose(sd, g["sd"], rtol=1e-8, atol=1e-11)
    ys = O.acq_closure(st, O.ACQ_EI, xi=0.01, y_max=float(g["y_max"]))(tr(g["xt"]))
    assert_allclose(ys, g["acq_ei"], rtol=1e-7, atol=1e-14)


def test_philox_oracle_known_answer_vectors():
    """oracle.philox4x32_10 against the published known-answer vectors of Philox4x32-10 (Random123
    kat_vectors: counter / key all zero, all ones, digits of pi)."""
    from oracle import gp_oracle as O

    kat = [
        ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
        ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
        ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
         (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
    ]
    for ctr, key, want in kat:
        got = O.philox4x32_10(*[[c] for c in ctr], *key)
        assert tuple(int(g[0]) for g in got) == want
    x = O.philox_uniform(7, [0, 1, 2**33 + 5], 3, [0, 0, -1], [1, 2, 1])
    assert x.shape == (3, 3) and np.all(x[:, 0] >= 0) and np.all(x[:, 0] < 1) and np.all(np.abs(x[:, 2]) <= 1)
    big = O.philox_uniform(99, np.arange(200_000), 2, [0, 0], [1, 1])
    assert abs(big.mean() - 0.5) < 2e-3 and abs(big.var() - 1 / 12) < 2e-3


def test_gphedge_fixture_shapes(golden):
    g = golden("gphedge_small")
    assert g["suggestions"].shape == (4, 2) and g["gains"].shape == (4, 3) and g["candidates"].shape == (4, 3, 2)
    assert np.all(g["gains"][0] == 0) and np.any(g["gains"][1] != 0)

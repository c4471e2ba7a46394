"""The extended-precision fixtures of the conditioned posteriors, sample paths and input gradients
(oracle/make_illcond_ext.py, tests/golden/illext_*.npz), without a GPU: the small case regenerates bit-equal from its
stored inputs, the stored draws are those of paths.draw_path_inputs, the analytic gradients agree with 50-digit
central differences, the truth agrees with itself, and the fixtures span the conditions the GPU tests
(tests/test_gpu_illcond_ext.py) are meant to stress."""
import mpmath as mp
import numpy as np
import pytest

from oracle import make_illcond as MI
from oracle import make_illcond_ext as XE

INPUTS = ("X", "y", "xt", "group", "P_incumbent", "P_edge", "P_believer", "believer_idx", "omega", "b", "w", "eps")


def _load(name):
    with np.load(XE.fixture_path(name)) as z:
        return {k: z[k] for k in z.files}


def _close_ulps(a, b, ulps=4):
    return np.all(np.abs(a - b) <= ulps * np.spacing(np.maximum(np.abs(a), np.abs(b))))


def test_small_case_regenerates_bit_equal():
    """The extended-precision results of the stored inputs are bit-equal to the fixture; the fp64 referee's (the
    BLAS build's) are compared at a tolerance."""
    want = _load(MI.SMALL_CASE)
    got = XE.make_case(MI.SMALL_CASE, inputs={k: want[k] for k in INPUTS})
    assert set(got) == set(want)
    for k in sorted(got):
        if k.startswith("sk_"):
            np.testing.assert_allclose(got[k], want[k], rtol=1e-6, atol=1e-12, err_msg=k)
        else:
            assert np.array_equal(np.asarray(got[k]), want[k]), k


@pytest.mark.parametrize("name", sorted(MI.CASES))
def test_inputs_and_draws_reproduce(name):
    """Every case has a fixture; its training inputs are illcond_<case>'s, the incumbent and edge sequences come
    from the builder (to a few ulp: libm), the believer picks are distinct candidates, and the path draws equal
    draw_path_inputs(RandomState(seed), ...) bit for bit."""
    from bayesianoptimization_b200.paths import draw_path_inputs

    c, r = MI.CASES[name], _load(name)
    with np.load(MI.fixture_path(name)) as z:
        for k in ("X", "y", "xt", "group"):
            assert np.array_equal(r[k], z[k]), k
    rs = np.random.RandomState(1000 + c["seed"])
    d = c["d"]
    dirs = rs.randn(XE.N_INC, d)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    inc = int(np.argmax(r["y"]))
    assert _close_ulps(r["P_incumbent"], r["X"][inc] + np.geomspace(1e-2, 1e-6, XE.N_INC)[:, None] * dirs)
    assert r["P_edge"].shape == (XE.N_EDGE, d)
    assert np.array_equal(r["P_edge"][XE.EDGE_REPEAT[0]], r["P_edge"][XE.EDGE_REPEAT[1]])  # the exact repeat
    idx = r["believer_idx"]
    assert len(set(idx.tolist())) == XE.N_BEL and np.array_equal(r["P_believer"], r["xt"][idx])
    draws = draw_path_inputs(np.random.RandomState(c["seed"]), XE.N_PATHS, XE.N_FEATURES, d, XE.NU[c["kern"]],
                             c["n"], c["alpha"] + (c.get("white") or 0.0))
    for k, v in zip(("omega", "b", "w", "eps"), draws):
        assert np.array_equal(r[k], v), k


def _posterior_mp(case, X, y, P=None):
    """x (scaled mp row) -> (mu, sd) of the 50-digit posterior, conditioned on P with the exact believer targets
    (mu_norm(P) = k(P, X) alpha_, alpha' = [alpha_; 0]) when P is given; K' factorised from scratch."""
    mp.mp.dps = MI.DPS
    n = len(X)
    c = mp.mpf(case.get("const") or 1.0)
    prior = c + mp.mpf(case.get("white") or 0.0)
    Xa = X if P is None else np.vstack([X, P])
    L = MI._cholesky(MI.kernel_matrix_mp(case, Xa))
    ym = [mp.mpf(float(v)) for v in y]
    mean = mp.fsum(ym) / n
    std = mp.sqrt(mp.fsum([(v - mean) ** 2 for v in ym]) / n)
    Lo = MI._cholesky(MI.kernel_matrix_mp(case, X))
    alpha_ = MI._backward(Lo, MI._forward(Lo, [(v - mean) / std for v in ym]))
    Xs = MI._scaled(case, Xa)

    def post(row):
        ks = [c * MI._cov(case["kern"], mp.fsum(MI._dsq(row, xr))) for xr in Xs]
        V = MI._forward(L, ks)
        return mp.fdot(ks[:n], alpha_) * std + mean, mp.sqrt((prior - mp.fdot(V, V)) * std * std)

    return post


def test_analytic_gradients_agree_with_central_differences():
    """On the small case, the stored value and gradient of every closure, on the original and on the conditioned GP,
    against 50-digit central differences (step 1e-15 ls) of the full posterior, on rows inside the cluster, at and
    1e-7 / 1e-9 from training rows, near the incumbent and uniform ones."""
    name = MI.SMALL_CASE
    case, r = MI.CASES[name], _load(name)
    ls = [mp.mpf(float(v)) for v in MI._ls_vec(case)]
    y_max = float(np.max(r["y"]))
    rows = [int(np.flatnonzero(r["group"] == g)[j]) for g, j in
            ((MI.G_CLUSTER, 0), (MI.G_TRAIN, 1), (MI.G_DUP7, 2), (MI.G_DUP9, 3), (MI.G_INC, 12), (MI.G_UNIFORM, 5))]
    h = mp.mpf("1e-15")
    for gname, P in (("orig", None), ("cond", r["P_incumbent"][:XE.N_COND_GRAD])):
        post = _posterior_mp(case, r["X"], r["y"], P)

        def closures(row):
            mu, sd = post(row)
            return XE._closures(mu, sd, [], [], y_max, list(r["mes_ystar"]))

        for t in rows:
            row = MI._scaled(case, r["xt"][t:t + 1])[0]
            base = closures(row)
            for j in range(case["d"]):
                up, dn = row[:], row[:]
                up[j] += h / ls[j]
                dn[j] -= h / ls[j]
                cu, cd = closures(up), closures(dn)
                for kind in XE.KINDS:
                    fd = float((cu[kind][0] - cd[kind][0]) / (2 * h))
                    g = r[f"gr_{gname}_{kind}_grad"][t]
                    v = r[f"gr_{gname}_{kind}_val"][t]
                    assert abs(float(base[kind][0]) - v) <= 1e-15 * abs(v), (gname, kind, t)
                    scale = np.max(np.abs(g)) + abs(r[f"gr_{gname}_{kind}_val"][t]) + 1e-300
                    assert abs(fd - g[j]) <= 1e-12 * scale, (gname, kind, t, j, fd, g[j])


@pytest.mark.parametrize("name", sorted(MI.CASES))
def test_truth_is_self_consistent(name):
    """Conditioning keeps the mean, never raises the variance and lowers it as the prefix grows; every pivot is
    positive; a believer pick's target is the original mean at that candidate; the acquisitions follow from mu and
    sigma; the referee is close to the truth."""
    from oracle import gp_oracle as O

    r = _load(name)
    with np.load(MI.fixture_path(name)) as z:
        mu0, var0 = z["mu"], z["var"]
    y_max = float(np.max(r["y"]))
    for s in XE.SEQS:
        assert np.all(r[f"{s}_pivot"] > 0)
        prev = var0
        for p in XE.prefixes(s):
            k = f"{s}_p{p}"
            assert np.array_equal(r[f"{k}_mu"], mu0), k
            assert np.all(r[f"{k}_var"] > 0) and np.all(r[f"{k}_var"] <= prev * (1 + 1e-14)), k
            prev = r[f"{k}_var"]
            sd = np.sqrt(r[f"{k}_var"])
            for kind, code in (("ucb", O.ACQ_UCB), ("ei", O.ACQ_EI), ("poi", O.ACQ_POI)):
                ref = O.base_acq(code, r[f"{k}_mu"], sd, kappa=MI.KAPPA, xi=MI.XI, y_max=y_max)
                np.testing.assert_allclose(r[f"{k}_acq_{kind}"], ref, rtol=1e-9, atol=1e-300, err_msg=f"{k} {kind}")
            np.testing.assert_allclose(r[f"sk_{k}_mu"], mu0, rtol=1e-5, atol=1e-5 * np.std(r["y"]))
    assert np.array_equal(r["believer_target"], mu0[r["believer_idx"]])
    for g, var in (("orig", var0), ("cond", r[f"incumbent_p{XE.N_COND_GRAD}_var"])):
        np.testing.assert_allclose(-r[f"gr_{g}_ucb_val"], mu0 + MI.KAPPA * np.sqrt(var), rtol=1e-14,
                                   atol=1e-15 * np.max(np.abs(mu0)))
    np.testing.assert_allclose(r["sk_path_val"], r["path_val"], rtol=1e-5, atol=1e-5 * np.std(r["y"]))


def test_fixtures_span_the_intended_conditions():
    piv = {}
    for name, c in MI.CASES.items():
        r = _load(name)
        diag = (c.get("const") or 1.0) + (c.get("white") or 0.0) + c["alpha"]
        piv[name] = min(float(np.min(r[f"{s}_pivot"])) for s in XE.SEQS) / np.sqrt(diag)
        # every exact pivot is at least about sqrt(alpha): the conditioned noise-free variance plus the jitter
        assert piv[name] >= 0.99 * np.sqrt(c["alpha"] / diag), name
    assert min(piv.values()) < 1e-4
    assert 1e-10 in {c["alpha"] for c in MI.CASES.values()}
    assert any(c.get("cluster") and c["d"] == 17 for c in MI.CASES.values())
    # the chained conditioning of c_m25_d3 (n = 121) on the 64 incumbent rows crosses the 128-row padding
    assert MI.CASES["c_m25_d3"]["n"] < 128 < MI.CASES["c_m25_d3"]["n"] + XE.N_INC

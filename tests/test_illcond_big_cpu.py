"""The double-double reference (oracle/dd.py) and the production-size fixtures it builds (oracle/make_illcond_big.py,
tests/golden/illbig_*.npz), without a GPU.

The reference is refereed by the 50-digit fixtures of oracle/make_illcond.py: on every one of them its results
rounded to fp64 are bit-equal to the stored truth, and on the small case its unrounded results agree with mpmath to
1e-23 (measured: 6.5e-25 on sigma^2, where cond(K) = 6e7 amplifies the 1e-32 roundoff).  Then the big fixtures:
covariance entries against mpmath, the smallest case regenerates bit-equal, and the fixtures span the conditions and
the device's size gates that tests/test_gpu_illcond_big.py is meant to stress."""
import mpmath as mp
import numpy as np
import pytest

from oracle import dd
from oracle import make_illcond as MI
from oracle import make_illcond_big as MB

TRUTH_KEYS = ("mu", "var", "sd", "acq_ucb", "acq_ei", "acq_poi", "alpha_", "lml", "lml_grad")
BIG = sorted(MB.CASES)


def _load(path):
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", sorted(MI.CASES))
def test_dd_matches_the_50_digit_fixtures(name):
    """K, L, alpha_, mu, sigma^2 (relative at every candidate, training rows and their 1e-7 / 1e-9 neighbours
    included), the acquisitions, the LML and its gradient: bit-equal after rounding to fp64."""
    c, r = MI.CASES[name], _load(MI.fixture_path(name))
    res, fit = dd.posterior(c, r["X"], r["y"], r["xt"], MI.KAPPA, MI.XI)
    n = len(r["X"])
    for k in TRUTH_KEYS:
        assert np.array_equal(np.asarray(res[k]), r[k]), k
    assert np.array_equal(dd.l_dense(fit)[np.tril_indices(n)], r["L_packed"])
    assert res["prior"] == r["prior"] and res["y_std"] == r["y_std"]


def test_dd_against_mpmath_unrounded():
    """The double-double values themselves (hi + lo) against 50 digits on the small case: K, L, alpha_ and sigma^2 within
    1e-23 relative to the largest entry (sigma^2 relative to itself)."""
    name = MI.SMALL_CASE
    c, r = MI.CASES[name], _load(MI.fixture_path(name))
    mp.mp.dps = MI.DPS
    fit = dd.Fit(c, r["X"], r["y"])
    n = fit.n
    K = MI.kernel_matrix_mp(c, r["X"])
    L = MI._cholesky(K)

    def err(pair, ref, rows, cols):
        e = max(abs(dd.to_mp(pair[0][i, j], pair[1][i, j]) - ref[i][j]) for i in rows for j in cols(i))
        return float(e / max(abs(ref[i][j]) for i in rows for j in cols(i)))

    e_K = err(fit.K, K, range(n), lambda i: range(i + 1))
    e_L = err(fit.L, L, range(n), lambda i: range(i + 1))
    ym = [mp.mpf(float(v)) for v in r["y"]]
    yn = [(v - fit.y_mean) / fit.y_std for v in ym]
    a = MI._backward(L, MI._forward(L, yn))
    e_a = float(max(abs(dd.to_mp(fit.alpha_[0][i], fit.alpha_[1][i]) - a[i]) for i in range(n)) / max(map(abs, a)))
    xs = dd.scaled(c, r["xt"][::8])
    Ks = fit.cross(xs)
    var = fit.variance(Ks, [n])[0]
    Xs, Xt = MI._scaled(c, r["X"]), MI._scaled(c, r["xt"][::8])
    e_v = 0.0
    for t, row in enumerate(Xt):
        V = MI._forward(L, [MI._cov(c["kern"], mp.fsum(MI._dsq(row, xr))) for xr in Xs])
        want = (fit.prior - mp.fdot(V, V)) * fit.y_std ** 2
        e_v = max(e_v, float(abs(var[t] - want) / want))
    print(f"\nK {e_K:.1e} L {e_L:.1e} alpha_ {e_a:.1e} var {e_v:.1e}")
    assert max(e_K, e_L, e_a, e_v) <= 1e-23  # measured K 4.0e-32 L 6.9e-28 alpha_ 1.1e-25 var 6.5e-25


@pytest.mark.parametrize("name", BIG)
def test_big_covariance_entries_against_mpmath(name):
    """300 random entries of K* (candidates against training rows) and of K: the double-double covariance within
    1e-29 of sklearn's formula at 50 digits (the entries are O(1) and the inputs exact)."""
    c, r = MB.CASES[name], MB.load(name)
    rs = np.random.RandomState(7)
    A = np.vstack([r["xt"][rs.randint(len(r["xt"]), size=200)], r["X"][rs.randint(len(r["X"]), size=100)]])
    B = r["X"][rs.randint(len(r["X"]), size=300)]
    kh, kl = dd.cross_cov(dd.scaled(c, A), dd.scaled(c, B), dd.CODES[c["kern"]], float(c.get("const") or 1.0))
    mp.mp.dps = MI.DPS
    cm = mp.mpf(c.get("const") or 1.0)
    As, Bs = MI._scaled(c, A), MI._scaled(c, B)
    worst = 0.0
    for i in range(len(A)):
        want = cm * MI._cov(c["kern"], mp.fsum(MI._dsq(As[i], Bs[i])))
        worst = max(worst, float(abs(dd.to_mp(kh[i, i], kl[i, i]) - want) / cm))
    print(f"\n{name} max |dk| / const {worst:.1e}")
    assert worst <= 1e-29


def test_smallest_big_case_regenerates_bit_equal():
    """The double-double results of the stored inputs are bit-equal to the fixture (fixed-order reductions, no FMA).
    cond(K) comes from LAPACK and sklearn's results from the BLAS build: those are compared at a tolerance."""
    want = MB.load(MB.SMALL_CASE)
    got = MB.make_case(MB.SMALL_CASE, inputs=tuple(want[k] for k in ("X", "y", "xt", "group", "P")))
    assert set(got) == set(want)
    with np.load(MB.fixture_path(MB.SMALL_CASE)) as z:  # and stored() writes what the fixture holds
        assert set(MB.stored(got, MB.CASES[MB.SMALL_CASE])) == set(z.files)
    platform = {k for k in got if k.startswith("sk_")} | {"cond"}
    for k in sorted(set(got) - platform):
        assert np.array_equal(np.asarray(got[k]), want[k]), k
    for k in sorted(platform):
        np.testing.assert_allclose(got[k], want[k], rtol=1e-6, atol=1e-9, err_msg=k)


def test_big_fixtures_have_their_inputs():
    """X and the uniform candidates are rebuilt from the seeds and match the fixture's digests (load() checks them);
    the stored rows are those the builders give, to a few ulp."""
    for name, c in MB.CASES.items():
        r = MB.load(name)
        X, y, xt, group, P = MB.problem(c)
        assert np.array_equal(r["X"], X) and len(r["xt"]) == MB.CANDIDATES, name
        assert np.array_equal(r["group"], group), name
        for k, v in (("y", y), ("xt", xt), ("P", P)):  # through libm: a few ulp
            assert np.all(np.abs(r[k] - v) <= 4 * np.spacing(np.maximum(np.abs(r[k]), np.abs(v)))), (name, k)


def test_big_fixtures_fit_the_repository():
    """Each fixture under 1 MB: the rows that are exact functions of the seeds are rebuilt, not stored."""
    import os

    for name in BIG:
        assert os.path.getsize(MB.fixture_path(name)) < 1_000_000, name


def test_load_refuses_inputs_that_differ(tmp_path):
    """A fixture whose digest does not match the rebuilt rows is refused, not silently compared with other inputs."""
    name = MB.SMALL_CASE
    with np.load(MB.fixture_path(name)) as z:
        r = {k: z[k] for k in z.files}
    r["X_sha256"] = np.array("0" * 64)
    p = tmp_path / "bad.npz"
    np.savez_compressed(p, **r)
    with pytest.raises(ValueError):
        MB.load(name, str(p))


def test_big_fixtures_span_the_intended_conditions():
    """cond(K) from 1e7 to 1e11; N past the refine gate of pruning (N > 896) on every case, with np = N at the C3 shape
    and N ragged against 64 and 128 elsewhere; d = 17 (no candidate registers); at least 32 candidate tiles of 128."""
    rs = {name: MB.load(name) for name in BIG}
    conds = {name: float(r["cond"]) for name, r in rs.items()}
    print("\n" + " ".join(f"{k} {v:.1e}" for k, v in conds.items()))
    assert min(conds.values()) < 1e7 and max(conds.values()) > 1e11
    ns = {name: len(r["X"]) for name, r in rs.items()}
    assert all(n > 896 for n in ns.values())
    assert ns["b_m25_c3"] == 4096 and rs["b_m25_c3"]["X"].shape[1] == 16
    assert sum(n % 64 != 0 for n in ns.values()) >= 3
    assert any(r["X"].shape[1] > 16 for r in rs.values())
    assert {c["kern"] for c in MB.CASES.values()} == {"m05", "m15", "m25", "rbf"}
    for r in rs.values():
        assert len(r["xt"]) == MB.CANDIDATES >= 32 * 128
        assert len(r["P"]) == MB.N_PEND


@pytest.mark.parametrize("name", BIG)
def test_big_fixture_is_self_consistent(name):
    """The stored truth agrees with itself in fp64: 0 < sigma^2 <= prior, sigma^2 falls with every pending row, the
    acquisitions follow from mu and sigma, and sklearn is near it.  Prints sklearn's errors against the truth."""
    from oracle import gp_oracle as O

    r = MB.load(name)
    prior = r["prior"] * r["y_std"] ** 2
    assert np.all(r["var"] > 1e-12 * prior) and np.all(r["var"] <= prior)
    v = [r["var"]] + [r[f"inc_p{p}_var"] for p in MB.PREFIXES]
    assert all(np.all(b <= a) and np.all(b > 0) for a, b in zip(v, v[1:]))
    np.testing.assert_allclose(r["sd"] ** 2, r["var"], rtol=1e-14)
    y_max = float(np.max(r["y"]))
    for kind, code in (("ucb", O.ACQ_UCB), ("ei", O.ACQ_EI), ("poi", O.ACQ_POI)):
        ref = O.base_acq(code, r["mu"], r["sd"], kappa=MI.KAPPA, xi=MI.XI, y_max=y_max)
        np.testing.assert_allclose(r[f"acq_{kind}"], ref, rtol=1e-9, atol=1e-300, err_msg=kind)
    assert np.all(r["inc_pivot"] > 0) and r["L_rows"].shape == (len(r["L_rows_idx"]), len(r["X"]))
    assert np.array_equal(np.diag(r["L_rows"][:, r["L_rows_idx"]]), r["L_diag"][r["L_rows_idx"]])
    e = dict(mu=np.max(np.abs(r["sk_mu"] - r["mu"]) / (np.abs(r["mu"]) + r["y_std"])),
             sd=np.max(np.abs(r["sk_sd"] - r["sd"]) / r["sd"]),
             alpha=np.max(np.abs(r["sk_alpha_"] - r["alpha_"])) / np.max(np.abs(r["alpha_"])),
             lml=abs(r["sk_lml"] - r["lml"]) / abs(r["lml"]),
             grad=np.max(np.abs(r["sk_lml_grad"] - r["lml_grad"])) / max(np.max(np.abs(r["lml_grad"])), 1.0))
    print(f"\n{name} cond {float(r['cond']):.1e} sklearn: " + " ".join(f"{k} {v:.1e}" for k, v in e.items()))
    assert e["mu"] <= 1e-4 and r["lml_grad"].shape == r["sk_lml_grad"].shape

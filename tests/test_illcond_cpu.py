"""The extended-precision fixtures of the ill-conditioned cases (oracle/make_illcond.py, tests/golden/illcond_*.npz),
without a GPU: one small case regenerates bit-equal to its fixture, and the fixtures span the conditions the GPU
tests (tests/test_gpu_illcond.py) are meant to stress."""
import numpy as np
import pytest

from oracle import make_illcond as MI


def _load(name):
    with np.load(MI.fixture_path(name)) as z:
        return {k: z[k] for k in z.files}


def _close_ulps(a, b, ulps=4):
    return np.all(np.abs(a - b) <= ulps * np.spacing(np.maximum(np.abs(a), np.abs(b))))


def test_small_case_regenerates_bit_equal():
    """The extended-precision results of the stored inputs are bit-equal to the fixture (mpmath does not depend on the
    platform).  cond(K) comes from LAPACK and sklearn's results from the BLAS build: those are compared at a
    tolerance."""
    want = _load(MI.SMALL_CASE)
    got = MI.make_case(MI.SMALL_CASE, inputs=(want["X"], want["y"], want["xt"], want["group"]))
    assert set(got) == set(want)
    platform = {k for k in got if k.startswith("sk_")} | {"cond"}
    for k in sorted(set(got) - platform):
        assert np.array_equal(np.asarray(got[k]), want[k]), k
    for k in sorted(platform):
        np.testing.assert_allclose(got[k], want[k], rtol=1e-6, atol=1e-12, err_msg=k)


def test_every_case_has_a_fixture_and_its_inputs():
    """The builders reproduce each fixture's inputs: X exactly (uniform draws only), y and the candidates to a few ulp
    (they go through libm's exp, sin and sqrt, which may differ in the last bit between builds)."""
    for name, c in MI.CASES.items():
        r = _load(name)
        X, y, xt, group = MI.problem(c)
        assert np.array_equal(r["X"], X), name
        assert _close_ulps(r["y"], y) and _close_ulps(r["xt"], xt), name
        assert np.array_equal(r["group"], group), name
        assert r["L_packed"].size == c["n"] * (c["n"] + 1) // 2


def test_fixtures_span_the_intended_conditions():
    conds = {name: float(_load(name)["cond"]) for name in MI.CASES}
    assert min(conds.values()) < 1e6 and max(conds.values()) > 1e11
    assert sum(1e8 <= v for v in conds.values()) >= 6
    assert {c["kern"] for c in MI.CASES.values()} == {"m05", "m15", "m25", "rbf"}
    assert any(np.iterable(c["ls"]) and c.get("const") and c.get("white") for c in MI.CASES.values())
    assert {c["alpha"] for c in MI.CASES.values()} >= {1e-6, 1e-8, 1e-10}
    clustered = [c for c in MI.CASES.values() if c.get("cluster")]
    assert {c["d"] for c in clustered} >= {2, 3, 6, 17}
    assert {c["cluster"][1] for c in clustered} >= {1e-2, 1e-3, 1e-4}
    # N crosses the 64-row blocks and the 128-row padding (the append case fills its capacity on purpose)
    assert all(c["n"] % 64 for name, c in MI.CASES.items() if not name.startswith("a_"))
    assert any(c["n"] > 128 for c in MI.CASES.values())


@pytest.mark.parametrize("name", sorted(MI.CASES))
def test_fixture_is_self_consistent(name):
    """The stored truth agrees with itself in fp64: sigma^2 = var, the acquisitions follow from mu and sigma, and the
    variance stays below the prior; sklearn is close to it (its error is measured by the GPU tests)."""
    from oracle import gp_oracle as O

    r = _load(name)
    prior = r["prior"] * r["y_std"] ** 2
    # sigma is compared relatively on every row: no true variance is a vanishing residue (at training rows it is
    # about alpha * prior)
    assert np.all(r["var"] > 1e-12 * prior) and np.all(r["var"] <= prior * (1 + 1e-12))
    np.testing.assert_allclose(r["sd"] ** 2, r["var"], rtol=1e-14)
    y_max = float(np.max(r["y"]))
    for kind, code in (("ucb", O.ACQ_UCB), ("ei", O.ACQ_EI), ("poi", O.ACQ_POI)):
        ref = O.base_acq(code, r["mu"], r["sd"], kappa=MI.KAPPA, xi=MI.XI, y_max=y_max)
        np.testing.assert_allclose(r[f"acq_{kind}"], ref, rtol=1e-9, atol=1e-300, err_msg=kind)
    np.testing.assert_allclose(r["sk_mu"], r["mu"], rtol=1e-5, atol=1e-5 * r["y_std"])
    assert r["lml_grad"].shape == r["sk_lml_grad"].shape

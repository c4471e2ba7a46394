"""The double-double sample paths (oracle/dd.py: dd_cos_sin, Paths) and the production-size fixtures they build
(oracle/make_paths_big.py, tests/golden/pathbig_*.npz), without a GPU.

dd_cos_sin is checked against mpmath at 60 digits, the path pipeline against the 50-digit paths of the twelve
illext_* fixtures (bit-equal after rounding), the truth against the training-row identity, and the fixtures for
their inputs, draws, coverage, size and bit-equal regeneration."""
import os

import mpmath as mp
import numpy as np
import pytest

from oracle import dd
from oracle import make_illcond as MI
from oracle import make_illcond_ext as XE
from oracle import make_paths_big as PB


def _load(path):
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


def _stored(name):
    return _load(PB.fixture_path(name))


def test_dd_cos_sin_against_mpmath():
    """1e5 arguments: uniform on [-10, 10], Cauchy-tailed up to 1e7, next to multiples of pi/2 (the worst case of the
    reduction) and every fixture's largest |omega . xs + b|; each with a random low part.  Absolute error <= 1e-30."""
    rs = np.random.RandomState(11)
    n = 100_000
    k = rs.randint(-2 ** 22, 2 ** 22, size=n // 4)
    near = np.array([float(v * mp.pi / 2) for v in k])
    largest = []
    for name in PB.PROBLEMS:
        with np.load(PB.fixture_path(name)) as z:
            largest += [float(z[f"phase_{s}"]) for s in PB.SETS]
    hi = np.concatenate([rs.uniform(-10, 10, n // 4), np.clip(rs.standard_cauchy(n // 4) * 100, -1e7, 1e7),
                         near, np.nextafter(near, np.inf), largest, np.negative(largest)])
    lo = rs.uniform(-0.5, 0.5, len(hi)) * np.spacing(hi)
    mp.mp.dps = 60
    worst, arg = 0.0, None
    for h, l in zip(hi, lo):
        ch, cl, sh, sl = dd.dd_cos_sin(h, l)
        a = mp.mpf(h) + mp.mpf(l)
        e = float(max(abs(mp.mpf(ch) + mp.mpf(cl) - mp.cos(a)), abs(mp.mpf(sh) + mp.mpf(sl) - mp.sin(a))))
        if e > worst:
            worst, arg = e, h
    mp.mp.dps = 50
    print(f"\n{len(hi)} arguments, largest |a| {np.max(np.abs(hi)):.1e}: max abs error {worst:.1e} at {arg!r}")
    assert max(largest) > 1e3  # the Matern 1/2 draws' Cauchy tail reaches past the first few periods
    assert worst <= 1e-30


@pytest.mark.parametrize("name", sorted(MI.CASES))
def test_dd_paths_match_the_50_digit_fixtures(name):
    """dd.Paths on the inputs and draws of illext_<case> (q = 4, L = 512): values, gradients and V bit-equal to the
    50-digit truth after rounding to fp64."""
    c, r = MI.CASES[name], _load(XE.fixture_path(name))
    fit = dd.Fit(c, r["X"], r["y"])
    P = dd.Paths(fit, r["omega"], r["b"], r["w"], r["eps"])
    xs = dd.scaled(c, r["xt"])
    val = np.array([[float(v) for v in row] for row in P.values(xs)])
    grad = np.array([[[float(v) for v in g] for g in row] for row in P.grads(xs)])
    assert np.array_equal(val, r["path_val"])
    assert np.array_equal(grad, r["path_grad"])
    assert np.array_equal((P.V[0] + P.V[1]).T, r["path_v"])


@pytest.mark.parametrize("name", PB.PROBLEMS)
def test_training_row_identity(name):
    """f(X_i) = y_mean + s_y (y_n,i - eps_i - sigma_n^2 V_i) at every training-row candidate, unrounded, on every set
    (the feature term and the update term agree with each other).  Measured 6.7e-29 .. 1.5e-26, and 9.5e-23 on
    b_rbf_long, where alpha = 1e-8 lets |V| reach 1e8 and each term c k V_i carries its 1e-32 roundoff times that."""
    r = _stored(name)
    bar = 1e-21 if name == "b_rbf_long" else 1e-25
    for s in PB.SETS:
        assert float(r[f"ident_{s}"]) <= bar, (s, float(r[f"ident_{s}"]))


def test_training_row_identity_small_case():
    """The same identity computed here on the smallest illext case, so that train_identity itself is exercised."""
    name = MI.SMALL_CASE
    c, r = MI.CASES[name], _load(XE.fixture_path(name))
    fit = dd.Fit(c, r["X"], r["y"])
    P = dd.Paths(fit, r["omega"], r["b"], r["w"], r["eps"])
    vals = P.values(fit.Xs)
    worst = max(abs(vals[i][p] - P.train_identity(i, p)) / (abs(vals[i][p]) + fit.y_std)
                for i in range(fit.n) for p in range(len(vals[0])))
    print(f"\n{name}: {float(worst):.1e}")
    assert worst <= 1e-25


def test_draw_helper_equals_the_restatement():
    """paths.draw_path_inputs (what sample_paths draws) equals thompson_oracle.draws on every set of every problem."""
    import thompson_oracle as TO

    for name in PB.PROBLEMS:
        c = PB.AB.case(name)
        for s, (q, L) in PB.SETS.items():
            a = PB.draws(name, s, 50)
            b = TO.draws(np.random.RandomState(PB.seed(name, s)), q, L, c["d"], PB.NU[c["kern"]], 50,
                         c["alpha"] + (c.get("white") or 0.0))
            assert all(np.array_equal(u, v) for u, v in zip(a, b)), (name, s)


def test_fixtures_have_their_inputs_and_fit_the_repository(tmp_path):
    """The inputs rebuild to the stored digests (load() refuses others); seeds as documented; each fixture under 1 MB."""
    total = 0
    for name in PB.PROBLEMS:
        r = PB.load(name)
        assert list(r["seeds"]) == [PB.seed(name, s) for s in PB.SETS]
        size = os.path.getsize(PB.fixture_path(name))
        total += size
        assert size < 1_000_000, name
    print(f"\ntotal {total / 1e6:.2f} MB")
    bad = _stored(PB.SMALL)
    bad["xt_sha256"] = np.array("0" * 64)
    np.savez_compressed(tmp_path / "bad.npz", **bad)
    with pytest.raises(ValueError):
        PB.load(PB.SMALL, str(tmp_path / "bad.npz"))


def test_fixtures_cover_the_intended_cases():
    """Every problem; QT classes 1, 4 and 16 and q < QT; d in {5, 6, 16, 17, 32}; L ragged against 64 and 256; the
    q16 values on every candidate and every row class in the others' subset; gradients on the 64 grad rows."""
    ds = set()
    for name in PB.PROBLEMS:
        r = PB.load(name)
        ds.add(r["X"].shape[1])
        classes = set(np.unique(r["group"]))
        assert classes == set(range(len(MI.GROUP_NAMES)))
        assert set(np.unique(r["group"][r["subset"]])) == classes and len(r["subset"]) == PB.SUBSET
        for s, (q, L) in PB.SETS.items():
            rows = PB.rows_of(s, r["group"])
            assert r[f"val_{s}"].shape == (len(rows), q) and np.all(np.isfinite(r[f"val_{s}"]))
            assert r[f"grad_{s}"].shape == (64, r["X"].shape[1]) and r[f"ref_err_{s}"].shape == (len(rows),)
            assert np.all(r[f"bound_{s}"] >= np.max(np.abs(r[f"val_{s}"]), axis=0))
            assert r[f"train_eval_{s}"].shape == (np.sum(r["group"] == MI.G_TRAIN),)
        assert len(r["val_q16"]) == len(r["xt"])
    assert ds == {5, 6, 16, 17, 32}
    qs = {q for q, _ in PB.SETS.values()}
    assert {1, 4, 16} <= qs and any(1 < q < 16 and q not in (4,) for q in qs)
    assert any(L % 64 and L % 256 for _, L in PB.SETS.values())


def test_smallest_fixture_regenerates_bit_equal():
    """The truth of the stored inputs is bit-equal to the fixture (fixed-order reductions, no FMA); the referee's
    errors come from LAPACK and BLAS and are compared at a tolerance."""
    want = PB.load(PB.SMALL)
    got = PB.make_problem(PB.SMALL, inputs=(want["X"], want["y"], want["xt"], want["group"]))
    stored = _stored(PB.SMALL)
    assert set(got) == set(stored)
    for k in sorted(got):
        if k.startswith("ref_"):  # the largest error, within a factor 10
            a, b = float(np.max(got[k])), float(np.max(stored[k]))
            assert b / 10 <= a <= 10 * b, (k, a, b)
        else:
            assert np.array_equal(np.asarray(got[k]), stored[k]), k

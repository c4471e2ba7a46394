"""The prune-matrix fixtures (oracle/make_prune_matrix.py, tests/golden/prunemx_*.npz) without a GPU:
  * every fixture rebuilds its X from the seeds and matches its digest, and stays under 1 MB; the stored top-k and gaps
    are those of the stored truth, ties to the lowest index;
  * on the problems shared with the illbig_* fixtures, the double-double mu and sigma^2 of the base candidates equal the
    stored truths there bit for bit, and extra candidates that copy another have the same truth;
  * tests/test_prune_cpu.py's numpy restatement of prune_bound_key (the single-point bound: max |k*_i| from sklearn's
    covariance), taken at the truth's mean rounded to fp64 and moved up by 4 ulps of |mu| + |y_max| + |xi| (the rounding
    of the data-unit mean and of a = mu - y_max - xi, which the device's value carries as well: at a 1e6 offset it
    exceeds the 1e-9 relative margin of EI where y_max lies below every mu), never lies above the truth's closure value
    -acq, for every prunable kind and parameter point, outside the never-prune rule;
  * o_offset_d2 regenerates bit for bit.
"""
import os

import numpy as np
import pytest

from oracle import make_illcond as MI
from oracle import make_illcond_big as MB
from oracle import make_prune_matrix as PM
from test_prune_cpu import bound_value, never_prune


@pytest.fixture(scope="module", params=PM.PROBLEMS)
def fx(request):
    return request.param, PM.load(request.param)


def test_fixture_shapes_and_order(fx):
    name, r = fx
    assert os.path.getsize(PM.fixture_path(name)) < 1 << 20
    m = len(r["xt"])
    assert m * 8 >= 32 * 128 and r["xt"].shape[1] == PM.case(name)["d"]
    assert np.all(np.isfinite(r["xt"])) and not np.all(np.isfinite(r["bad_rows"]), axis=1).any()
    assert np.sum(r["src"] >= 0) == PM.SHARED and np.array_equal(r["src"][r["src"] >= 0], np.arange(PM.SHARED))
    far = np.min(np.abs(r["xt"]), axis=1) >= 1e3
    assert far.sum() >= 12 and np.allclose(r["var_hi"][far], r["prior"] * np.std(r["y"]) ** 2, rtol=1e-9, atol=0)
    for kind in PM.KINDS:
        t = r[kind]
        assert t.shape == ((len(PM.KAPPAS) if kind == "ucb" else 9), m) and np.all(np.isfinite(t))
        order = np.argsort(-t, axis=1, kind="stable")[:, :PM.TOPK]
        assert np.array_equal(order, r[f"top_{kind}"])
        assert np.all(r[f"gap_{kind}"] >= 0)
    # the exact copies: the same rows, the same truth
    d = r["dup_of"]
    assert (d >= 0).sum() > 8
    assert np.array_equal(r["xt"][d >= 0], r["xt"][d[d >= 0]])
    assert np.array_equal(r["mu_hi"][d >= 0], r["mu_hi"][d[d >= 0]])
    # y_max below every mu: PoI is 1 at every candidate (ties broken by the lowest index)
    assert np.all(r["poi"][:3] == 1.0) and np.all(r["y_max"][:3] < np.min(r["mu_hi"]))


@pytest.mark.parametrize("name", PM.SHARED_PROBLEMS)
def test_shared_truth_equals_illbig(name):
    r, b = PM.load(name), MB.load(name)
    s = r["src"] >= 0
    assert np.array_equal(r["xt"][s], b["xt"][:PM.SHARED])
    assert np.array_equal(r["mu_hi"][s], b["mu"][:PM.SHARED])
    assert np.array_equal(r["var_hi"][s], b["var"][:PM.SHARED])


def test_bound_below_truth(fx):
    name, r = fx
    from sklearn.gaussian_process.kernels import WhiteKernel

    c = PM.case(name)
    kern = MI.sk_kernel(c)
    if isinstance(kern.k2 if hasattr(kern, "k2") else None, WhiteKernel):
        kern = kern.k1  # the noise term adds nothing off the diagonal
    x = r["xt"]
    kmax = np.max(np.abs(kern(x, r["X"])), axis=1)
    const, white = float(c.get("const") or 1.0), float(c.get("white") or 0.0)
    prior, kdiag = const + white, const + white + c["alpha"]
    y = r["y"]
    y_std = float(np.std(y))
    mu = r["mu_hi"]
    worst = {}
    for kind in PM.KINDS:
        params = r["kappa"] if kind == "ucb" else zip(r["y_max"], r["xi"])
        for j, p in enumerate(params):
            kappa, (y_max, xi) = (p, (0.0, 0.0)) if kind == "ucb" else (0.0, p)
            dmu = 4 * np.finfo(float).eps * (np.abs(mu) + abs(y_max) + abs(xi))
            lb = bound_value(kind, mu + dmu, kmax, prior, kdiag, y_std, y_max, kappa, xi)
            keep = never_prune(kind, mu, lb, y_max, xi)
            exact = -r[kind][j]
            bad = ~keep & (lb > exact)
            assert not bad.any(), (kind, j, np.flatnonzero(bad)[:5], (lb - exact)[bad][:5])
            worst[kind, j] = int(np.sum(~keep & (lb <= exact)))
    print(f"\n{name}: candidates bounded per (kind, point) {min(worst.values())} .. {max(worst.values())}")


def test_regenerates_bit_for_bit(tmp_path):
    name = "o_offset_d2"
    PM.main(["--only", name, "--out", str(tmp_path)])
    with np.load(PM.fixture_path(name)) as a, np.load(tmp_path / f"prunemx_{name}.npz") as b:
        assert sorted(a.files) == sorted(b.files)
        for k in a.files:
            assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), k

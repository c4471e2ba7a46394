"""The refine stages of selection-only pruning (DESIGN.md 4.9), restated in numpy.

predict_refine_kernel (csrc/predict16.cuh) bounds the variance by the leading row blocks of V = L^-1 k*:
    r_b = sum of V_i^2 over the first b row blocks <= k*^T K^-1 k*   (the remaining terms are squares),
    var_ub = max(0, min(prior, prior - r_b + eps * prior)),
and keys the candidate exactly as the single-point bound does.  predict_units_kernel evaluates the survivors in units
of consecutive row blocks; every unit stores its per-row-block, per-(row slab, lane group) sums of squares and the
tile's finisher adds them in the order of the unsplit phase B.  Here:
  (a) the refined bound lies below the exact closure value for b = 1, 2, 4 on well- and ill-conditioned (clustered)
      training sets, training copies and near-duplicates included;
  (b) the finisher's sum equals the unsplit sum bit for bit for every cut into groups, the cuts tile the row blocks,
      and a running sum per group (what the units must not store) does not reproduce it.
"""
import numpy as np
import pytest
from scipy.linalg import cholesky, solve_triangular
from sklearn.gaussian_process import GaussianProcessRegressor

from test_prune_cpu import ABS_MARGIN, KERNELS, REL_MARGIN, VAR_EPS, exact_value, never_prune

ROWS = 16  # rows per row block here (PBM = 128 on the device)


def refined_bound(kind, mu, r, prior, y_std, y_max, kappa, xi):
    """v_lb per candidate from r <= k*^T K^-1 k* (normalised units): prune_var_ub + prune_bound_key."""
    from scipy.stats import norm

    var_ub = np.maximum(0.0, np.minimum(prior, prior - r + VAR_EPS * prior))
    sd = np.sqrt(var_ub * y_std * y_std)
    a = mu - y_max - xi
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == "ucb":
            base = np.maximum(mu, mu + kappa * sd)
            scale = np.abs(mu) + np.abs(kappa * sd)
        elif kind == "ei":
            z = a / sd
            base = a * norm.cdf(z) + sd * norm.pdf(z)
            scale = np.abs(base)
        else:
            base = np.where(a < 0, norm.cdf(a / sd), 1.0)
            scale = np.abs(base)
    return -base - (REL_MARGIN * scale + ABS_MARGIN)


def training_set(layout, rs, n, d):
    if layout == "uniform":
        return rs.uniform(size=(n, d))
    # clustered: a few centres with points 1e-4 apart, the ill-conditioned sets of tests/test_gpu_illcond.py in small
    centres = rs.uniform(size=(n // 10, d))
    return centres[rs.randint(len(centres), size=n)] + 1e-4 * rs.randn(n, d)


@pytest.mark.parametrize("layout", ["uniform", "clustered"])
@pytest.mark.parametrize("kname", sorted(KERNELS))
@pytest.mark.parametrize("kind,kappa", [("ei", 0.0), ("poi", 0.0), ("ucb", 2.576), ("ucb", -1.0)])
def test_refined_bound_below_exact(layout, kname, kind, kappa):
    rs = np.random.RandomState(5)
    n, d, alpha, xi = 120, 4, 1e-6, 0.01
    X = training_set(layout, rs, n, d)
    y = np.sin(3 * X.sum(1)) + 0.05 * rs.randn(n)
    gp = GaussianProcessRegressor(kernel=KERNELS[kname](d), alpha=alpha, normalize_y=True, optimizer=None).fit(X, y)
    x = np.vstack([rs.uniform(size=(3000, d)), X[:20], X[-20:], X[:20] + 1e-7, X[:20] + 1e-3])
    mu, sd = gp.predict(x, return_std=True)
    exact = exact_value(kind, mu, sd, y.max(), kappa, xi)
    K = gp.kernel_(X) + alpha * np.eye(n)
    V = solve_triangular(cholesky(K, lower=True), gp.kernel_(X, x), lower=True)  # [n][candidates]
    prior = gp.kernel_.diag(x[:1])[0]
    prev = None
    for b in (1, 2, 4):
        r = np.sum(V[:b * ROWS] ** 2, axis=0)
        lb = refined_bound(kind, mu, r, prior, gp._y_train_std, y.max(), kappa, xi)
        keep = never_prune(kind, mu, lb, y.max(), xi)
        assert np.all(lb[~keep] <= exact[~keep]), (b, (lb - exact)[~keep].max())
        if prev is not None and kind != "poi":  # more rows never loosen the variance bound
            assert np.all(r >= prev)
        prev = r


def unit_cut(nb, groups, j):
    """First row block of group j: unit_cut of predict16.cuh."""
    if j >= groups:
        return nb
    total = nb * (nb + 1) // 2
    ib = 0
    while ib < nb and ib * (ib + 1) // 2 * groups < total * j:
        ib += 1
    return ib


def tree(v):
    """The xor-shuffle tree over the 8 lane groups (4, 8, 16), then the four row slabs in order."""
    w = ((v[:, 0] + v[:, 1]) + (v[:, 2] + v[:, 3])) + ((v[:, 4] + v[:, 5]) + (v[:, 6] + v[:, 7]))
    return ((w[0] + w[1]) + w[2]) + w[3]


def unsplit(s):
    """predict16_phase_b: csq += s(ib) per (row slab, lane group), ib = 0, 1, ..."""
    csq = np.zeros(s.shape[1:])
    for ib in range(s.shape[0]):
        csq = csq + s[ib]
    return tree(csq)


@pytest.mark.parametrize("nb", [8, 32, 64])
@pytest.mark.parametrize("groups", [1, 2, 3, 4, 16, 32])
def test_split_sum_is_bit_equal(nb, groups):
    rs = np.random.RandomState(nb * 100 + groups)
    s = rs.uniform(size=(nb, 4, 8, 128)) * 10.0 ** rs.randint(-12, 3, size=(nb, 4, 8, 128))
    cuts = [unit_cut(nb, groups, j) for j in range(groups + 1)]
    assert cuts[0] == 0 and cuts[-1] == nb and all(a <= b for a, b in zip(cuts, cuts[1:]))
    part = np.full_like(s, np.nan)  # what the units store: s(ib) itself, each row block by exactly one unit
    for a, b in zip(cuts, cuts[1:]):
        assert np.all(np.isnan(part[a:b]))
        part[a:b] = s[a:b]
    assert not np.isnan(part).any()
    ref = unsplit(s)
    assert np.array_equal(unsplit(part).view(np.uint64), ref.view(np.uint64))
    if groups in (3, 4) and nb >= 32:  # running sums per unit, added afterwards, are a different rounding
        run = np.zeros(s.shape[1:])
        for a, b in zip(cuts, cuts[1:]):
            g = np.zeros(s.shape[1:])
            for ib in range(a, b):
                g = g + s[ib]
            run = run + g
        assert not np.array_equal(tree(run).view(np.uint64), ref.view(np.uint64))


def test_cuts_balance_k_tiles():
    """Row block ib costs ib + 1 k-tile groups; no group of the default split is far above the mean."""
    nb, groups = 32, 16
    cuts = [unit_cut(nb, groups, j) for j in range(groups + 1)]
    cost = [sum(ib + 1 for ib in range(a, b)) for a, b in zip(cuts, cuts[1:])]
    assert sum(cost) == nb * (nb + 1) // 2
    assert max(cost) <= 2 * sum(cost) / groups

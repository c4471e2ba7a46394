"""The refine levels of selection-only pruning (DESIGN.md 4.9), restated in numpy.

The refine stage stores each survivor's running sums over row blocks [0, b) per (row slab, lane group), before the
xor tree; a level carries them on over [b, b') and keys the survivor from their tree sum; the final stage carries them
on to the last row block.  Here:
  (a) a prefix carried across any cut of the row blocks into levels reproduces the unsplit sum bit for bit, and a
      running sum per level, added afterwards, does not;
  (b) every level's key is a lower bound of the exact closure value, on the well- and ill-conditioned sets of
      tests/test_prune_refine_cpu.py;
  (c) the schedule: unit_cut with a start block tiles [b0, nb) with balanced k-tile counts, the one level ends at 2b,
      and the final rounds (8, then the rest) cover the survivor tiles, at most one tile per SM each (the rounds'
      stop rule is tests/test_prune_rounds_cpu.py's).
"""
import numpy as np
import pytest
from scipy.linalg import cholesky, solve_triangular
from sklearn.gaussian_process import GaussianProcessRegressor

from test_prune_cpu import KERNELS, exact_value, never_prune
from test_prune_refine_cpu import ROWS, refined_bound, training_set, tree, unsplit

K_REFINE_MAX_TILES = 128


def unit_cut(b0, nb, groups, j):
    """First row block of group j over [b0, nb): unit_cut of predict16.cuh."""
    if j >= groups:
        return nb
    base = b0 * (b0 + 1) // 2
    total = nb * (nb + 1) // 2 - base
    ib = b0
    while ib < nb and (ib * (ib + 1) // 2 - base) * groups < total * j:
        ib += 1
    return ib


def refine_blocks(nb, blocks=4):
    """prune_refine_blocks of b200bo.cu: B200BO_PRUNE_REFINE_BLOCKS (default 4), at least 1, clamped to nb / 8"""
    return min(max(blocks, 1), nb // 8)


def level_ends(b, nb):
    """the level of prune_refine_stages in b200bo.cu: one, to 2b"""
    return [2 * b]


def final_round_tiles(r, t0, grid):
    """final_round_tiles of predict16.cuh: 8, then the rest, at most grid each"""
    return min(8 if r == 0 else K_REFINE_MAX_TILES - t0, grid)


def carried(s, cuts):
    """The refine stage's prefix over [0, cuts[0]), carried through each level [cuts[i], cuts[i+1])."""
    pre = np.zeros(s.shape[1:])
    for ib in range(cuts[0]):
        pre = pre + s[ib]
    for a, b in zip(cuts, cuts[1:]):
        for ib in range(a, b):
            pre = pre + s[ib]
    return tree(pre)


@pytest.mark.parametrize("nb", [8, 32, 64])
def test_carried_prefix_is_bit_equal(nb):
    rs = np.random.RandomState(nb)
    s = rs.uniform(size=(nb, 4, 8, 128)) * 10.0 ** rs.randint(-12, 3, size=(nb, 4, 8, 128))
    ref = unsplit(s).view(np.uint64)
    for b in range(1, nb // 8 + 1):
        for cuts in ([b, nb], [b, 2 * b, nb], [b, 2 * b, 4 * b, nb], [b] + sorted(set(rs.randint(b, nb, 3))) + [nb]):
            assert np.array_equal(carried(s, cuts).view(np.uint64), ref), cuts
    # a running sum per level, added to the prefix afterwards, is another rounding
    b = max(1, nb // 8)
    pre = np.zeros(s.shape[1:])
    for ib in range(b):
        pre = pre + s[ib]
    lev = np.zeros(s.shape[1:])
    for ib in range(b, nb):
        lev = lev + s[ib]
    assert not np.array_equal(tree(pre + lev).view(np.uint64), ref)


@pytest.mark.parametrize("layout", ["uniform", "clustered"])
@pytest.mark.parametrize("kname", sorted(KERNELS))
@pytest.mark.parametrize("kind,kappa", [("ei", 0.0), ("poi", 0.0), ("ucb", 2.576), ("ucb", -1.0)])
def test_level_keys_below_exact(layout, kname, kind, kappa):
    rs = np.random.RandomState(7)
    n, d, alpha, xi = 128, 4, 1e-6, 0.01
    X = training_set(layout, rs, n, d)
    y = np.sin(3 * X.sum(1)) + 0.05 * rs.randn(n)
    gp = GaussianProcessRegressor(kernel=KERNELS[kname](d), alpha=alpha, normalize_y=True, optimizer=None).fit(X, y)
    x = np.vstack([rs.uniform(size=(3000, d)), X[:20], X[-20:], X[:20] + 1e-7, X[:20] + 1e-3])
    mu, sd = gp.predict(x, return_std=True)
    exact = exact_value(kind, mu, sd, y.max(), kappa, xi)
    K = gp.kernel_(X) + alpha * np.eye(n)
    V = solve_triangular(cholesky(K, lower=True), gp.kernel_(X, x), lower=True)
    prior = gp.kernel_.diag(x[:1])[0]
    nb = n // ROWS
    for b in (1, 2):
        for end in [b] + level_ends(b, nb):  # the refine stage's key, then each level's
            r = np.sum(V[:end * ROWS] ** 2, axis=0)
            lb = refined_bound(kind, mu, r, prior, gp._y_train_std, y.max(), kappa, xi)
            keep = never_prune(kind, mu, lb, y.max(), xi)
            assert np.all(lb[~keep] <= exact[~keep]), (b, end, (lb - exact)[~keep].max())


@pytest.mark.parametrize("nb", [8, 32, 64])
@pytest.mark.parametrize("groups", [1, 2, 3, 4, 16, 32])
def test_cuts_with_start_block(nb, groups):
    for b0 in range(0, nb // 2 + 1):
        cuts = [unit_cut(b0, nb, groups, j) for j in range(groups + 1)]
        assert cuts[0] == b0 and cuts[-1] == nb and all(a <= b for a, b in zip(cuts, cuts[1:])), (b0, cuts)
        cost = [sum(ib + 1 for ib in range(a, b)) for a, b in zip(cuts, cuts[1:])]
        # no group exceeds the mean by more than one row block's k-tiles
        assert max(cost) <= sum(cost) / groups + nb, (b0, cost)
    # b0 = 0 is the cut of the lead stage
    for j in range(groups + 1):
        total = nb * (nb + 1) // 2
        ib = 0
        while ib < nb and ib * (ib + 1) // 2 * groups < total * j:
            ib += 1
        assert unit_cut(0, nb, groups, j) == (nb if j >= groups else ib)


@pytest.mark.parametrize("nb", [8, 16, 32, 64, 128])
def test_level_schedule(nb):
    # the default and the B200BO_PRUNE_REFINE_BLOCKS values of tests/test_gpu_prune_matrix.py, clamped
    for blocks in (4, 1, 64):
        b = refine_blocks(nb, blocks)
        ends = level_ends(b, nb)
        assert ends == [2 * b] and b < ends[0] < nb, (blocks, b, ends)


# SM counts: below, at and around the first round of 8 and the 120 tiles after it, the H100 PCIe (114) and SXM (132)
@pytest.mark.parametrize("grid", [1, 7, 8, 9, 64, 114, 119, 120, 121, 127, 128, 132])
def test_round_schedule(grid):
    """The final stage's rounds as final_rounds_kernel (predict16.cuh) loops over them: t0 from 0 while t0 <
    kRefineMaxTiles, t1 = t0 + final_round_tiles(r, t0, gridDim.x), with no cap on the round count (grid 1: 128 rounds
    of one tile)."""
    t0, sizes = 0, []
    while t0 < K_REFINE_MAX_TILES:
        t = final_round_tiles(len(sizes), t0, grid)
        assert 0 < t <= grid
        sizes.append(t)
        t0 += t
    assert t0 == K_REFINE_MAX_TILES
    assert sizes[0] == min(8, grid)
    if grid >= K_REFINE_MAX_TILES - 8:
        assert sizes == [8, 120]
    else:
        assert sizes[1:-1] == [grid] * (len(sizes) - 2) and 0 < sizes[-1] <= grid


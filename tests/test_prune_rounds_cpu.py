"""The merged k-th key, the final rounds and the shared K* of pruning's refine stages (DESIGN.md 4.9), restated in
numpy.

  (a) merge_kth_kernel: the k-th smallest value over the union of the per-CTA lists is >= the final k-th value (it is
      the k-th of values already produced) and <= the least k-th value of any single list (the key before it);
  (b) the stages: lead tiles in bound order, the refine stage against the merged key, the survivors sorted by
      max(single-point key, refined key) and evaluated in rounds of 8 tiles and then the rest (final_round_tiles), a
      round skipping the tiles whose first key is above the key merged before it, return the records of a full
      argsort, on well-conditioned, clustered and ill-conditioned (tests/golden) training sets;
  (c) unit_mu_from_ks: mu = K* alpha_ recomputed from the stored K* by one fma chain per (part, column), chunks
      ascending and rows part * 16 .. part * 16 + 15 of each, is phase A's mu bit for bit on IEEE doubles, and a
      chain in plain row order is not.
"""
import os
from fractions import Fraction

import numpy as np
import pytest
from scipy.linalg import cholesky, solve_triangular
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import Matern

from test_prune_cpu import KERNELS, exact_value, never_prune
from test_prune_refine_cpu import refined_bound

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TILE = 8  # candidates per tile here (PBN = 128 on the device)
LEAD = 8  # kLeadTiles
MAX_TILES = 24  # kRefineMaxTiles, scaled down with the tile
FIRST_ROUND = 8  # tiles of the first final round, then the rest


def kth(values, k):
    """the k-th smallest of the values, or inf when there are fewer (the word is left unchanged)"""
    v = np.sort(np.asarray(values, dtype=np.float64))
    return v[k - 1] if len(v) >= k else np.inf


def stages(lb1, lbr, value, k):
    """(evaluated candidates, merged key after the lead, per-list key after the lead, keys before each round):
    the lead, refine and final stages over candidates keyed by lb1 (single point) and lbr (refined)."""
    m = len(value)
    perm = np.argsort(lb1, kind="stable")
    ntiles = -(-m // TILE)
    tiles = [perm[t * TILE:(t + 1) * TILE] for t in range(ntiles)]
    lead = tiles[:LEAD]
    # one CTA finishes each lead tile: its list holds that tile's values only
    old_key = min(kth(value[t], k) for t in lead)
    evaluated = [c for t in lead for c in t]
    key = min(old_key, kth(value[evaluated], k))
    merged = key
    surv = []
    for t in tiles[LEAD:]:
        if lb1[t[0]] > key or len(surv) > MAX_TILES * TILE:
            break
        surv += [c for c in t if lbr[c] <= key and lb1[c] <= key]
    if len(surv) > MAX_TILES * TILE:  # the tile kernel takes over in bound order
        for t in tiles[LEAD:]:
            if lb1[t[0]] > key:
                break
            evaluated += list(t)
            key = min(key, kth(value[evaluated], k))
        return np.array(evaluated), merged, old_key, []
    skey = np.maximum(lb1, lbr)
    surv = sorted(surv, key=lambda c: skey[c])
    stiles = [surv[t * TILE:(t + 1) * TILE] for t in range(-(-len(surv) // TILE))]
    t0, r, before = 0, 0, []
    while t0 < MAX_TILES:
        t1 = t0 + (FIRST_ROUND if r == 0 else MAX_TILES - t0)
        before.append(key)
        for t in stiles[t0:t1]:
            if skey[t[0]] > key:  # sorted: every later tile of the round is skipped too
                break
            evaluated += t
        key = min(key, kth(value[evaluated], k))
        t0, r = t1, r + 1
    return np.array(evaluated), merged, old_key, before


def records(value, idx, k):
    """argmin (first NaN, else the least value, ties to the lowest index) and the top-k in (value, index) order"""
    order = sorted(zip(value, idx), key=lambda p: (np.isnan(p[0]), p[0], p[1]))
    nan = [i for v, i in zip(value, idx) if np.isnan(v)]
    return (min(nan) if nan else order[0][1]), [i for _, i in order[:k]]


def problem(layout, rs, d=3):
    if layout == "golden":
        z = np.load(os.path.join(GOLDEN, "illcond_c_m25_d3.npz"))
        X, y = z["X"], z["y"]
        return X, y, np.vstack([z["xt"], rs.uniform(X.min(0), X.max(0), size=(2500, X.shape[1]))])
    n = 120
    if layout == "uniform":
        X = rs.uniform(size=(n, d))
    else:
        centres = rs.uniform(size=(n // 10, d))
        X = centres[rs.randint(len(centres), size=n)] + 1e-4 * rs.randn(n, d)
    y = np.sin(3 * X.sum(1)) + 0.05 * rs.randn(n)
    return X, y, np.vstack([rs.uniform(size=(2500, d)), X[:20], X[:20] + 1e-7])


@pytest.mark.parametrize("layout", ["uniform", "clustered", "golden"])
@pytest.mark.parametrize("kname", sorted(KERNELS))
@pytest.mark.parametrize("kind,kappa", [("ei", 0.0), ("poi", 0.0), ("ucb", 2.576)])
@pytest.mark.parametrize("k", [1, 10, 64])
def test_rounds_return_the_records(layout, kname, kind, kappa, k):
    rs = np.random.RandomState(17)
    X, y, x = problem(layout, rs)
    n, d, alpha, xi = len(X), X.shape[1], 1e-6, 0.01
    gp = GaussianProcessRegressor(kernel=KERNELS[kname](d), alpha=alpha, normalize_y=True, optimizer=None).fit(X, y)
    mu, sd = gp.predict(x, return_std=True)
    value = exact_value(kind, mu, sd, y.max(), kappa, xi)  # the closure value -acq, smaller is better
    K = gp.kernel_(X) + alpha * np.eye(n)
    Ks = gp.kernel_(X, x)
    V = solve_triangular(cholesky(K, lower=True), Ks, lower=True)
    prior = gp.kernel_.diag(x[:1])[0]
    r1 = np.max(Ks ** 2 / np.diag(K)[:, None], axis=0)  # the single-point term
    rb = np.sum(V[:16] ** 2, axis=0)  # the leading rows of L^-1
    lb1 = refined_bound(kind, mu, r1, prior, gp._y_train_std, y.max(), kappa, xi)
    lbr = refined_bound(kind, mu, rb, prior, gp._y_train_std, y.max(), kappa, xi)
    for lb in (lb1, lbr):
        keep = never_prune(kind, mu, lb, y.max(), xi)
        lb[keep] = -np.inf
        assert np.all(lb <= value)
    ev, merged, old_key, before = stages(lb1, lbr, value, k)
    assert len(set(ev.tolist())) == len(ev)
    final = kth(value, k)
    assert final <= merged <= old_key
    assert all(a >= b for a, b in zip(before, before[1:])) and all(b >= final for b in before)
    idx = np.arange(len(x))
    assert records(value[ev], idx[ev], k) == records(value, idx, k), (len(ev), len(x))


def fma(a, b, c):
    """IEEE fma of doubles: the exact a * b + c, rounded once"""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def phase_a_mu(ks, al, parts=4, chunk=64, r=8):
    """phase_a_impl's mu chain: per part, chunks ascending, rows part * rows .. in steps of R = 8"""
    rows = chunk // parts
    out = []
    for p in range(parts):
        acc = 0.0
        for ch in range(len(al) // chunk):
            for r0 in range(p * rows, (p + 1) * rows, r):
                for q in range(r):
                    acc = fma(al[ch * chunk + r0 + q], ks[ch * chunk + r0 + q], acc)
        out.append(acc)
    return out


def unit_mu(ks, al, parts=4, chunk=64):
    """unit_mu_from_ks: per part, n0 = part * rows, step chunk, rows n0 .. n0 + rows - 1"""
    rows = chunk // parts
    out = []
    for p in range(parts):
        acc = 0.0
        for n0 in range(p * rows, len(al), chunk):
            for q in range(rows):
                acc = fma(al[n0 + q], ks[n0 + q], acc)
        out.append(acc)
    return out


@pytest.mark.parametrize("fixture", ["illcond_c_m25_d3", "illbig_b_m25_c3"])
def test_mu_from_stored_ks_is_bit_equal(fixture):
    z = np.load(os.path.join(GOLDEN, fixture + ".npz"))
    al = np.asarray(z["alpha_"], dtype=np.float64)
    npad = -(-len(al) // 128) * 128
    al = np.concatenate([al, np.zeros(npad - len(al))])[:512]  # padded rows have alpha_ 0 and K* 0
    X = z["X"] if "X" in z.files else np.random.RandomState(3).uniform(size=(len(z["alpha_"]), 16))
    xt = z["xt"] if "xt" in z.files else z["xt_head"]
    kern = Matern(nu=2.5, length_scale=0.7)
    for c in range(4):
        ks = np.zeros(len(al))
        nreal = min(len(X), len(al))
        ks[:nreal] = kern(xt[c:c + 1], X[:nreal])[0]
        a = phase_a_mu(ks, al)
        b = unit_mu(ks, al)
        assert np.array_equal(np.array(a).view(np.uint64), np.array(b).view(np.uint64))
    # the order matters: one chain over the rows in plain order is another rounding on these alpha_
    rs = np.random.RandomState(1)
    al2 = rs.randn(256) * 10.0 ** rs.randint(-3, 9, size=256)
    ks2 = rs.uniform(size=256)
    plain = 0.0
    for i in range(256):
        plain = fma(al2[i], ks2[i], plain)
    parts = unit_mu(ks2, al2)
    assert phase_a_mu(ks2, al2) == parts
    assert plain != ((parts[0] + parts[1]) + parts[2]) + parts[3]

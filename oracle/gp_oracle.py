"""CPU oracle for the GP-surrogate + acquisition hot path.  TEST INFRASTRUCTURE ONLY.

This module is a numpy/scipy *restatement* of the arithmetic the reference
(bayesian-optimization/BayesianOptimization v3.3.0) reaches through scikit-learn 1.9.0 /
SciPy 1.18.1 on the path  suggest() -> gp.fit -> gp.predict(return_std) -> base_acq -> argmin.
It is the checker the CUDA path is compared with; it is never the product.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may import it.

Pinning: the restatement is checked (tests/test_oracle_golden.py) against
  * fixtures in tests/golden/*.npz produced by ``oracle/make_golden.py`` from the UNMODIFIED
    reference (``R/bayes_opt``) driving the live sklearn/scipy stack, and
  * the live ``sklearn.gaussian_process.GaussianProcessRegressor`` (a dependency of the
    reference that is installed in this image and on the GPU machine).
The reference's own tests hold no golden vectors for K, L, alpha, mu, sigma or acquisition
values (SURVEY.md section 8c) - the live computation is the oracle of record.

Citations:  R/ = R/,  SK/ = site-packages/sklearn/,  SP/ = site-packages/scipy/.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
from scipy.linalg import cho_solve, cholesky, solve_triangular
from scipy.spatial.distance import cdist, pdist, squareform
from scipy.special import ndtr

KIND_MATERN = 0
KIND_RBF = 1

ACQ_UCB = 0
ACQ_EI = 1
ACQ_POI = 2

_SQRT2PI = math.sqrt(2.0 * math.pi)


# --------------------------------------------------------------------------------------
# kernels  (SK/gaussian_process/kernels.py:1685-1786 Matern.__call__, :1530-1587 RBF.__call__)
# --------------------------------------------------------------------------------------
def _matern_from_dists(dists: np.ndarray, nu: float) -> np.ndarray:
    """SK/gaussian_process/kernels.py:1722-1731."""
    if nu == 0.5:
        return np.exp(-dists)
    if nu == 1.5:
        K = dists * math.sqrt(3)
        return (1.0 + K) * np.exp(-K)
    if nu == 2.5:
        K = dists * math.sqrt(5)
        return (1.0 + K + K**2 / 3.0) * np.exp(-K)
    if nu == np.inf:
        return np.exp(-(dists**2) / 2.0)
    raise NotImplementedError("general-nu Matern is outside the hot path")


def kernel_cross(Xa, Xb, *, kind=KIND_MATERN, nu=2.5, length_scale=1.0, const=1.0):
    """k(Xa, Xb): direct-difference distances via cdist, as sklearn does
    (SK/gaussian_process/kernels.py:1720, :1552-1553).  ``const`` is an optional
    ConstantKernel factor (SK/gaussian_process/kernels.py:1222-1260, Product :857)."""
    Xa = np.atleast_2d(Xa)
    Xb = np.atleast_2d(Xb)
    ls = np.asarray(length_scale, dtype=float)
    if kind == KIND_RBF:
        d2 = cdist(Xa / ls, Xb / ls, metric="sqeuclidean")
        K = np.exp(-0.5 * d2)
    else:
        d = cdist(Xa / ls, Xb / ls, metric="euclidean")
        K = _matern_from_dists(d, nu)
    return const * K if const != 1.0 else K


def kernel_train(X, *, kind=KIND_MATERN, nu=2.5, length_scale=1.0, const=1.0, eval_gradient=False):
    """k(X, X) with unit diagonal; optional gradient wrt log(length_scale) (isotropic) or
    each log(length_scale_j) (anisotropic).  SK/gaussian_process/kernels.py:1716,1740-1786
    (Matern) and :1548-1573 (RBF).  Returns K or (K, dK[n,n,p])."""
    X = np.atleast_2d(X)
    ls = np.asarray(length_scale, dtype=float)
    aniso = ls.ndim > 0 and ls.size > 1
    if kind == KIND_RBF:
        d2 = pdist(X / ls, metric="sqeuclidean")
        K = squareform(np.exp(-0.5 * d2))
        np.fill_diagonal(K, 1)
        if eval_gradient:
            if not aniso:
                G = (K * squareform(d2))[:, :, None]
            else:
                G = (X[:, None, :] - X[None, :, :]) ** 2 / (ls**2)
                G = G * K[..., None]
    else:
        dists = pdist(X / ls, metric="euclidean")
        K = squareform(_matern_from_dists(dists, nu))
        np.fill_diagonal(K, 1)
        if eval_gradient:
            if aniso:
                D = (X[:, None, :] - X[None, :, :]) ** 2 / (ls**2)
            else:
                D = squareform(dists**2)[:, :, None]
            if nu == 0.5:
                den = np.sqrt(D.sum(axis=2))[:, :, None]
                div = np.zeros_like(D)
                np.divide(D, den, out=div, where=den != 0)
                G = K[..., None] * div
            elif nu == 1.5:
                G = 3 * D * np.exp(-np.sqrt(3 * D.sum(-1)))[..., None]
            elif nu == 2.5:
                tmp = np.sqrt(5 * D.sum(-1))[..., None]
                G = 5.0 / 3.0 * D * (tmp + 1) * np.exp(-tmp)
            elif nu == np.inf:
                G = D * K[..., None]
            else:
                raise NotImplementedError
            if not aniso:
                G = G.sum(-1)[:, :, None]
    if const != 1.0:
        # Product(ConstantKernel, k): K = c*k ; d/dlog(c) = c*k ; d/dlog(l) = c*dk
        if eval_gradient:
            G = np.concatenate([(const * K)[:, :, None], const * G], axis=2)
        K = const * K
    return (K, G) if eval_gradient else K


# --------------------------------------------------------------------------------------
# GP state, fit at fixed theta, LML, predict  (SK/gaussian_process/_gpr.py)
# --------------------------------------------------------------------------------------
@dataclass
class GPState:
    X: np.ndarray
    y_norm: np.ndarray
    y_mean: float
    y_std: float
    L: np.ndarray
    alpha_: np.ndarray
    kind: int = KIND_MATERN
    nu: float = 2.5
    length_scale: object = 1.0
    const: float = 1.0
    alpha: float = 1e-6
    extra: dict = field(default_factory=dict)


def normalize_y(y, normalize=True):
    """SK/gaussian_process/_gpr.py:275-285 + SK/preprocessing/_data.py:116-119."""
    y = np.asarray(y, dtype=float)
    if not normalize:
        return y, 0.0, 1.0
    m = np.mean(y, axis=0)
    s = np.std(y, axis=0)
    if s == 0.0:
        s = 1.0
    return (y - m) / s, float(m), float(s)


def fit_fixed(X, y, *, kind=KIND_MATERN, nu=2.5, length_scale=1.0, const=1.0, alpha=1e-6,
              normalize=True) -> GPState:
    """Tail of GaussianProcessRegressor.fit at a given theta: K, K_ii += alpha, L = chol(K),
    alpha_ = K^-1 y   (SK/gaussian_process/_gpr.py:349-367).  Raises np.linalg.LinAlgError
    when K is not positive definite, as SP/linalg/_decomp_cholesky.py:58 does."""
    X = np.ascontiguousarray(X, dtype=float)
    yn, m, s = normalize_y(y, normalize)
    K = kernel_train(X, kind=kind, nu=nu, length_scale=length_scale, const=const)
    K[np.diag_indices_from(K)] += alpha
    L = cholesky(K, lower=True, check_finite=False)
    a = cho_solve((L, True), yn, check_finite=False)
    return GPState(X=X, y_norm=yn, y_mean=m, y_std=s, L=L, alpha_=a, kind=kind, nu=nu,
                   length_scale=length_scale, const=const, alpha=alpha)


def lml_and_grad(X, y_norm, *, kind=KIND_MATERN, nu=2.5, length_scale=1.0, const=1.0,
                 alpha=1e-6, eval_gradient=True):
    """log-marginal likelihood and its gradient wrt log-hyper-parameters
    (SK/gaussian_process/_gpr.py:541-656).  Non-PD K -> (-inf, zeros) (:590-593)."""
    out = kernel_train(X, kind=kind, nu=nu, length_scale=length_scale, const=const,
                       eval_gradient=eval_gradient)
    K, G = out if eval_gradient else (out, None)
    K = K.copy()
    K[np.diag_indices_from(K)] += alpha
    try:
        L = cholesky(K, lower=True, check_finite=False)
    except np.linalg.LinAlgError:
        return (-np.inf, np.zeros(G.shape[2])) if eval_gradient else -np.inf
    a = cho_solve((L, True), y_norm, check_finite=False)
    lml = -0.5 * float(y_norm @ a) - np.log(np.diag(L)).sum() - K.shape[0] / 2 * np.log(2 * np.pi)
    if not eval_gradient:
        return lml
    inner = np.outer(a, a) - cho_solve((L, True), np.eye(K.shape[0]), check_finite=False)
    grad = 0.5 * np.einsum("ij,jik->k", inner, G)
    return lml, grad


def predict(st: GPState, Xc, return_std=True):
    """GaussianProcessRegressor.predict (SK/gaussian_process/_gpr.py:446-500): mean = s*K*a+m,
    V = L^-1 K*^T (ONE forward solve), var = diag - sum V^2, negatives -> 0, std = sqrt(var*s^2)."""
    Xc = np.atleast_2d(Xc)
    Ks = kernel_cross(Xc, st.X, kind=st.kind, nu=st.nu, length_scale=st.length_scale, const=st.const)
    mu = st.y_std * (Ks @ st.alpha_) + st.y_mean
    if not return_std:
        return mu
    V = solve_triangular(st.L, Ks.T, lower=True, check_finite=False)
    var = np.full(Xc.shape[0], st.const, dtype=float)  # kernel_.diag(X): ones (* const)
    var -= np.einsum("ij,ji->i", V.T, V)
    var[var < 0] = 0.0
    return mu, np.sqrt(var * st.y_std**2)


def predict_chunked(st: GPState, Xc, chunk=1 << 14):
    mus, sds = [], []
    for i in range(0, Xc.shape[0], chunk):
        m, s = predict(st, Xc[i:i + chunk])
        mus.append(m)
        sds.append(s)
    return np.concatenate(mus), np.concatenate(sds)


# --------------------------------------------------------------------------------------
# acquisition  (R/bayes_opt/acquisition.py:485, :660-661, :847-849) and constraints
# (R/bayes_opt/constraint.py:191-221)
# --------------------------------------------------------------------------------------
def base_acq(kind, mean, std, *, kappa=2.576, xi=0.01, y_max=None):
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == ACQ_UCB:
            return mean + kappa * std
        if y_max is None:
            raise ValueError("y_max is not set")
        a = mean - y_max - xi
        z = a / std
        if kind == ACQ_POI:
            return ndtr(z)
        if kind == ACQ_EI:
            return a * ndtr(z) + std * (np.exp(-z**2 / 2.0) / _SQRT2PI)
    raise ValueError(kind)


def _frozen_norm_cdf(b, loc, scale):
    """scipy.stats.norm(loc, scale).cdf(b): NaN unless scale > 0 (rv_continuous argcheck), else
    ndtr((b-loc)/scale)  (SP/stats/_distn_infrastructure.py cdf, _continuous_distns.py:370)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        v = ndtr((b - loc) / scale)
    return np.where(scale > 0, v, np.nan)


def constraint_prob(states, lb, ub, Xc, chunk=1 << 14):
    """prod_j [Phi((ub_j-mu_j)/sd_j) - Phi((lb_j-mu_j)/sd_j)], with lb=-inf -> 0, ub=+inf -> 1
    (R/bayes_opt/constraint.py:200-221; scipy's frozen norm gives NaN for scale<=0...0/0)."""
    lb = np.atleast_1d(lb)
    ub = np.atleast_1d(ub)
    res = np.ones(Xc.shape[0])
    with np.errstate(divide="ignore", invalid="ignore"):
        for j, st in enumerate(states):
            mu, sd = predict_chunked(st, Xc, chunk)
            p_lo = _frozen_norm_cdf(lb[j], mu, sd) if lb[j] != -np.inf else 0.0
            p_hi = _frozen_norm_cdf(ub[j], mu, sd) if ub[j] != np.inf else 1.0
            res = res * (p_hi - p_lo)
    return res


def acq_closure(st: GPState, kind, *, kappa=2.576, xi=0.01, y_max=None, constraint=None,
                chunk=1 << 14):
    """The negated acquisition the reference minimises (R/bayes_opt/acquisition.py:171-219).
    ``constraint`` = (states, lb, ub) or None."""
    d = st.X.shape[1]

    def acq(x):
        x = np.asarray(x, dtype=float).reshape(-1, d)
        mu, sd = predict_chunked(st, x, chunk)
        v = -1 * base_acq(kind, mu, sd, kappa=kappa, xi=xi, y_max=y_max)
        if constraint is not None:
            v = v * constraint_prob(constraint[0], constraint[1], constraint[2], x, chunk)
        return v

    return acq


def argmin_topk(ys, k):
    """R/bayes_opt/acquisition.py:313-317: argmin (first NaN wins, lowest index on ties) and the
    k smallest by a stable sort.  NOTE: the reference uses np.argsort's default introsort, whose
    order among exactly tied values is unspecified; the oracle (and the CUDA path) use the
    stable order (value, index) - identical whenever values are distinct."""
    i = int(np.argmin(ys))
    order = np.argsort(ys, kind="stable")[:k]
    return i, float(ys[i]), order


# ---------------------------------------------------------------------------------------------------
# Throughput-mode candidate source: Philox4x32-10 (Salmon, Moraes, Dror, Shaw: "Parallel random numbers:
# as easy as 1, 2, 3", SC'11), restated with numpy uint64 arithmetic.  The reference has no counterpart
# (it draws candidates from MT19937 on the host, R/bayes_opt/target_space.py:565-603); this pins the CUDA
# generator in csrc/select.cuh bit for bit:
#   counter = (row_lo32, row_hi32, col // 2, 0), key = (seed_lo32, seed_hi32)
#   word    = o0 | o1 << 32 (even col) or o2 | o3 << 32 (odd col);  u = (word >> 11) * 2^-53
#   x       = lo + (hi - lo) * u      (two roundings)
# ---------------------------------------------------------------------------------------------------
def philox4x32_10(c0, c1, c2, c3, k0, k1):
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
    mask = np.uint64(0xFFFFFFFF)
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & mask for c in (c0, c1, c2, c3))
    k0, k1 = np.uint64(k0) & mask, np.uint64(k1) & mask
    s32 = np.uint64(32)
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2  # 32x32 -> 64 bit products (no overflow in uint64)
        c0, c1, c2, c3 = ((p1 >> s32) ^ c1 ^ k0) & mask, p1 & mask, ((p0 >> s32) ^ c3 ^ k1) & mask, p0 & mask
        k0, k1 = (k0 + W0) & mask, (k1 + W1) & mask
    return c0, c1, c2, c3


def philox_uniform(seed, rows, d, lo, hi):
    """Candidate rows `rows` (global indices) of the throughput-mode matrix: shape (len(rows), d)."""
    rows = np.asarray(rows, dtype=np.int64).astype(np.uint64)
    lo, hi = np.asarray(lo, dtype=np.float64), np.asarray(hi, dtype=np.float64)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    out = np.empty((len(rows), d))
    with np.errstate(over="ignore"):
        for b in range((d + 1) // 2):
            o0, o1, o2, o3 = philox4x32_10(rows & np.uint64(0xFFFFFFFF), rows >> np.uint64(32),
                                           np.full(len(rows), b, dtype=np.uint64), np.zeros(len(rows), dtype=np.uint64),
                                           seed & 0xFFFFFFFF, seed >> 32)
            for half, (a, bb) in enumerate(((o0, o1), (o2, o3))):
                j = 2 * b + half
                if j >= d:
                    break
                w = a | (bb << np.uint64(32))
                u = (w >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
                out[:, j] = lo[j] + (hi[j] - lo[j]) * u
    return out

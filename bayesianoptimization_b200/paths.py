"""Posterior sample paths of a fitted device GP - the function draws behind Thompson sampling.

``B200GaussianProcessRegressor.sample_paths(n_paths, n_features, random_state)`` returns a ``PosteriorPaths``:
q fixed, smooth functions drawn from the GP posterior by pathwise conditioning (Wilson et al., ICML 2020),

    path_p(x) = s_y * ( sum_l W[l, p] phi_l(xs) + sum_i V[i, p] k(xs, Xs_i) ) + y_mean,    xs = transform(x) / ls
    phi_l(xs) = sqrt(2 c / L) cos(omega_l . xs + b_l)
    V = K^-1 (y_norm - Phi(Xs) W - eps)

The first sum is a random-Fourier-feature draw from the prior (an approximation with L features), the second an
exact data-dependent update.  A path samples the latent function: the WhiteKernel term is observation noise, it
enters eps and K's diagonal and not the path.  Evaluating a path costs O(N d + L d) per candidate, with no N^2
term, and q paths share one candidate tile (``csrc/paths.cuh``).

Every random number comes from the caller's RandomState, drawn on the host in the order of ``draw_path_inputs``;
the arrays cross the C ABI as they are.  This module needs numpy/sklearn and the CUDA library, not ``bayes_opt``.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
from sklearn.utils import check_random_state

from . import _lib as B

_NU = {B.NU_05: 0.5, B.NU_15: 1.5, B.NU_25: 2.5, B.NU_INF: np.inf}


def draw_path_inputs(rs, n_paths, n_features, d, nu, n, noise_var):
    """The draws of q = n_paths paths with L = n_features features, consumed from ``rs`` in exactly this order:

        z     = rs.standard_normal((L, d))
        u     = rs.chisquare(2 nu, L)                 (Matern nu in {0.5, 1.5, 2.5} only)
        omega = z * sqrt(2 nu / u)[:, None]           (multivariate t, 2 nu dof; omega = z for RBF / nu = inf)
        b     = rs.uniform(0, 2 pi, L)
        w     = rs.standard_normal((L, q))
        eps   = rs.standard_normal((n, q)) * sqrt(noise_var)

    omega is the spectral draw of the unit-length-scale kernel: the length scales are already divided out of xs."""
    L, q = int(n_features), int(n_paths)
    z = rs.standard_normal((L, d))
    if np.isinf(nu):
        omega = z
    else:
        u = rs.chisquare(2.0 * nu, L)
        omega = z * np.sqrt(2.0 * nu / u)[:, None]
    b = rs.uniform(0.0, 2.0 * np.pi, L)
    w = rs.standard_normal((L, q))
    eps = rs.standard_normal((n, q)) * np.sqrt(noise_var)
    return omega, b, w, eps


def _row_paths(path_idx, m, q):
    """path_idx as the (m,) int32 array of the C ABI.  Values are clipped to [-1, q] only so that the narrowing
    cannot wrap: an index outside [0, q) stays outside and the ABI rejects it."""
    pidx = np.asarray(path_idx)
    if pidx.dtype.kind not in "iu":
        raise ValueError(f"path_idx must be integers, got dtype {pidx.dtype}")
    pidx = pidx.reshape(-1)
    if pidx.shape[0] != m:
        raise ValueError(f"path_idx has {pidx.shape[0]} entries for {m} rows")
    return np.ascontiguousarray(np.where(pidx < 0, -1, np.minimum(pidx, q)), dtype=np.int32)


class _PathsHandle:
    """Owns one b200bo_paths*."""

    def __init__(self):
        self.ptr = C.c_void_p()

    def __del__(self):
        try:
            if self.ptr:
                B.lib().b200bo_paths_destroy(self.ptr)
                self.ptr = C.c_void_p()
        except Exception:  # interpreter shutdown
            pass


class PosteriorPaths:
    """q posterior sample paths of a fitted B200GaussianProcessRegressor, evaluated on the GP's fit device.

    ``paths(X)`` -> (M, q) values in data units; ``argmin_topk`` / ``argmin_topk_philox`` rank -path_p per path
    on the device.  The paths own copies of the GP state they evaluate: refitting the GP afterwards does not
    change them."""

    def __init__(self, gp, n_paths=1, n_features=4096, random_state=None):
        from .gpr import parse_kernel

        if isinstance(n_paths, bool) or not isinstance(n_paths, (int, np.integer)) or not 1 <= n_paths <= B.MAX_PATHS:
            raise ValueError(f"n_paths must be an integer in [1, {B.MAX_PATHS}], got {n_paths!r}")
        if isinstance(n_features, bool) or not isinstance(n_features, (int, np.integer)) or n_features < 1:
            raise ValueError(f"n_features must be a positive integer, got {n_features!r}")
        gp._ensure_device_fit()  # "GP is not fitted" when it is not
        ek = parse_kernel(gp.kernel_)
        h = gp._handle()
        L = B.lib()
        self.n_paths = int(n_paths)
        self.n_features = int(n_features)
        self.dim = gp.X_train_.shape[1]
        self.device = int(gp.device)
        self.devices = [self.device]
        self._xform = gp.__dict__.get("_b200_xform", ("device", None))
        self._d = int(L.b200bo_gp_dim(h.ptr))  # after a host-side transform (one-hot): the transformed width
        n = int(L.b200bo_gp_n(h.ptr))
        rs = check_random_state(random_state)
        omega, b, w, eps = draw_path_inputs(rs, self.n_paths, self.n_features, self._d, _NU[ek.nu],
                                            n, float(gp.alpha) + ek.noise)
        self._handle = _PathsHandle()
        B.check(L.b200bo_paths_create(h.ptr, self.n_paths, self.n_features, B.as_dp(B.c_f64(omega)),
                                      B.as_dp(B.c_f64(b)), B.as_dp(B.c_f64(w)), B.as_dp(B.c_f64(eps)),
                                      C.byref(self._handle.ptr)))

    # the selection entry points: _c_select and _c_select + "_philox", called with _args() in front
    _c_select = "b200bo_paths_argmin_topk"

    def _args(self):
        return (self._handle.ptr,)

    def _candidates(self, X):
        X = B.c_f64(np.asarray(X, dtype=np.float64).reshape(-1, self.dim))
        mode, arg = self._xform
        if mode == "host":  # the batch-dependent transform (categorical one-hot), as FusedAcquisition applies it
            X = B.c_f64(np.asarray(arg(X), dtype=np.float64))
        return X

    def __call__(self, X):
        """(M, q) path values at the rows of X (data units)."""
        X = self._candidates(X)
        out = np.empty((X.shape[0], self.n_paths))
        B.check(B.lib().b200bo_paths_eval(self._handle.ptr, B.as_dp(X), X.shape[0], B.as_dp(out)))
        return out

    def eval_rows(self, X, path_idx):
        """(M,) values: row i of X on path path_idx[i] only, bit-equal to ``self(X)[i, path_idx[i]]`` at 1/q of its
        cost.  An index outside [0, q) raises ValueError."""
        X = self._candidates(X)
        pidx = _row_paths(path_idx, X.shape[0], self.n_paths)
        out = np.empty(X.shape[0])
        B.check(B.lib().b200bo_paths_eval_rows(self._handle.ptr, B.as_dp(X), pidx.ctypes.data_as(C.POINTER(C.c_int32)),
                                               X.shape[0], B.as_dp(out)))
        return out

    def grad_rows(self, X, path_idx):
        """(vals (M,), grads (M, d)): row i of X on path path_idx[i], the value bit-equal to ``eval_rows`` and its
        analytic gradient with respect to the row (``b200bo_paths_grad_rows``).  Host-side input transforms are not
        differentiated."""
        if self._xform[0] == "host":
            raise NotImplementedError("analytic gradients with a host-side kernel transform")
        X = self._candidates(X)
        pidx = _row_paths(path_idx, X.shape[0], self.n_paths)
        vals, grads = np.empty(X.shape[0]), np.empty((X.shape[0], self.dim))
        B.check(B.lib().b200bo_paths_grad_rows(self._handle.ptr, B.as_dp(X), pidx.ctypes.data_as(C.POINTER(C.c_int32)),
                                               X.shape[0], B.as_dp(vals), B.as_dp(grads)))
        return vals, grads

    def argmin_topk(self, X, k):
        """Per path p: np.argmin and the k smallest (np.argsort order) of -path_p (ConstrainedPaths: -merit_p) over
        the rows of X.  Returns (idx (q,), values (q,), [top-k indices of path p for p < q])."""
        X = self._candidates(X)
        k = int(k)
        q = self.n_paths
        bv, bi = np.empty(q), np.empty(q, dtype=np.int64)
        tv, ti = np.empty(q * max(k, 1)), np.empty(q * max(k, 1), dtype=np.int64)
        B.check(getattr(B.lib(), self._c_select)(*self._args(), B.as_dp(X), X.shape[0], k, B.as_dp(bv),
                                                 bi.ctypes.data_as(C.POINTER(C.c_int64)), B.as_dp(tv),
                                                 ti.ctypes.data_as(C.POINTER(C.c_int64))))
        tops = [t[t >= 0] for t in ti[:q * k].reshape(q, k)]
        return bi, bv, tops

    def argmin_topk_philox(self, seed, bounds, m, k, index_base=0):
        """Throughput mode: per path, the selection over m candidates generated inside the kernel (Philox4x32-10
        keyed by (seed, global row index), the layout of FusedAcquisition.argmin_topk_philox).
        Returns (idx (q,), values (q,), x_best (q, d), [top-k indices], [top-k rows])."""
        if self._xform[0] == "host":
            raise NotImplementedError("device candidate generation with a host-side kernel transform")
        bounds = np.asarray(bounds, dtype=np.float64).reshape(self.dim, 2)
        lo, hi = B.c_f64(bounds[:, 0]), B.c_f64(bounds[:, 1])
        return self._select_philox("_philox", (B.as_dp(lo), B.as_dp(hi)), seed, m, k, index_base)

    def argmin_topk_philox_tr(self, seed, lo, hi, center, p, m, k, index_base=0):
        """``argmin_topk_philox`` over the trust-region source (``b200bo_*_argmin_topk_philox_tr``): the centre with a
        random subset of its coordinates redrawn in the box [lo, hi], each perturbed with probability p besides one
        forced column per row (DESIGN.md 4.18).  Same returns."""
        if self._xform[0] == "host":
            raise NotImplementedError("device candidate generation with a host-side kernel transform")
        lo, hi, center = (B.c_f64(np.asarray(a, dtype=np.float64).reshape(self.dim)) for a in (lo, hi, center))
        return self._select_philox("_philox_tr", (B.as_dp(lo), B.as_dp(hi), B.as_dp(center), float(p)), seed, m, k,
                                   index_base)

    def _select_philox(self, suffix, source, seed, m, k, index_base):
        """The selection entry _c_select + suffix over a device candidate source: its arguments `source` go between
        the seed and m."""
        k, q, d = int(k), self.n_paths, self.dim
        kk = max(k, 1)
        bv, bi, bx = np.empty(q), np.empty(q, dtype=np.int64), np.empty((q, d))
        tv, ti, tx = np.empty(q * kk), np.empty(q * kk, dtype=np.int64), np.empty((q * kk, d))
        B.check(getattr(B.lib(), self._c_select + suffix)(
            *self._args(), int(seed) & 0xFFFFFFFFFFFFFFFF, *source, int(m), int(index_base), k,
            B.as_dp(bv), bi.ctypes.data_as(C.POINTER(C.c_int64)), B.as_dp(bx), B.as_dp(tv),
            ti.ctypes.data_as(C.POINTER(C.c_int64)), B.as_dp(tx)))
        ti, tx = ti[:q * k].reshape(q, k), tx[:q * k].reshape(q, k, d)
        keep = ti >= 0
        return bi, bv, bx, [ti[r][keep[r]] for r in range(q)], [tx[r][keep[r]] for r in range(q)]

    def bound(self):
        """(q,) B_p >= |path_p(x)| for every x (computed at creation from the path's own weights)."""
        out = np.empty(self.n_paths)
        B.check(B.lib().b200bo_paths_bound(self._handle.ptr, B.as_dp(out)))
        return out


class ConstrainedPaths:
    """Joint posterior paths of a target GP and J constraint GPs, ranked feasible-first (SCBO: Eriksson & Poloczek,
    "Scalable Constrained Bayesian Optimization", AISTATS 2021).  Path p of every set is one joint draw; per
    candidate x and path p, with f the target path and c_j constraint path j (data units):

        viol_p(x)  = sum_j (max(0, lb_j - c_j) + max(0, c_j - ub_j))            (0 iff every lb_j <= c_j <= ub_j)
        merit_p(x) = f  if viol_p(x) == 0,  else  -T_p (1 + viol_p(x)),    T_p = 2 B_p + 1 (target.bound())

    Every infeasible merit lies below every feasible one, and among infeasible candidates the smallest violation
    ranks first, so no feasible point needs to be registered.  The interface is PosteriorPaths': ``paths(X)`` ->
    (M, q) merit, ``raw(X)`` -> (M, G, q) values, ``argmin_topk`` / ``argmin_topk_philox`` rank -merit_p on the
    device (``b200bo_cpaths_*``), so ``PathAcquisition(ConstrainedPaths(...))`` is a device closure."""

    def __init__(self, target, constraints, lb, ub):
        sets = [target, *constraints]
        if not constraints:
            raise ValueError("ConstrainedPaths needs at least one constraint set (use PosteriorPaths without)")
        if len(sets) > B.MAX_GPS:
            raise ValueError(f"at most {B.MAX_GPS - 1} constraint sets are supported, got {len(constraints)}")
        lb = np.asarray(lb, dtype=np.float64).reshape(-1)
        ub = np.asarray(ub, dtype=np.float64).reshape(-1)
        if lb.shape != (len(constraints),) or ub.shape != (len(constraints),):
            raise ValueError(f"lb and ub need one entry per constraint set ({len(constraints)})")
        if not np.all(lb <= ub):
            raise ValueError("constraint bounds: lb > ub")
        for j, s in enumerate(constraints):
            if s.n_paths != target.n_paths:
                raise ValueError(f"constraint set {j} has {s.n_paths} paths, the target {target.n_paths}")
            if s.dim != target.dim:
                raise ValueError(f"constraint set {j} has d={s.dim}, the target d={target.dim}")
            if s.device != target.device:
                raise ValueError(f"constraint set {j} lives on device {s.device}, the target on {target.device}")
        modes = [s._xform for s in sets]
        host = [a for m, a in modes if m == "host"]
        # `==`, not `is`: the reference hands every GP `space.kernel_transform`, a new bound method per access
        if host and (len(host) != len(modes) or any(h != host[0] for h in host)):
            raise NotImplementedError("the sets use different host-side input transforms")
        self.target, self.constraints = target, list(constraints)
        self._sets = sets  # keeps every handle alive as long as this object
        self._ptrs = (C.c_void_p * len(sets))(*[s._handle.ptr.value for s in sets])
        self._lb, self._ub = B.c_f64(lb), B.c_f64(ub)
        self._xform = modes[0]
        self.n_paths = target.n_paths
        self.n_sets = len(sets)
        self.dim = target.dim
        self.device = target.device
        self.devices = [self.device]

    def _args(self):
        return self._ptrs, self.n_sets, B.as_dp(self._lb), B.as_dp(self._ub)

    def _candidates(self, X):
        return PosteriorPaths._candidates(self, X)  # the host-side transform, once for every set

    def _eval(self, X, raw):
        X = self._candidates(X)
        m, q = X.shape[0], self.n_paths
        merit = np.empty((m, q))
        out = np.empty((m, self.n_sets, q)) if raw else None
        B.check(B.lib().b200bo_cpaths_eval(*self._args(), B.as_dp(X), m, B.as_dp(merit),
                                           B.as_dp(out) if raw else None))
        return out if raw else merit

    def __call__(self, X):
        """(M, q) merit at the rows of X."""
        return self._eval(X, raw=False)

    def raw(self, X):
        """(M, G, q) path values at the rows of X: [:, 0] the target's, [:, j] constraint set j's (data units)."""
        return self._eval(X, raw=True)

    def eval_rows(self, X, path_idx):
        """(M,) merit: row i of X on path path_idx[i] only, bit-equal to ``self(X)[i, path_idx[i]]``."""
        X = self._candidates(X)
        pidx = _row_paths(path_idx, X.shape[0], self.n_paths)
        out = np.empty(X.shape[0])
        B.check(B.lib().b200bo_cpaths_eval_rows(*self._args(), B.as_dp(X), pidx.ctypes.data_as(C.POINTER(C.c_int32)),
                                                X.shape[0], B.as_dp(out)))
        return out

    # PosteriorPaths' selection over the b200bo_cpaths_* entry points, ranking -merit_p
    _c_select = "b200bo_cpaths_argmin_topk"
    argmin_topk = PosteriorPaths.argmin_topk
    argmin_topk_philox = PosteriorPaths.argmin_topk_philox
    argmin_topk_philox_tr = PosteriorPaths.argmin_topk_philox_tr
    _select_philox = PosteriorPaths._select_philox


class PathAcquisition:
    """Acquisition closure over path 0 of a PosteriorPaths: x (M,d)|(d,) -> (M,) values of -path(x), with the
    device selection of the random stage (``argmin_topk``, ``argmin_topk_philox``) in the signatures of
    ``FusedAcquisition``, so the hooks of the acquisition seam rank and refine it on the device."""

    def __init__(self, paths):
        self.paths = paths
        self.devices = paths.devices
        if not hasattr(paths, "grad_rows"):
            self.value_and_grad = None  # not offered: the refinement stays on the stencil

    def __call__(self, x):
        return -self.paths(x)[:, 0]

    def value_and_grad(self, x):
        """(vals (M,), grads (M, d)) of -path_0.  Offered over unconstrained paths only: a ConstrainedPaths merit is
        piecewise and has no ``grad_rows``."""
        x = np.asarray(x, dtype=np.float64).reshape(-1, self.paths.dim)
        v, g = self.paths.grad_rows(x, np.zeros(x.shape[0], dtype=np.int32))
        return -v, -g

    def argmin_topk(self, x, k):
        idx, val, tops = self.paths.argmin_topk(x, k)
        return int(idx[0]), float(val[0]), tops[0]

    def argmin_topk_philox(self, seed, bounds, m, k, index_base=0):
        idx, val, bx, ti, tx = self.paths.argmin_topk_philox(seed, bounds, m, k, index_base)
        return int(idx[0]), float(val[0]), bx[0], ti[0], tx[0]

    def argmin_topk_philox_tr(self, seed, lo, hi, center, p, m, k, index_base=0):
        idx, val, bx, ti, tx = self.paths.argmin_topk_philox_tr(seed, lo, hi, center, p, m, k, index_base)
        return int(idx[0]), float(val[0]), bx[0], ti[0], tx[0]


class PathBatchAcquisition:
    """Closure over ALL q paths of a PosteriorPaths / ConstrainedPaths, for batch Thompson sampling
    (``ThompsonSampling.suggest_batch``): ``acq(x, path_idx)`` -> (M,) values of -path_{path_idx[i]}(x_i), one device
    call whatever mix of paths the rows belong to (the lockstep refinement of q x n_smart runs).  ``path(p)`` is the
    single-path closure x -> -path_p(x) with the same values."""

    def __init__(self, paths):
        self.paths = paths
        self.devices = paths.devices
        self.n_paths = paths.n_paths
        if not hasattr(paths, "grad_rows"):
            self.value_and_grad = None  # not offered: the refinement stays on the stencil

    def __call__(self, x, path_idx):
        return -self.paths.eval_rows(x, path_idx)

    def value_and_grad(self, x, path_idx):
        """(vals (M,), grads (M, d)) of -path_{path_idx[i]}(x_i); unconstrained paths only."""
        v, g = self.paths.grad_rows(x, path_idx)
        return -v, -g

    def path(self, p):
        p, dim = int(p), self.paths.dim

        def acq(x):
            x = np.asarray(x, dtype=np.float64).reshape(-1, dim)
            return self(x, np.full(x.shape[0], p, dtype=np.int32))

        return acq

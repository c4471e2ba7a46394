"""Device closure of the acquisition seam and the batched L-BFGS-B driver.

``FusedAcquisition`` is what replaces the closure built by ``AcquisitionFunction._get_acq``
(R/bayes_opt/acquisition.py:171-219): x (M,d)|(d,) -> (M,) values of  -base_acq(mu, sigma) [* p_constraint]
evaluated for the whole batch by ONE fused sm_90a launch (``b200bo_acq_eval``), plus the selection
step of ``_random_sample_minimize`` (:311-317) on the device (``b200bo_acq_argmin_topk``).  With more than
one device (``B200GaussianProcessRegressor(devices=[...])``) the candidate rows are sharded over the
replicas and the per-device (argmin, top-k) records are merged by one NCCL all-gather
(``b200bo_multi_gpu_*``, SURVEY.md 8e).

``lockstep_lbfgsb`` advances the n_smart independent L-BFGS-B runs of ``_smart_minimize`` (:365-366)
together so that every round of objective / finite-difference-stencil requests of ALL seeds is one device
call; each run still sees exactly the values it would see alone.

This module needs only numpy/scipy/sklearn and the CUDA library - not ``bayes_opt``.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
import threading

import numpy as np
from scipy.optimize import minimize

from . import _lib as B
from .gpr import B200GaussianProcessRegressor


def _as_b200_gp(gp):
    if not isinstance(gp, B200GaussianProcessRegressor):
        raise TypeError(
            "the B200 acquisition functions need a B200GaussianProcessRegressor (got "
            f"{type(gp).__name__}); use bayesianoptimization_b200.enable(optimizer) or construct "
            "the GP with B200GaussianProcessRegressor - there is no CPU fallback")
    return gp


_NEEDS_Y_MAX = (B.ACQ_EI, B.ACQ_POI, B.ACQ_LOGEI, B.ACQ_LOGPOI)


class FusedAcquisition:
    """Callable closure over fitted device GPs.

    kind      B.ACQ_UCB / ACQ_EI / ACQ_POI / ACQ_MES / ACQ_LOGEI / ACQ_LOGPOI / ACQ_NEI / ACQ_LOGNEI / ACQ_CNEI /
              ACQ_LOGCNEI
    gp        fitted B200GaussianProcessRegressor (target)
    constraint  object with .model (list of device GPs), .lb, .ub  (bayes_opt ConstraintModel) or None
    params    either fixed ``kappa``/``xi``/``y_max`` values or ``owner``: an acquisition object whose
              current kappa / xi / y_max are read at every call, as the reference closure does
              (it calls self.base_acq at call time, R/bayes_opt/acquisition.py:207,217).
    max_values  ACQ_MES only: the K (1..16) samples y* of the maximum, data units (include/b200bo.h).  They are
              set on every device handle of the target GP each time the specs are built, so several MES closures
              over one GP, called alternately, each see their own samples.
    fantasies   ACQ_NEI / ACQ_LOGNEI only: ``gp.noiseless_fantasies(...)``.  The spec's gps[0] is its noiseless handle;
              candidate transforms and the device come from ``gp``.  One device; always fp64 (DESIGN.md 4.13).
              ACQ_CNEI / ACQ_LOGCNEI: the target's, as for NEI.
    constraint_fantasies  ACQ_CNEI / ACQ_LOGCNEI only: one ``noiseless_fantasies`` per constraint GP, in
              ``constraint.model`` order, each with the S of ``fantasies``.  The spec's gps[j] are their noiseless handles
              (DESIGN.md 4.15).
    """

    def __init__(self, kind, gp, constraint=None, kappa=0.0, xi=0.0, y_max=None, owner=None, max_values=None,
                 fantasies=None, constraint_fantasies=None):
        gp = _as_b200_gp(gp)
        self.kind = int(kind)
        self._ystar = None
        self._fant = None
        self._cfant = None
        if self.kind in (B.ACQ_CNEI, B.ACQ_LOGCNEI):
            n_con = 0 if constraint is None else len(constraint.model)
            cf = list(constraint_fantasies or [])
            if fantasies is None or len(cf) != n_con:
                raise ValueError("CNEI needs the target's fantasies and one per constraint GP "
                                 "(B200GaussianProcessRegressor.noiseless_fantasies)")
            if any(len(g.device_list()) > 1 for g in [gp, *(constraint.model if n_con else [])]):
                raise NotImplementedError("constrained noisy expected improvement runs on one device: a GP is "
                                          "multi-device")
            self._fant, self._cfant = fantasies, cf
        elif constraint_fantasies is not None:
            raise ValueError("constraint_fantasies belong to ACQ_CNEI / ACQ_LOGCNEI only")
        elif self.kind in (B.ACQ_NEI, B.ACQ_LOGNEI):
            if fantasies is None:
                raise ValueError("NEI needs fantasies (B200GaussianProcessRegressor.noiseless_fantasies)")
            if len(gp.device_list()) > 1:
                raise NotImplementedError("noisy expected improvement runs on one device: the GP is multi-device")
            self._fant = fantasies
        elif fantasies is not None:
            raise ValueError("fantasies belong to ACQ_NEI / ACQ_LOGNEI / ACQ_CNEI / ACQ_LOGCNEI only")
        if self.kind == B.ACQ_MES:
            ys = B.c_f64(np.asarray(max_values if max_values is not None else [], dtype=np.float64).reshape(-1))
            if not 1 <= ys.size <= B.MAX_PATHS or not np.all(np.isfinite(ys)):
                raise ValueError(f"MES needs 1..{B.MAX_PATHS} finite max_values, got {max_values!r}")
            self._ystar = ys
        elif max_values is not None:
            raise ValueError("max_values belong to ACQ_MES only")
        self.dim = gp.X_train_.shape[1]
        self._gps = [gp]
        self._bounds = [(0.0, 0.0)]
        self._owner = owner
        self._fixed = (float(kappa), float(xi), None if y_max is None else float(y_max))
        if constraint is not None:
            models = constraint.model
            if len(models) + 1 > B.MAX_GPS:
                raise NotImplementedError(f"at most {B.MAX_GPS - 1} constraint GPs are supported")
            for j, cgp in enumerate(models):
                self._gps.append(_as_b200_gp(cgp))
                self._bounds.append((float(constraint.lb[j]), float(constraint.ub[j])))
        devs = self._gps[0].device_list()
        for g in self._gps[1:]:
            if g.device_list() != devs:
                raise ValueError("all GPs of one acquisition call must live on the same device list")
        self.devices = devs
        self._path = B.PATH_AUTO
        self._specs = None
        self._sig = None

    # ---- spec construction (one b200bo_acq per device) ------------------------------------------
    def _params(self):
        if self._owner is None:
            return self._fixed
        o = self._owner
        y_max = getattr(o, "y_max", None)
        if self.kind in _NEEDS_Y_MAX and y_max is None:
            o.base_acq(np.zeros(1), np.ones(1))  # raises the reference's own "y_max is not set" ValueError
        return float(getattr(o, "kappa", 0.0)), float(getattr(o, "xi", 0.0)), y_max

    def _build_specs(self):
        # an LML evaluation in between re-uses the factor buffers: refit lazily, then (re)bind handles
        handles = [g._device_handles() for g in self._gps]  # [gp][device]
        if self._fant is not None:
            handles[0] = [self._fant.handle]  # the noiseless handle holding the fantasies
        for j, f in enumerate(self._cfant or []):
            handles[1 + j] = [f.handle]
        sig = tuple(h.ptr.value for hs in handles for h in hs)
        kappa, xi, y_max = self._params()
        if self.kind in _NEEDS_Y_MAX and y_max is None:
            raise ValueError("y_max is not set. If you are calling this method outside of suggest(), "
                             "you must set y_max manually.")
        if self._specs is None or sig != self._sig:
            specs = (B.AcqSpec * len(self.devices))()
            for dv in range(len(self.devices)):
                sp = specs[dv]
                sp.kind = self.kind
                sp.n_gps = len(self._gps)
                for g in range(len(self._gps)):
                    sp.gps[g] = handles[g][dv].ptr.value
                    sp.lb[g], sp.ub[g] = self._bounds[g]
            self._specs, self._sig, self._keep = specs, sig, handles
        if self._ystar is not None:
            for h in handles[0]:
                B.check(B.lib().b200bo_gp_set_max_values(h.ptr, B.as_dp(self._ystar), self._ystar.size))
        for sp in self._specs:
            sp.kappa, sp.xi = kappa, xi
            sp.y_max = 0.0 if y_max is None else float(y_max)
            sp.path = self._path
        return self._specs

    @property
    def spec(self):
        """The b200bo_acq of the primary device (device-resident entry points, bench.py)."""
        return self._build_specs()[0]

    def _candidates(self, x):
        x = B.c_f64(np.asarray(x, dtype=np.float64).reshape(-1, self.dim))
        # NaN / inf in x: the kernels count non-finite coordinates while loading them and the C entry point returns
        # B200BO_ERR_ARG -> ValueError("Input X contains NaN or infinity.") as sklearn's validate_data would - no
        # separate pass over the batch on the host
        # kernels with a host-side input transform (categorical one-hot): every GP of the call must
        # see the same transformed batch, as in the reference where they share space.kernel_transform
        for g in self._gps:
            g._ensure_device_fit()
        modes = [g.__dict__.get("_b200_xform", ("device", None)) for g in self._gps]
        host = [a for m, a in modes if m == "host"]
        if host:
            # `==`, not `is`: the reference hands every GP `space.kernel_transform`, a bound method - each attribute
            # access makes a new method object, equal iff same function of the same space
            if len(host) != len(modes) or any(h != host[0] for h in host):
                raise NotImplementedError("GPs of one acquisition call use different host-side input transforms")
            x = self._gps[0]._device_candidates(x)
        return x

    @contextlib.contextmanager
    def refine_mode(self):
        """Inside an optimiser run the objective and its finite-difference stencil arrive as batches of
        different sizes; B.PATH_STABLE makes the kernel choice a function of the model size only, so both
        are summed in the same order (a smooth offset between two kernels would become a gradient bias of
        offset/1.5e-8)."""
        prev, self._path = self._path, B.PATH_STABLE
        try:
            yield self
        finally:
            self._path = prev

    # ---- evaluation ------------------------------------------------------------------------------
    def __call__(self, x, shard_offsets=None):
        x = self._candidates(x)
        specs = self._build_specs()
        m = x.shape[0]
        out = np.empty(m)
        if len(self.devices) == 1:
            B.check(B.lib().b200bo_acq_eval(C.byref(specs[0]), B.as_dp(x), m, B.as_dp(out)))
        else:
            off = None
            if shard_offsets is not None:
                off = np.ascontiguousarray(shard_offsets, dtype=np.int64)
                if off.shape != (len(self.devices) + 1,) or off[0] != 0 or off[-1] != m or np.any(np.diff(off) < 0):
                    raise ValueError("shard_offsets must be len(devices)+1 non-decreasing row offsets from 0 to len(x)")
            B.check(B.lib().b200bo_multi_gpu_acq_eval(
                specs, len(self.devices), B.as_dp(x), m,
                off.ctypes.data_as(C.POINTER(C.c_int64)) if off is not None else None, B.as_dp(out)))
        return out

    def value_and_grad(self, x):
        """(vals (M,), grads (M, d)): the closure value and its analytic gradient with respect to x
        (``b200bo_acq_value_grad``, DESIGN.md 4.10).  One device; host-side input transforms are not differentiated."""
        if len(self.devices) != 1:
            raise NotImplementedError("value_and_grad runs on one device (multi-device gradient sharding is not built)")
        for g in self._gps:
            g._ensure_device_fit()
            if g.__dict__.get("_b200_xform", ("device", None))[0] == "host":
                raise NotImplementedError("analytic gradients with a host-side kernel transform")
        x = B.c_f64(np.asarray(x, dtype=np.float64).reshape(-1, self.dim))
        specs = self._build_specs()
        m = x.shape[0]
        vals, grads = np.empty(m), np.empty((m, self.dim))
        B.check(B.lib().b200bo_acq_value_grad(C.byref(specs[0]), B.as_dp(x), m, B.as_dp(vals), B.as_dp(grads)))
        return vals, grads

    def argmin_topk(self, x, k):
        """Evaluate + np.argmin + k smallest (value, index) on the device(s)
        (R/bayes_opt/acquisition.py:312-317).  Returns (argmin index, min value, top-k indices)."""
        x = self._candidates(x)
        specs = self._build_specs()
        k = int(k)
        best_val = C.c_double()
        best_idx = C.c_int64()
        tv = np.empty(max(k, 1))
        ti = np.empty(max(k, 1), dtype=np.int64)
        tip = ti.ctypes.data_as(C.POINTER(C.c_int64))
        if len(self.devices) == 1:
            B.check(B.lib().b200bo_acq_argmin_topk(C.byref(specs[0]), B.as_dp(x), x.shape[0], k, C.byref(best_val),
                                                   C.byref(best_idx), B.as_dp(tv), tip, None))
        else:
            B.check(B.lib().b200bo_multi_gpu_acq_argmin_topk(specs, len(self.devices), B.as_dp(x), x.shape[0], k,
                                                             C.byref(best_val), C.byref(best_idx), B.as_dp(tv), tip))
        ti = ti[:k]
        return best_idx.value, best_val.value, ti[ti >= 0]

    def argmin_topk_philox(self, seed, bounds, m, k, index_base=0):
        """Throughput mode (candidate_source="device_philox"): the m candidates are generated inside the
        fused kernel from Philox4x32-10 keyed by (seed, global row index) - they never exist in host
        memory or HBM.  Row i, column j is lo_j + u*(hi_j - lo_j) with u the 53-bit uniform of counter
        (i, j//2) (layout documented in csrc/select.cuh).  Returns (index, value, x_best,
        top-k indices, top-k rows)."""
        specs = self._build_specs()
        for g in self._gps:
            if g.__dict__.get("_b200_xform", ("device", None))[0] == "host":
                raise NotImplementedError("device candidate generation with a host-side kernel transform")
        bounds = B.c_f64(np.asarray(bounds, dtype=np.float64).reshape(self.dim, 2))
        lo, hi = B.c_f64(bounds[:, 0]), B.c_f64(bounds[:, 1])
        k = int(k)
        best_val, best_idx = C.c_double(), C.c_int64()
        bx = np.empty(self.dim)
        tv, ti, tx = np.empty(max(k, 1)), np.empty(max(k, 1), dtype=np.int64), np.empty((max(k, 1), self.dim))
        args = (int(seed) & 0xFFFFFFFFFFFFFFFF, B.as_dp(lo), B.as_dp(hi), int(m), int(index_base), k, C.byref(best_val),
                C.byref(best_idx), B.as_dp(bx), B.as_dp(tv), ti.ctypes.data_as(C.POINTER(C.c_int64)), B.as_dp(tx))
        if len(self.devices) == 1:
            B.check(B.lib().b200bo_acq_argmin_topk_philox(C.byref(specs[0]), *args))
        else:
            B.check(B.lib().b200bo_multi_gpu_acq_argmin_topk_philox(specs, len(self.devices), *args))
        keep = ti[:k] >= 0
        return best_idx.value, best_val.value, bx, ti[:k][keep], tx[:k][keep]


# ---------------------------------------------------------------------------------------------------
# batched L-BFGS-B
# ---------------------------------------------------------------------------------------------------
def _workers_supported():
    """SciPy >= 1.16 lets minimize() map the objective over the 2-point stencil through a pluggable
    ``workers`` callable (SP/optimize/_numdiff.py)."""
    try:
        from packaging import version
        from scipy import __version__ as scipy_version

        return version.parse(scipy_version) >= version.parse("1.16.0")
    except Exception:  # pragma: no cover
        return False


def _predicted_stencil(x0, lb, ub, eps=1e-8):
    """The d points x0 + h_i e_i that SciPy's 2-point scheme will request right after f(x0) (L-BFGS-B always
    evaluates the gradient at the point where it evaluated f): computed with SciPy's OWN helpers
    (SP/optimize/_numdiff.py: approx_derivative's abs_step branch + _adjust_scheme_to_bounds), so the points
    are bit-identical.  A wrong prediction only costs a cache miss."""
    from scipy.optimize._numdiff import _adjust_scheme_to_bounds, _eps_for_method

    x0 = np.asarray(x0, dtype=np.float64)
    sign_x0 = (x0 >= 0).astype(x0.dtype) * 2 - 1
    dx = (x0 + eps) - x0
    h = np.where(dx == 0, _eps_for_method(x0.dtype, np.dtype(np.float64), "2-point") * sign_x0 *
                 np.maximum(1.0, np.abs(x0)), eps).astype(x0.dtype)
    h, _ = _adjust_scheme_to_bounds(x0, h, 1, "1-sided", lb, ub)
    pts = np.tile(x0, (x0.size, 1))
    idx = np.arange(x0.size)
    pts[idx, idx] = x0 + h
    return pts


class _FusedObjective:
    """Objective + stencil map for ONE L-BFGS-B run over a batch evaluator ``evaluate(rows) -> values``.
    f(x) and the d stencil points of the gradient SciPy asks for next are evaluated in ONE call (d+1 rows);
    the stencil request is then served from the cache.  Same points, same values, same iterates as the
    reference's one-row-at-a-time loop (R/bayes_opt/acquisition.py:366) - half the device calls of a
    batched stencil alone."""

    def __init__(self, evaluate, bounds):
        self.evaluate = evaluate
        b = np.asarray(bounds, dtype=np.float64)
        self.lb, self.ub = b[:, 0].copy(), b[:, 1].copy()
        self.cache = {}
        self.speculate = _workers_supported() and os.environ.get("B200BO_SPECULATE", "1") != "0"

    def fun(self, x):
        x = np.asarray(x, dtype=np.float64)
        if self.speculate and x.ndim == 1 and np.all(x >= self.lb) and np.all(x <= self.ub):
            try:
                pts = _predicted_stencil(x, self.lb, self.ub)
            except Exception:  # SciPy internals moved: plain evaluation
                self.speculate, pts = False, None
            if pts is not None:
                ys = self.evaluate(np.vstack([x[None, :], pts]))
                self.cache = {p.tobytes(): y for p, y in zip(pts, ys[1:])}
                return ys[:1]
        return self.evaluate(np.atleast_2d(x))

    def stencil_map(self, _f, iterable):
        xs = [np.asarray(x, dtype=np.float64) for x in iterable]
        if not xs:
            return []
        hits = [self.cache.get(x.tobytes()) for x in xs]
        if all(h is not None for h in hits):
            return [np.atleast_1d(h) for h in hits]
        return [np.atleast_1d(y) for y in self.evaluate(np.vstack(xs))]

    def options(self):
        return {"workers": self.stencil_map} if _workers_supported() else None


def stencil_options(acq):
    """L-BFGS-B options that evaluate the d finite-difference points x + h_i e_i in ONE call of ``acq``
    instead of d single-row calls: same points, same differences, same iterates."""
    if not _workers_supported():
        return None

    def batched_map(fun, iterable):
        xs = [np.asarray(x, dtype=float) for x in iterable]
        if not xs:
            return []
        ys = np.asarray(acq(np.vstack(xs)), dtype=float)
        return [np.atleast_1d(y) for y in ys]

    return {"workers": batched_map}


class _LockstepEvaluator:
    """Serves the pending objective requests of several concurrently running SciPy minimisations with
    ONE call of the (device) closure.  Each minimisation runs in its own thread and blocks in
    ``evaluate`` until every still-active run has submitted its request; the last one to arrive
    evaluates the concatenated batch.  Per-candidate results of the fused kernels do not depend on what
    else is in the batch, so each run sees exactly the values it would see alone.  With several devices
    run r's rows go to device r mod G (SURVEY.md 8e)."""

    def __init__(self, acq, n_active, run_paths=None):
        self.acq = acq
        self.cv = threading.Condition()
        self.pending, self.results = {}, {}
        self.active = n_active
        self.error = None
        self.n_dev = len(getattr(acq, "devices", [0]))
        self.run_paths = run_paths

    def _flush(self):
        keys = sorted(self.pending, key=lambda k: (k % self.n_dev, k)) if self.n_dev > 1 else list(self.pending)
        xs = [self.pending[k] for k in keys]
        kw = {}
        if self.run_paths is not None:
            kw["path_idx"] = np.concatenate([np.full(len(x), self.run_paths[k], dtype=np.int32)
                                             for k, x in zip(keys, xs)])
        try:
            if self.n_dev > 1:
                counts = np.zeros(self.n_dev + 1, dtype=np.int64)
                for k, x in zip(keys, xs):
                    counts[(k % self.n_dev) + 1] += len(x)
                ys = np.asarray(self.acq(np.vstack(xs), shard_offsets=np.cumsum(counts), **kw), dtype=float)
            else:
                ys = np.asarray(self.acq(np.vstack(xs), **kw), dtype=float)
            off = 0
            for k, x in zip(keys, xs):
                self.results[k] = ys[off:off + len(x)]
                off += len(x)
        except BaseException as e:  # propagate to every waiting run
            self.error = e
        self.pending.clear()
        self.cv.notify_all()

    def evaluate(self, key, x):
        with self.cv:
            if self.error is not None:
                raise self.error
            self.pending[key] = np.atleast_2d(np.asarray(x, dtype=float))
            if len(self.pending) >= self.active:
                self._flush()
            while key not in self.results and self.error is None:
                self.cv.wait()
            if self.error is not None:
                raise self.error
            return self.results.pop(key)

    def finish(self, key):
        with self.cv:
            self.active -= 1
            if self.pending and len(self.pending) >= self.active:
                self._flush()


def _batched_lbfgsb(acq, seeds, bounds, maxcor=10, ftol=2.2204460492503131e-09, gtol=1e-5, eps=1e-8,
                    maxfun=15000, maxiter=15000, maxls=20, run_paths=None, grad=False):
    """All L-BFGS-B runs of ``_smart_minimize`` advanced TOGETHER by one Python thread around SciPy's own
    compiled core (``scipy.optimize._lbfgsb.setulb``): the driver loop of ``_minimize_lbfgsb``
    (SP/optimize/_lbfgsb_py.py:290-420: task handling, iteration / evaluation limits, warnflag -> success) and the
    2-point gradient of ``ScalarFunction`` (f(x) then (f(x + h_i e_i) - f(x)) / ((x_i + h_i) - x_i) with h from
    SciPy's ``_adjust_scheme_to_bounds``) are restated for S runs at once, so a round costs ONE device call of
    S*(d+1) rows and ~0.1 ms of host time instead of S Python optimiser frames taking turns on the GIL
    (measured: 2.4 ms per round for 10 runs).  Same core, same arithmetic, same iterates: x, fun, nit, nfev, status
    and success equal ``scipy.optimize.minimize(..., method="L-BFGS-B")`` bit for bit (tests/test_host_cpu.py).
    Raises ImportError / AttributeError when SciPy's private pieces are not the ones this was written against
    (the caller then uses the thread-per-run driver).

    grad=True: ``acq.value_and_grad(rows[, path_idx])`` supplies f and its analytic gradient, so a round is ONE row
    per pending run and nfev counts one per evaluation; the driver is otherwise the same, and the results equal
    ``scipy.optimize.minimize(fun, jac=True, method="L-BFGS-B")`` bit for bit."""
    from scipy.optimize import OptimizeResult
    from scipy.optimize import _lbfgsb_py as _sp

    setulb = _sp._lbfgsb.setulb
    int_dtype = np.int64 if _sp.HAS_ILP64 else np.int32
    b = np.asarray(bounds, dtype=np.float64)
    lb, ub = b[:, 0].copy(), b[:, 1].copy()
    if (lb > ub).any():
        raise ValueError("LBFGSB - one of the lower bounds is greater than an upper bound.")
    n = lb.size
    m = maxcor
    factr = ftol / np.finfo(float).eps
    nbd = np.zeros(n, dtype=int_dtype)
    low_bnd, upper_bnd = np.zeros(n), np.zeros(n)
    for i in range(n):
        lo_f, hi_f = not np.isinf(lb[i]), not np.isinf(ub[i])
        if lo_f:
            low_bnd[i] = lb[i]
        if hi_f:
            upper_bnd[i] = ub[i]
        nbd[i] = {(False, False): 0, (True, False): 1, (True, True): 2, (False, True): 3}[(lo_f, hi_f)]

    class Run:
        pass

    n_dev = len(getattr(acq, "devices", [0]))
    runs = []
    for k, s in enumerate(seeds):
        r = Run()
        r.dev = k % n_dev  # SURVEY.md 8e: seed r -> GPU r mod G
        r.path = None if run_paths is None else int(run_paths[k])
        r.x = np.array(np.clip(np.asarray(s, dtype=np.float64).ravel(), lb, ub), dtype=np.float64)
        r.f = np.array(0.0, dtype=np.float64)
        r.g = np.zeros(n, dtype=np.float64)
        r.wa = np.zeros(2 * m * n + 5 * n + 11 * m * m + 8 * m, np.float64)
        r.iwa = np.zeros(3 * n, dtype=int_dtype)
        r.task = np.zeros(2, dtype=int_dtype)
        r.ln_task = np.zeros(2, dtype=int_dtype)
        r.lsave = np.zeros(4, dtype=int_dtype)
        r.isave = np.zeros(44, dtype=int_dtype)
        r.dsave = np.zeros(29, dtype=np.float64)
        r.nit = r.nfev = r.njev = 0
        r.xe = None  # point of the cached (f, g), as ScalarFunction memoises it
        r.done = False
        runs.append(r)

    def evaluate_pending_grad(pending):
        """f and the analytic gradient at r.x for every pending run: one row per run."""
        kw = {}
        if run_paths is not None:
            kw["path_idx"] = np.array([r.path for r in pending], dtype=np.int32)
        rows = np.vstack([r.x for r in pending])
        fs, gs = acq.value_and_grad(rows, **kw)
        for i, r in enumerate(pending):
            r.f = float(fs[i])
            r.g = np.array(gs[i], dtype=np.float64)
            r.xe = rows[i].copy()
            r.nfev += 1
            r.njev += 1

    def evaluate_pending(pending):
        """f and the 2-point gradient at r.x for every pending run: one batch of (d+1) rows per run."""
        if grad:
            return evaluate_pending_grad(pending)
        if n_dev > 1:
            pending = sorted(pending, key=lambda r: r.dev)  # stable: rows of one device are contiguous
        blocks = []
        for r in pending:
            x0 = r.x.copy()
            pts = _predicted_stencil(x0, lb, ub, eps)
            blocks.append((x0, pts))
        rows = np.vstack([np.vstack([x0[None, :], pts]) for x0, pts in blocks])
        kw = {}
        if run_paths is not None:
            kw["path_idx"] = np.repeat(np.array([r.path for r in pending], dtype=np.int32), 1 + n)
        if n_dev > 1:
            counts = np.zeros(n_dev + 1, dtype=np.int64)
            for r in pending:
                counts[r.dev + 1] += 1 + n
            ys = np.asarray(acq(rows, shard_offsets=np.cumsum(counts), **kw), dtype=np.float64)
        else:
            ys = np.asarray(acq(rows, **kw), dtype=np.float64)
        off = 0
        for r, (x0, pts) in zip(pending, blocks):
            f0 = float(ys[off])
            idx = np.arange(n)
            dx = pts[idx, idx] - x0                      # (x0_i + h_i) - x0_i, as SP/optimize/_numdiff.py forms it
            r.g = (ys[off + 1:off + 1 + n] - f0) / dx
            r.f = f0
            r.xe = x0
            r.nfev += 1 + n
            r.njev += 1
            off += 1 + n

    evaluate_pending(runs)  # ScalarFunction.__init__ evaluates f and g at x0 before the first setulb call
    active = list(runs)
    while active:
        pending = []
        for r in active:
            while True:
                r.g = r.g.astype(np.float64)
                setulb(m, r.x, low_bnd, upper_bnd, nbd, r.f, r.g, factr, gtol, r.wa, r.iwa, r.task, r.lsave,
                       r.isave, r.dsave, maxls, r.ln_task)
                if r.task[0] == 3:
                    if r.xe is not None and np.array_equal(r.x, r.xe):
                        continue  # fun_and_grad(x) at the memoised point: no new evaluation
                    pending.append(r)
                    break
                if r.task[0] == 1:
                    r.nit += 1
                    if r.nit >= maxiter:
                        r.task[0], r.task[1] = 5, 504
                    elif r.nfev > maxfun:
                        r.task[0], r.task[1] = 5, 502
                    continue
                r.done = True
                break
        if pending:
            evaluate_pending(pending)
        active = [r for r in active if not r.done]
    out = []
    for r in runs:
        if r.task[0] == 4:
            warnflag = 0
        elif r.nfev > maxfun or r.nit >= maxiter:
            warnflag = 1
        else:
            warnflag = 2
        msg = _sp.status_messages[int(r.task[0])] + ": " + _sp.task_messages[int(r.task[1])]
        out.append(OptimizeResult(fun=r.f, jac=r.g, nfev=r.nfev, njev=r.njev, nit=r.nit, status=warnflag, message=msg,
                                  x=r.x, success=(warnflag == 0)))
    return out


def _on_path(acq, p, dim):
    """The objective of a run of path p over a closure ``acq(rows, path_idx)``."""

    def fun(x):
        rows = np.asarray(x, dtype=np.float64).reshape(-1, dim)
        return acq(rows, path_idx=np.full(rows.shape[0], p, dtype=np.int32))

    return fun


def _with_grad(acq, p, dim):
    """``fun(x) -> (f, g)`` for scipy's jac=True over ``acq.value_and_grad`` (path p when given)."""

    def fun(x):
        rows = np.asarray(x, dtype=np.float64).reshape(1, dim)
        kw = {} if p is None else {"path_idx": np.full(1, p, dtype=np.int32)}
        f, g = acq.value_and_grad(rows, **kw)
        return float(f[0]), np.array(g[0], dtype=np.float64)

    return fun


def lockstep_lbfgsb(acq, x_seeds, bounds, lockstep=True, run_paths=None, grad=False):
    """``[minimize(acq, seed, bounds=bounds, method="L-BFGS-B") for seed in x_seeds]`` (the loop at
    R/bayes_opt/acquisition.py:365-366) with the runs advanced in lockstep.  B200BO_LOCKSTEP=0 (or a
    single seed) selects the plain sequential loop.

    run_paths: None, or one path index per seed for a closure ``acq(rows, path_idx)`` over several sample paths
    (paths.PathBatchAcquisition): run r minimises path run_paths[r], and every merged call passes the path of each
    of its rows.

    grad=True: the runs use the analytic gradient of ``acq.value_and_grad`` instead of the 2-point stencil (one row
    per run and round); a single seed or B200BO_LOCKSTEP=0 runs ``minimize(fun, jac=True)`` on the same method."""
    seeds = [np.asarray(s, dtype=float) for s in x_seeds]
    dim = np.asarray(bounds).shape[0]
    if grad:
        if len(seeds) > 1 and lockstep and os.environ.get("B200BO_LOCKSTEP", "1") != "0":
            try:
                return _batched_lbfgsb(acq, seeds, bounds, run_paths=run_paths, grad=True)
            except (ImportError, AttributeError, KeyError, TypeError):
                pass  # SciPy's private L-BFGS-B pieces differ: one minimize(jac=True) per run
        return [minimize(_with_grad(acq, None if run_paths is None else int(run_paths[i]), dim), s, jac=True,
                         bounds=bounds, method="L-BFGS-B") for i, s in enumerate(seeds)]
    fun = [acq if run_paths is None else _on_path(acq, int(run_paths[i]), dim) for i in range(len(seeds))]
    if len(seeds) <= 1 or not lockstep or os.environ.get("B200BO_LOCKSTEP", "1") == "0":
        out = []
        for s, f in zip(seeds, fun):
            if lockstep:
                obj = _FusedObjective(lambda rows, f=f: np.asarray(f(rows), dtype=float), bounds)
                out.append(minimize(obj.fun, s, bounds=bounds, method="L-BFGS-B", options=obj.options()))
            else:
                out.append(minimize(f, s, bounds=bounds, method="L-BFGS-B"))
        return out
    if _workers_supported() and os.environ.get("B200BO_LBFGSB_DRIVER", "batched") == "batched":
        try:
            return _batched_lbfgsb(acq, seeds, bounds, run_paths=run_paths)
        except (ImportError, AttributeError, KeyError, TypeError):
            pass  # SciPy's private L-BFGS-B pieces differ from the ones the batched driver restates: thread driver
    ev = _LockstepEvaluator(acq, len(seeds), run_paths=run_paths)
    results, errors = [None] * len(seeds), [None] * len(seeds)

    def run(i):
        try:
            obj = _FusedObjective(lambda rows: ev.evaluate(i, rows), bounds)
            results[i] = minimize(obj.fun, seeds[i], bounds=bounds, method="L-BFGS-B", options=obj.options())
        except BaseException as e:
            errors[i] = e
        finally:
            ev.finish(i)

    threads = [threading.Thread(target=run, args=(i,), daemon=True) for i in range(len(seeds))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for e in errors:
        if e is not None:
            raise e
    return results

"""B200GaussianProcessRegressor - the GP-object seam of the drop-in boundary (SURVEY.md 8b.1).

A subclass of sklearn's ``GaussianProcessRegressor`` (the object the reference constructs at
R/bayes_opt/bayesian_optimization.py:124-130 and R/bayes_opt/constraint.py:72-81) whose
``fit`` / ``predict`` / ``log_marginal_likelihood`` run on the GPU through the C ABI in
``include/b200bo.h``.  Host logic (hyper-parameter search driver, RNG consumption, attribute
names, error types) mirrors SK/gaussian_process/_gpr.py so the reference's callers cannot tell
the difference; every matrix operation runs in hand-written sm_90a kernels.  There is no CPU
fallback: unsupported kernels raise NotImplementedError, a missing CUDA library raises
ImportError, a missing device raises B200Error.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
import warnings
from operator import itemgetter

import numpy as np
import scipy.optimize
from sklearn.base import clone
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, Product, Sum, WhiteKernel
from sklearn.utils import check_random_state
from sklearn.utils.optimize import _check_optimize_result

from . import _lib as B


def find_transform(kernel):
    """Input transform of a kernel produced by bayes_opt's ``wrap_kernel`` (R/bayes_opt/parameter.py:457-495),
    else None.  The reference keeps ``transform`` in the closure of the generated class (the ``_transform``
    attribute it also sets does not survive ``sklearn.base.clone``), so both places are searched."""
    t = getattr(kernel, "_transform", None)
    if t is not None:
        return t
    call = type(kernel).__dict__.get("__call__")
    code = getattr(call, "__code__", None)
    if code is not None and call.__closure__:
        for name, cell in zip(code.co_freevars, call.__closure__):
            if name == "transform":
                return cell.cell_contents
    if type(kernel).__name__ == "WrappedKernel":
        raise NotImplementedError("wrapped kernel whose transform cannot be located")
    return None


# --------------------------------------------------------------------------------------------
# kernel parsing: sklearn kernel object -> engine spec
# --------------------------------------------------------------------------------------------
class EngineKernel:
    """What the device needs to know about a sklearn kernel, plus the theta <-> parameter map."""

    def __init__(self, family, nu, const_value, length_scale, const_free, ls_free, const_first,
                 noise=0.0, noise_free=False, noise_first=False):
        self.family = family
        self.nu = nu
        self.const_value = float(const_value)
        self.length_scale = np.atleast_1d(np.asarray(length_scale, dtype=np.float64)).copy()
        self.const_free = const_free    # ConstantKernel present and not "fixed"
        self.ls_free = ls_free
        self.const_first = const_first  # theta order: [const, ls] (k1=Constant) or [ls, const]
        self.noise = float(noise)       # WhiteKernel term of a Sum (0 = absent)
        self.noise_free = noise_free
        self.noise_first = noise_first  # Sum(WhiteKernel, k): the noise theta comes first

    def c_spec(self):
        self._ls_keep = np.ascontiguousarray(self.length_scale, dtype=np.float64)
        return B.KernelSpec(self.family, self.nu, int(self._ls_keep.size), 0, self.const_value,
                            B.as_dp(self._ls_keep), self.noise)

    def with_theta(self, theta):
        """Engine kernel with the free hyper-parameters replaced by exp(theta)."""
        theta = np.asarray(theta, dtype=np.float64)
        k = EngineKernel(self.family, self.nu, self.const_value, self.length_scale, self.const_free,
                         self.ls_free, self.const_first, self.noise, self.noise_free, self.noise_first)
        nls = self.length_scale.size if self.ls_free else 0
        pos = 0
        if self.noise_free and self.noise_first:
            k.noise = float(np.exp(theta[pos]))
            pos += 1
        if self.const_free and self.const_first:
            k.const_value = float(np.exp(theta[pos]))
            pos += 1
        if self.ls_free:
            k.length_scale = np.exp(theta[pos:pos + nls])
            pos += nls
        if self.const_free and not self.const_first:
            k.const_value = float(np.exp(theta[pos]))
            pos += 1
        if self.noise_free and not self.noise_first:
            k.noise = float(np.exp(theta[pos]))
            pos += 1
        if pos != theta.size:
            raise ValueError("theta has the wrong number of entries")
        return k

    def select_grad(self, g_dev):
        """Device gradient order is [const (if free)], ls..., [noise (if free)]; reorder/select to theta order."""
        nls = self.length_scale.size
        off = 1 if self.const_free else 0
        g_c = g_dev[:off]
        g_l = g_dev[off:off + nls] if self.ls_free else g_dev[:0]
        g_n = g_dev[off + nls:off + nls + 1] if self.noise_free else g_dev[:0]
        inner = [g_c, g_l] if self.const_first else [g_l, g_c]
        return np.concatenate([g_n] + inner if self.noise_first else inner + [g_n])


_NU_CODES = {0.5: B.NU_05, 1.5: B.NU_15, 2.5: B.NU_25, np.inf: B.NU_INF}


def _parse_base(k):
    if isinstance(k, Matern):  # also matches WrappedKernel subclasses of Matern
        if k.nu not in _NU_CODES:
            raise NotImplementedError(
                f"Matern(nu={k.nu}) is not supported by the device engine (nu in 0.5, 1.5, 2.5, inf)")
        return B.KERNEL_MATERN, _NU_CODES[k.nu], k.length_scale, k.hyperparameter_length_scale.fixed
    if isinstance(k, RBF):
        return B.KERNEL_RBF, B.NU_INF, k.length_scale, k.hyperparameter_length_scale.fixed
    raise NotImplementedError(
        f"kernel {type(k).__name__} is not supported by the device engine; supported: Matern, RBF, "
        "optionally multiplied by a ConstantKernel, optionally wrapped by bayes_opt wrap_kernel")


def parse_kernel(kernel) -> EngineKernel:
    """sklearn kernel -> EngineKernel.  Supported set: {Matern nu in (.5,1.5,2.5,inf), RBF},
    iso/anisotropic, x ConstantKernel (either order), + WhiteKernel (either order).  Anything else:
    NotImplementedError."""
    if isinstance(kernel, Sum):
        k1, k2 = kernel.k1, kernel.k2
        if isinstance(k1, WhiteKernel) == isinstance(k2, WhiteKernel):
            raise NotImplementedError("only {Matern, RBF}[* ConstantKernel] + WhiteKernel sums are supported")
        white, other, first = (k1, k2, True) if isinstance(k1, WhiteKernel) else (k2, k1, False)
        if isinstance(other, Sum):
            raise NotImplementedError("nested kernel sums are not supported by the device engine")
        ek = parse_kernel(other)
        ek.noise = float(white.noise_level)
        ek.noise_free = not white.hyperparameter_noise_level.fixed
        ek.noise_first = first
        return ek
    if isinstance(kernel, Product):
        k1, k2 = kernel.k1, kernel.k2
        if isinstance(k1, ConstantKernel) and not isinstance(k2, ConstantKernel):
            fam, nu, ls, ls_fixed = _parse_base(k2)
            return EngineKernel(fam, nu, k1.constant_value, ls, not k1.hyperparameter_constant_value.fixed,
                                not ls_fixed, True)
        if isinstance(k2, ConstantKernel) and not isinstance(k1, ConstantKernel):
            fam, nu, ls, ls_fixed = _parse_base(k1)
            return EngineKernel(fam, nu, k2.constant_value, ls, not k2.hyperparameter_constant_value.fixed,
                                not ls_fixed, False)
        raise NotImplementedError("only ConstantKernel * {Matern, RBF} products are supported")
    fam, nu, ls, ls_fixed = _parse_base(kernel)
    return EngineKernel(fam, nu, 1.0, ls, False, not ls_fixed, True)


def _find_transform_deep(kernel):
    """find_transform on the kernel itself or, for Product / Sum, on its operands."""
    t = find_transform(kernel)
    if t is None and isinstance(kernel, (Product, Sum)):
        t = _find_transform_deep(kernel.k1) or _find_transform_deep(kernel.k2)
    return t


def probe_transform(kernel, d):
    """bayes_opt's wrap_kernel (R/bayes_opt/parameter.py:457-495) stores the input transform on
    the kernel as ``_transform``.  The engine supports per-dimension identity / np.round; the
    transform is identified by probing it (it is an opaque callable)."""
    t = _find_transform_deep(kernel)
    if t is None:
        return None
    probe = np.array([[0.3 + j for j in range(d)], [1.7 - j for j in range(d)], [2.5 + j for j in range(d)]])
    out = np.asarray(t(probe.copy()), dtype=float)
    if out.shape != probe.shape:
        raise NotImplementedError(
            "kernel input transform changes the dimension (categorical one-hot) - not supported "
            "by the device engine yet")
    codes = np.zeros(d, dtype=np.int32)
    for j in range(d):
        if np.array_equal(out[:, j], probe[:, j]):
            codes[j] = B.XFORM_IDENTITY
        elif np.array_equal(out[:, j], np.round(probe[:, j])):
            codes[j] = B.XFORM_ROUND
        else:
            raise NotImplementedError("unsupported kernel input transform on dimension %d" % j)
    return None if not codes.any() else codes


def resolve_transform(kernel, d):
    """How the kernel's input transform is applied:
      ("device", codes|None)  per-dimension identity / np.round, done inside the CUDA kernels;
      ("host", fn)            any other transform (e.g. the reference's categorical one-hot, which is
                              batch-dependent: R/bayes_opt/parameter.py:434-449) - the opaque Python
                              callable is applied to the batch on the host exactly where the reference
                              applies it (WrappedKernel.__call__, parameter.py:484-487) and the device
                              sees the transformed coordinates."""
    t = _find_transform_deep(kernel)
    if t is None:
        return "device", None
    try:
        return "device", probe_transform(kernel, d)
    except NotImplementedError:
        return "host", t


def apply_transform(mode, arg, X):
    if mode == "host":
        return B.c_f64(np.asarray(arg(X), dtype=np.float64))
    return X


def to_b200_gp(gp, device=0, devices=None, precision="fp64"):
    """A B200GaussianProcessRegressor with the hyper-parameters, kernel object and RandomState of a
    sklearn GaussianProcessRegressor (the object the reference builds privately)."""
    if isinstance(gp, B200GaussianProcessRegressor):
        return gp
    return B200GaussianProcessRegressor(device=device, devices=devices, precision=precision,
                                        **gp.get_params(deep=False))


# restart-worker handles, shared per device (see fit); release_worker_pool() frees them
_POOL_LOCK = threading.Lock()
_POOLS = {}


def release_worker_pool():
    """Free the device memory held by the shared restart-worker handles (they are re-created on demand)."""
    with _POOL_LOCK:
        _POOLS.clear()


class _Handle:
    """Owns one b200bo_gp*."""

    def __init__(self, device):
        self.ptr = C.c_void_p()
        B.check(B.lib().b200bo_gp_create(C.byref(self.ptr), int(device)))

    def __del__(self):
        try:
            if self.ptr:
                B.lib().b200bo_gp_destroy(self.ptr)
                self.ptr = C.c_void_p()
        except Exception:  # interpreter shutdown
            pass


class B200GaussianProcessRegressor(GaussianProcessRegressor):
    """GaussianProcessRegressor whose numerics run on an H100 (fp64).

    Same constructor as sklearn's plus ``device`` (CUDA ordinal of the fit), ``devices`` (optional list of
    ordinals: the fitted state is replicated there and large acquisition batches / the L-BFGS-B seeds are
    sharded over them, SURVEY.md 8e) and ``precision``: "fp64" (exact,
    parity 1e-5, default) or "fp32" (the N^2 term of predict on wgmma tensor cores as 3xTF32 with
    fp32 accumulation; fit, K*, the mean and the acquisition epilogue stay fp64; tolerance 1e-3).  ``fit`` mirrors
    SK/gaussian_process/_gpr.py:233-368 (incl. the 1 + n_restarts_optimizer L-BFGS-B runs and the
    exact RandomState draws at :328-333); ``predict`` mirrors :370-500 for return_std;
    ``log_marginal_likelihood`` mirrors :541-656.
    """

    def __init__(self, kernel=None, *, alpha=1e-10, optimizer="fmin_l_bfgs_b", n_restarts_optimizer=0,
                 normalize_y=False, copy_X_train=True, n_targets=None, random_state=None, device=0,
                 precision="fp64", devices=None):
        super().__init__(kernel=kernel, alpha=alpha, optimizer=optimizer,
                         n_restarts_optimizer=n_restarts_optimizer, normalize_y=normalize_y,
                         copy_X_train=copy_X_train, n_targets=n_targets, random_state=random_state)
        self.device = device
        self.precision = precision
        self.devices = devices  # optional list of CUDA ordinals: predict/acquisition batches shard over them

    # ---- device plumbing -----------------------------------------------------------------
    def _handle(self) -> _Handle:
        h = self.__dict__.get("_b200_handle")
        if h is None:
            h = _Handle(self.device)
            self.__dict__["_b200_handle"] = h
        return h

    def __getstate__(self):
        state = super().__getstate__() if hasattr(super(), "__getstate__") else self.__dict__.copy()
        state = dict(state)
        state.pop("_b200_handle", None)
        state.pop("_b200_restart_handles", None)
        state.pop("_b200_replicas", None)
        state.pop("_b200_noiseless", None)
        state["_b200_device_fitted"] = False
        return state

    def _ensure_device_fit(self):
        """After unpickling / deepcopy the device factor is gone: rebuild it at kernel_.theta (a GP conditioned on
        pending points: the fit on the registered rows, then the conditioning on the pending ones)."""
        if not self.__dict__.get("_b200_device_fitted", False):
            if not hasattr(self, "X_train_"):
                raise B.B200Error("GP is not fitted")
            n_reg = self.__dict__.get("_b200_conditioned")
            if n_reg is None:
                self._device_fit(parse_kernel(self.kernel_))
                return
            self._device_fit(parse_kernel(self.kernel_), self.X_train_[:n_reg], self._y_raw[:n_reg])
            pending = B.c_f64(self.X_train_[n_reg:])
            if -(-n_reg // 128) * 128 < self.X_train_.shape[0]:  # no slack for the pending rows: fork
                self.__dict__["_b200_handle"] = self._fork_handle(pending.shape[0])
            B.check(B.lib().b200bo_gp_condition(self._handle().ptr, B.as_dp(pending), pending.shape[0], None))

    def _bare_copy(self):
        """A new regressor with this one's fitted attributes and none of its device state (handles, replicas, cached
        factor reads, the noiseless regressor of NEI)."""
        out = type(self).__new__(type(self))
        skip = ("_b200_handle", "_b200_restart_handles", "_b200_replicas", "_b200_L", "_b200_alpha", "_b200_noiseless")
        out.__dict__.update({k: v for k, v in self.__dict__.items() if k not in skip})
        return out

    def _fork_handle(self, extra_rows):
        h = _Handle.__new__(_Handle)
        h.ptr = C.c_void_p()
        B.check(B.lib().b200bo_gp_fork(self._handle().ptr, int(extra_rows), C.byref(h.ptr)))
        return h

    def _device_fit(self, ek: EngineKernel, X_train=None, y_raw=None):
        h = self._handle()
        X_train = self.X_train_ if X_train is None else X_train
        y = B.c_f64(self._y_raw if y_raw is None else y_raw)
        mode, arg = resolve_transform(self.kernel_, X_train.shape[1])
        self.__dict__["_b200_xform"] = (mode, arg)
        X = apply_transform(mode, arg, B.c_f64(X_train))
        d = X.shape[1]
        codes = arg if mode == "device" else None
        L = B.lib()
        if codes is not None:
            B.check(L.b200bo_gp_set_transform(h.ptr, codes.ctypes.data_as(C.POINTER(C.c_int32)), d))
        else:
            B.check(L.b200bo_gp_set_transform(h.ptr, None, d))
        spec = ek.c_spec()
        info = C.c_int64(0)
        rc = L.b200bo_gp_fit(h.ptr, B.as_dp(X), B.as_dp(y), X.shape[0], d, C.byref(spec),
                             float(self.alpha), int(bool(self.normalize_y)), C.byref(info))
        B.check(rc)
        if self.precision not in ("fp64", "fp32"):
            raise ValueError("precision must be 'fp64' or 'fp32'")
        B.check(L.b200bo_gp_set_precision(h.ptr, B.PRECISION_FP32 if self.precision == "fp32" else B.PRECISION_FP64))
        self.__dict__["_b200_fit_sig"] = self._fit_signature(ek)
        self.__dict__["_b200_device_fitted"] = True
        self.__dict__.pop("_b200_L", None)
        self.__dict__.pop("_b200_alpha", None)
        self.__dict__.pop("_b200_replicas", None)

    def device_list(self):
        """CUDA ordinals this GP evaluates on: [device] or the ``devices`` option (fit device first)."""
        if not self.devices:
            return [int(self.device)]
        devs = [int(x) for x in self.devices]
        if int(self.device) in devs:
            devs.remove(int(self.device))
        return [int(self.device)] + devs

    def _device_handles(self):
        """One fitted handle per device of device_list(): the primary plus replicas of its fitted state
        (b200bo_gp_replicate: peer copies of Xs, L^-1, alpha_ over NVLink; no re-factorisation)."""
        self._ensure_device_fit()
        devs = self.device_list()
        main = self._handle()
        if len(devs) == 1:
            return [main]
        reps = self.__dict__.get("_b200_replicas")
        if reps is None or [d for d, _ in reps] != devs[1:]:
            reps = []
            for dv in devs[1:]:
                h = _Handle.__new__(_Handle)
                h.ptr = C.c_void_p()
                B.check(B.lib().b200bo_gp_replicate(main.ptr, int(dv), C.byref(h.ptr)))
                reps.append((dv, h))
            self.__dict__["_b200_replicas"] = reps
        return [main] + [h for _, h in reps]

    # sklearn exposes L_ and alpha_ as attributes; materialise them lazily from the device
    @property
    def L_(self):
        if "_b200_L" not in self.__dict__:
            self._ensure_device_fit()
            n = self.X_train_.shape[0]
            out = np.empty((n, n))
            B.check(B.lib().b200bo_gp_get(self._handle().ptr, B.GET_L, B.as_dp(out), n * n))
            self.__dict__["_b200_L"] = out
        return self.__dict__["_b200_L"]

    @L_.setter
    def L_(self, v):
        self.__dict__["_b200_L"] = v

    @property
    def alpha_(self):
        if "_b200_alpha" not in self.__dict__:
            self._ensure_device_fit()
            n = self.X_train_.shape[0]
            out = np.empty(n)
            B.check(B.lib().b200bo_gp_get(self._handle().ptr, B.GET_ALPHA, B.as_dp(out), n))
            self.__dict__["_b200_alpha"] = out
        return self.__dict__["_b200_alpha"]

    @alpha_.setter
    def alpha_(self, v):
        self.__dict__["_b200_alpha"] = v

    # ---- fit -------------------------------------------------------------------------------
    def fit(self, X, y):
        """SK/gaussian_process/_gpr.py:233-368 with the arithmetic on the device."""
        if self.kernel is None:
            self.kernel_ = ConstantKernel(1.0, constant_value_bounds="fixed") * RBF(
                1.0, length_scale_bounds="fixed")
        else:
            self.kernel_ = clone(self.kernel)
        self._rng = check_random_state(self.random_state)
        X = np.array(X, dtype=np.float64, copy=True)
        if X.ndim != 2:  # sklearn's validate_data rejects the same inputs
            raise ValueError(f"Expected 2D array, got {X.ndim}D array instead: reshape your data with "
                             "array.reshape(-1, 1) for a single feature or array.reshape(1, -1) for a single sample.")
        y = np.asarray(y, dtype=np.float64)
        if y.ndim == 2 and y.shape[1] == 1:
            y = y[:, 0]
        if y.ndim != 1:
            raise NotImplementedError("multi-output targets are not supported by the device engine")
        if X.shape[0] != y.shape[0]:
            raise ValueError("X and y have inconsistent numbers of samples")
        if not (np.all(np.isfinite(X)) and np.all(np.isfinite(y))):
            raise ValueError("Input contains NaN or infinity.")
        if np.iterable(self.alpha):
            raise NotImplementedError("per-sample alpha is not supported by the device engine")
        self.n_features_in_ = X.shape[1]
        self.__dict__.pop("_b200_conditioned", None)
        ek = parse_kernel(self.kernel_)  # raises NotImplementedError for unsupported kernels
        if ek.length_scale.size not in (1, X.shape[1]):
            raise ValueError("Anisotropic kernel must have the same number of dimensions as data "
                             f"({ek.length_scale.size}!={X.shape[1]})")

        # normalisation statistics exactly as sklearn computes them (:275-285)
        if self.normalize_y:
            self._y_train_mean = np.mean(y, axis=0)
            s = np.std(y, axis=0)
            self._y_train_std = 1.0 if s == 0.0 else s
            y_norm = (y - self._y_train_mean) / self._y_train_std
        else:
            self._y_train_mean = np.zeros(1)
            self._y_train_std = np.ones(1)
            y_norm = y
        prev = None
        if self.__dict__.get("_b200_device_fitted", False) and hasattr(self, "_y_raw"):
            prev = (self.X_train_, self._y_raw, self.__dict__.get("_b200_fit_sig"))
        self.X_train_ = X
        self.y_train_ = y_norm
        self._y_raw = y.copy()
        self.__dict__["_b200_device_fitted"] = False

        if self.optimizer is not None and self.kernel_.n_dims > 0:
            h = self._handle()
            L = B.lib()
            mode, arg = resolve_transform(self.kernel_, X.shape[1])
            Xd = apply_transform(mode, arg, B.c_f64(X))
            codes = arg if mode == "device" else None
            B.check(L.b200bo_gp_set_transform(
                h.ptr, codes.ctypes.data_as(C.POINTER(C.c_int32)) if codes is not None else None,
                Xd.shape[1]))
            B.check(L.b200bo_gp_set_data(h.ptr, B.as_dp(Xd), B.as_dp(B.c_f64(y)), Xd.shape[0], Xd.shape[1],
                                         int(bool(self.normalize_y))))

            def make_obj(handle):
                def obj_func(theta, eval_gradient=True):
                    if eval_gradient:
                        lml, grad = self._device_lml(ek.with_theta(theta), True, handle)
                        return -lml, -grad
                    return -self._device_lml(ek.with_theta(theta), False, handle)

                return obj_func

            # the 1 + n_restarts_optimizer starting points (:321-340); the restarts' thetas are drawn
            # from self._rng in the reference's order - the draws do not depend on the optimisations
            bounds = self.kernel_.bounds
            starts = [self.kernel_.theta]
            if self.n_restarts_optimizer > 0:
                if not np.isfinite(bounds).all():
                    raise ValueError("Multiple optimizer restarts (n_restarts_optimizer>0) "
                                     "requires that all bounds are finite.")
                for _ in range(self.n_restarts_optimizer):
                    starts.append(self._rng.uniform(bounds[:, 0], bounds[:, 1]))
            # worker handles (5 N^2 doubles + a captured CUDA graph each) come from ONE pool per device shared by
            # every GP of the process (target + constraint GPs fit one after the other), not one pool per GP
            locked = _POOL_LOCK.acquire(blocking=False)
            try:
                workers = None
                if locked:
                    try:
                        workers = self._restart_workers(len(starts), Xd, y, codes)
                    except B.B200Error:  # e.g. out of memory for the worker buffers: sequential loop
                        _POOLS.pop(int(self.device), None)
                        L.b200bo_gp_set_private_stream(h.ptr, 0)
                if workers is None:
                    obj_func = make_obj(h)
                    optima = [self._constrained_optimization(obj_func, t0, bounds) for t0 in starts]
                else:
                    optima = self._run_restarts_concurrently(workers, make_obj, starts, bounds)
            finally:
                if locked:
                    _POOL_LOCK.release()
            lml_values = list(map(itemgetter(1), optima))
            self.kernel_.theta = optima[np.argmin(lml_values)][0]
            self.kernel_._check_bounds_params()
            self.log_marginal_likelihood_value_ = -np.min(lml_values)
            ek = parse_kernel(self.kernel_)
            self._device_fit(ek)
        else:
            if not self._try_incremental(prev, X, y, ek):
                self._device_fit(ek)
            self.__dict__["_b200_lml_value"] = None  # computed on first access (one more factorisation)
        return self

    # sklearn always leaves a float here; with optimizer=None it costs one extra factorisation, so the
    # value is produced on first access instead of inside every fit()
    @property
    def log_marginal_likelihood_value_(self):
        v = self.__dict__.get("_b200_lml_value")
        if v is None and hasattr(self, "X_train_"):
            v = self.log_marginal_likelihood(self.kernel_.theta, clone_kernel=True)
            self.__dict__["_b200_lml_value"] = v
        return v

    @log_marginal_likelihood_value_.setter
    def log_marginal_likelihood_value_(self, v):
        self.__dict__["_b200_lml_value"] = v

    # ---- concurrent restarts -----------------------------------------------------------------
    _MAX_RESTART_WORKERS = 8
    _RESTART_POOL_BYTES = 24 << 30
    _RESTART_MIN_N = 192  # below this an LML evaluation is ~0.3 ms: worker handles cost more than they save

    def _restart_workers(self, n_starts, Xd, y, codes):
        """Handles for running the independent L-BFGS-B starts concurrently (one host thread + one
        CUDA stream + one set of factor buffers each), or None for the sequential loop.  An LML
        evaluation at these sizes is a chain of ~200 dependent launches that leaves most SMs idle;
        several chains in flight fill them.  Every run sees exactly the objective values it would see
        alone, so the optima are those of the sequential loop.  B200BO_PARALLEL_RESTARTS=0 disables."""
        if n_starts < 2 or self.optimizer != "fmin_l_bfgs_b" or Xd.shape[0] < self._RESTART_MIN_N:
            return None
        if os.environ.get("B200BO_PARALLEL_RESTARTS", "1") == "0":
            return None
        n_workers = min(n_starts, self._MAX_RESTART_WORKERS)
        npad = -(-Xd.shape[0] // 128) * 128
        if (n_workers - 1) * 5 * 8 * npad * npad > self._RESTART_POOL_BYTES:
            return None
        L = B.lib()
        pool = _POOLS.setdefault(int(self.device), [])
        while len(pool) < n_workers - 1:
            pool.append(_Handle(self.device))
        handles = [self._handle()] + pool[:n_workers - 1]
        yc = B.c_f64(y)
        for i, hd in enumerate(handles):
            B.check(L.b200bo_gp_set_private_stream(hd.ptr, 1))
            if i == 0:
                continue  # the main handle already holds the data
            B.check(L.b200bo_gp_set_transform(
                hd.ptr, codes.ctypes.data_as(C.POINTER(C.c_int32)) if codes is not None else None, Xd.shape[1]))
            B.check(L.b200bo_gp_set_data(hd.ptr, B.as_dp(Xd), B.as_dp(yc), Xd.shape[0], Xd.shape[1],
                                         int(bool(self.normalize_y))))
        return handles

    def _run_restarts_concurrently(self, handles, make_obj, starts, bounds):
        results, errors = [None] * len(starts), []
        lock = threading.Lock()
        nxt = [0]

        def work(handle):
            obj = make_obj(handle)
            while True:
                with lock:
                    i = nxt[0]
                    nxt[0] += 1
                if i >= len(starts) or errors:
                    return
                try:
                    results[i] = self._constrained_optimization(obj, starts[i], bounds)
                except BaseException as e:  # re-raised in the calling thread
                    errors.append(e)
                    return

        threads = [threading.Thread(target=work, args=(hd,), daemon=True) for hd in handles]
        try:
            for t in threads:
                t.start()
            for t in threads:
                t.join()
        finally:
            B.lib().b200bo_gp_set_private_stream(handles[0].ptr, 0)  # main handle back on the default stream
        if errors:
            raise errors[0]
        return results

    def _try_incremental(self, prev, X, y, ek):
        """Fixed hyper-parameters (optimizer=None) and the new training set = the previous one plus
        appended rows: extend the device factor in O(N^2) per row instead of re-factorising
        (SURVEY.md 8f rank 3).  Same results as a from-scratch fit to round-off."""
        if prev is None or self.__dict__.get("_b200_handle") is None:
            return False
        Xp, yp, sig = prev
        k = X.shape[0] - Xp.shape[0]
        if not (0 < k <= 8) or X.shape[1] != Xp.shape[1] or sig != self._fit_signature(ek):
            return False
        if not (np.array_equal(X[:-k], Xp) and np.array_equal(y[:-k], yp)):
            return False
        mode, arg = resolve_transform(self.kernel_, X.shape[1])
        if mode != "device":
            return False
        L = B.lib()
        h = self._handle()
        for i in range(Xp.shape[0], X.shape[0]):
            info = C.c_int64(0)
            rc = L.b200bo_gp_append(h.ptr, B.as_dp(B.c_f64(X[i])), float(y[i]), C.byref(info))
            if rc == B.ERR_STATE:
                return False  # capacity exhausted: full refit
            B.check(rc)
        self.__dict__["_b200_xform"] = (mode, arg)
        self.__dict__["_b200_device_fitted"] = True
        self.__dict__.pop("_b200_L", None)
        self.__dict__.pop("_b200_alpha", None)
        return True

    def _fit_signature(self, ek):
        return (ek.family, ek.nu, ek.const_value, tuple(ek.length_scale.tolist()), ek.noise, float(self.alpha),
                bool(self.normalize_y), self.precision)

    def _constrained_optimization(self, obj_func, initial_theta, bounds):
        """SK/gaussian_process/_gpr.py:658-674."""
        if self.optimizer == "fmin_l_bfgs_b":
            opt_res = scipy.optimize.minimize(obj_func, initial_theta, method="L-BFGS-B", jac=True,
                                              bounds=bounds)
            _check_optimize_result("lbfgs", opt_res)
            return opt_res.x, opt_res.fun
        if callable(self.optimizer):
            return self.optimizer(obj_func, initial_theta, bounds=bounds)
        raise ValueError(f"Unknown optimizer {self.optimizer}.")

    def _device_lml(self, ek: EngineKernel, eval_gradient, handle=None):
        h = handle if handle is not None else self._handle()
        spec = ek.c_spec()
        lml = C.c_double(0.0)
        ntheta_dev = (1 if ek.const_free else 0) + ek.length_scale.size + (1 if ek.noise_free else 0)
        grad = np.zeros(ntheta_dev)
        B.check(B.lib().b200bo_gp_lml(h.ptr, C.byref(spec), float(self.alpha),
                                      int(ek.const_free) | (2 if ek.noise_free else 0),
                                      C.byref(lml), B.as_dp(grad) if eval_gradient else None))
        self.__dict__["_b200_device_fitted"] = False  # factor buffers now hold this theta
        if eval_gradient:
            return lml.value, ek.select_grad(grad)
        return lml.value

    def log_marginal_likelihood(self, theta=None, eval_gradient=False, clone_kernel=True):
        """SK/gaussian_process/_gpr.py:541-656."""
        if theta is None:
            if eval_gradient:
                raise ValueError("Gradient can only be evaluated for theta!=None")
            return self.log_marginal_likelihood_value_
        if clone_kernel:
            kernel = self.kernel_.clone_with_theta(theta)
        else:
            kernel = self.kernel_
            kernel.theta = theta
        h = self._handle()
        mode, arg = resolve_transform(self.kernel_, self.X_train_.shape[1])
        X = apply_transform(mode, arg, B.c_f64(self.X_train_))
        codes = arg if mode == "device" else None
        L = B.lib()
        B.check(L.b200bo_gp_set_transform(
            h.ptr, codes.ctypes.data_as(C.POINTER(C.c_int32)) if codes is not None else None, X.shape[1]))
        B.check(L.b200bo_gp_set_data(h.ptr, B.as_dp(X), B.as_dp(B.c_f64(self._y_raw)), X.shape[0],
                                     X.shape[1], int(bool(self.normalize_y))))
        out = self._device_lml(parse_kernel(kernel), eval_gradient)
        return out

    # ---- predict ---------------------------------------------------------------------------
    def predict(self, X, return_std=False, return_cov=False):
        """SK/gaussian_process/_gpr.py:370-500 (return_std path) on the device."""
        if return_std and return_cov:
            raise RuntimeError("At most one of return_std or return_cov can be requested.")
        X = np.array(X, dtype=np.float64)
        if X.ndim != 2:
            raise ValueError(f"Expected 2D array, got {X.ndim}D array instead: reshape your data with "
                             "array.reshape(-1, 1) for a single feature or array.reshape(1, -1) for a single sample.")
        if not np.all(np.isfinite(X)):
            raise ValueError("Input contains NaN or infinity.")
        if not hasattr(self, "X_train_"):  # unfitted: GP prior (:417-443), no device work to do
            if self.kernel is None:
                kernel = ConstantKernel(1.0, constant_value_bounds="fixed") * RBF(
                    1.0, length_scale_bounds="fixed")
            else:
                kernel = self.kernel
            y_mean = np.zeros(X.shape[0])
            if return_cov:
                return y_mean, kernel(X)
            if return_std:
                return y_mean, np.sqrt(kernel.diag(X))
            return y_mean
        if X.shape[1] != self.X_train_.shape[1]:
            raise ValueError(f"X has {X.shape[1]} features, but the GP was fitted with "
                             f"{self.X_train_.shape[1]} features.")
        self._ensure_device_fit()
        Xc = self._device_candidates(B.c_f64(X))
        m = Xc.shape[0]
        if return_cov:  # :464-475, device: K(X*,X*) - V^T V
            mu = np.empty(m)
            cov = np.empty((m, m))
            B.check(B.lib().b200bo_gp_predict_cov(self._handle().ptr, B.as_dp(Xc), m, B.as_dp(mu), B.as_dp(cov)))
            return mu, cov
        mu = np.empty(m)
        sd = np.empty(m) if return_std else None
        nclamp = C.c_int64(0)
        B.check(B.lib().b200bo_gp_predict(self._handle().ptr, B.as_dp(Xc), m, B.as_dp(mu),
                                          B.as_dp(sd) if return_std else None, C.byref(nclamp)))
        if return_std:
            if nclamp.value > 0:
                warnings.warn("Predicted variances smaller than 0. Setting those variances to 0.")
            return mu, sd
        return mu

    # ---- Kriging believer --------------------------------------------------------------------
    def condition_on_pending(self, X, extra_rows=0):
        """The GP conditioned on pending points ``X`` (n_pending, d) whose values are not known yet, each with the
        Kriging-believer target: the posterior mean mu(x) (Ginsbourger, Le Riche & Carraro 2010; DESIGN.md 4.11).
        The hyper-parameters and the y normalisation stay those of the fit, so the posterior mean is unchanged
        everywhere and the standard deviation shrinks near the pending points - the whole effect of the fantasy.
        One O(N^2) row update per point (``b200bo_gp_condition``); nothing is refitted.

        Returns a fitted regressor: ``X_train_`` is the augmented set, ``y_train_`` / ``_y_raw`` end with the believer
        values, ``kernel_`` is this GP's.  On a GP that is not itself conditioned, the result is a new object on a
        fork of the device state (``b200bo_gp_fork``) and this GP is untouched; on a conditioned GP the call
        conditions in place (and returns self) while the device capacity holds the rows, and forks otherwise.
        ``extra_rows`` reserves capacity in a fork for that many later in-place calls.  Multi-device GPs and
        host-side (categorical) input transforms raise NotImplementedError; a non-positive pivot raises
        np.linalg.LinAlgError, as ``fit`` does."""
        X = np.array(X, dtype=np.float64)
        if X.ndim == 1:
            X = X.reshape(1, -1)
        if X.ndim != 2 or not hasattr(self, "X_train_") or X.shape[1] != self.X_train_.shape[1]:
            raise ValueError("X must be (n_pending, d) with the d of a fitted GP")
        if not np.all(np.isfinite(X)):
            raise ValueError("Input contains NaN or infinity.")
        if isinstance(extra_rows, bool) or not isinstance(extra_rows, (int, np.integer)) or extra_rows < 0:
            raise ValueError(f"extra_rows must be an integer >= 0, got {extra_rows!r}")
        if len(self.device_list()) > 1:
            raise NotImplementedError("conditioning on pending points runs on one device: the GP is multi-device")
        self._ensure_device_fit()
        if self.__dict__.get("_b200_xform", ("device", None))[0] == "host":
            raise NotImplementedError("conditioning on pending points with a host-side (categorical) kernel transform")
        n, p = self.X_train_.shape[0], X.shape[0]
        n_reg = self.__dict__.get("_b200_conditioned")
        mu = np.empty(p)
        Xc = B.c_f64(X)
        L = B.lib()
        out = self
        # in place on a conditioned GP; B200BO_ERR_STATE (checked before any work) means no slack left: fork
        rc = L.b200bo_gp_condition(self._handle().ptr, B.as_dp(Xc), p, B.as_dp(mu)) if n_reg is not None else B.ERR_STATE
        if rc == B.ERR_STATE:
            out = self._bare_copy()
            out.__dict__["_b200_handle"] = self._fork_handle(p + int(extra_rows))
            out.__dict__["_b200_conditioned"] = n if n_reg is None else n_reg
            rc = L.b200bo_gp_condition(out._handle().ptr, B.as_dp(Xc), p, B.as_dp(mu))
        if rc != B.OK:
            out.__dict__["_b200_device_fitted"] = False  # rebuilt from X_train_ on the next use
        B.check(rc)
        out.X_train_ = np.vstack([self.X_train_, Xc])
        out.y_train_ = np.concatenate([self.y_train_, (mu - self._y_train_mean) / self._y_train_std])
        out._y_raw = np.concatenate([self._y_raw, mu])
        out.__dict__.pop("_b200_L", None)
        out.__dict__.pop("_b200_alpha", None)
        return out

    def _device_candidates(self, X):
        """Candidates as the device sees them (host-side transform applied when the kernel carries
        one the CUDA kernels do not implement)."""
        mode, arg = self.__dict__.get("_b200_xform", ("device", None))
        return apply_transform(mode, arg, X)

    # sample_y (SK/gaussian_process/_gpr.py:502-539) is inherited: it only calls
    # self.predict(X, return_cov=True), which runs on the device.

    def sample_paths(self, n_paths=1, n_features=4096, random_state=None):
        """``n_paths`` (1..16) posterior sample paths of the latent function, as smooth functions that can be
        evaluated anywhere (paths.PosteriorPaths): the prior part is a random-Fourier-feature draw with
        ``n_features`` features, the data update is exact.  The draws come from ``random_state``
        (``check_random_state``) in the order of ``paths.draw_path_inputs``.  The reference has no counterpart;
        unlike ``sample_y`` the cost per evaluated point does not grow with the number of points."""
        from .paths import PosteriorPaths

        return PosteriorPaths(self, n_paths, n_features, random_state)

    def noiseless_fantasies(self, n_samples, jitter=1e-6, incumbent=None, random_state=None, pending=None,
                            extra_rows=0):
        """S = ``n_samples`` (1..16) joint samples of the noise-free function values at the training inputs, for noisy
        expected improvement (DESIGN.md 4.13, ``b200bo_gp_set_fantasies``).

        The noiseless GP has this GP's inputs, hyper-parameters and y statistics, no WhiteKernel term and
        alpha = tau = min(alpha, jitter).  When the fitted noise variance sigma_n^2 = alpha + noise_level equals tau
        (no WhiteKernel, alpha <= jitter) it is this GP itself and nothing is factorised again; otherwise it is a second
        regressor on a device handle of its own, always in fp64.  From ``random_state`` (``check_random_state``) it
        draws Z = standard_normal((n, S)), then E = standard_normal((n, S)).  ``incumbent`` is the (n,) mask of the
        rows whose fantasy values may be the incumbent best_s (all rows when None).  Returns a ``NoiselessFantasies``.

        ``pending`` ((p, d), points suggested and not yet registered) and ``extra_rows`` (room for that many later
        ``NoiselessFantasies.condition_on_pending`` rows) draw the values at pending points jointly with the fantasies
        (DESIGN.md 4.14, ``b200bo_gp_condition_fantasies``): after Z and E, ``standard_normal((p + extra_rows, S))``;
        then the noiseless regressor is forked with that capacity and the fork is conditioned on ``pending``.  This GP
        and the noiseless regressor are never modified.  With neither argument nothing is forked or drawn beyond Z, E.
        One device (multi-device GPs raise NotImplementedError, and with pending rows so do host-side, categorical,
        input transforms); a non-PD K0 or pending pivot raises np.linalg.LinAlgError naming ``jitter``."""
        S = int(n_samples)
        if isinstance(n_samples, bool) or S != n_samples or not 1 <= S <= B.MAX_PATHS:
            raise ValueError(f"n_samples must be an integer in [1, {B.MAX_PATHS}], got {n_samples!r}")
        jitter = float(jitter)
        if not jitter > 0.0 or not np.isfinite(jitter):
            raise ValueError(f"jitter must be a positive float, got {jitter!r}")
        if not hasattr(self, "X_train_"):
            raise B.B200Error("GP is not fitted")
        if len(self.device_list()) > 1:
            raise NotImplementedError("noisy expected improvement runs on one device: the GP is multi-device")
        if self.__dict__.get("_b200_conditioned") is not None:
            raise NotImplementedError("noisy expected improvement on a GP conditioned on pending points")
        if isinstance(extra_rows, bool) or not isinstance(extra_rows, (int, np.integer)) or extra_rows < 0:
            raise ValueError(f"extra_rows must be an integer >= 0, got {extra_rows!r}")
        d = self.X_train_.shape[1]
        P = np.empty((0, d)) if pending is None else np.array(pending, dtype=np.float64)
        if P.ndim == 1 and P.size == d:
            P = P.reshape(1, d)
        if P.size == 0:
            P = P.reshape(0, d)
        if P.ndim != 2 or P.shape[1] != d:
            raise ValueError("pending must be (n_pending, d) with the d of the fitted GP")
        if not np.all(np.isfinite(P)):
            raise ValueError("Input contains NaN or infinity.")
        rows = P.shape[0] + int(extra_rows)
        n = self.X_train_.shape[0]
        mask = np.ones(n, dtype=np.uint8) if incumbent is None else np.asarray(incumbent, dtype=bool).astype(np.uint8)
        if mask.shape != (n,):
            raise ValueError(f"incumbent must be a mask of the {n} training rows")
        if not mask.any():
            raise ValueError("the incumbent mask selects no training row")
        self._ensure_device_fit()
        if rows and self.__dict__.get("_b200_xform", ("device", None))[0] == "host":
            raise NotImplementedError("pending points for noisy expected improvement with a host-side (categorical) "
                                      "kernel transform")
        ek = parse_kernel(self.kernel_)
        alpha = float(self.alpha)
        tau = min(alpha, jitter)
        rs = check_random_state(random_state)
        Z = B.c_f64(rs.standard_normal((n, S)))
        E = B.c_f64(rs.standard_normal((n, S)))
        Zp = B.c_f64(rs.standard_normal((rows, S))) if rows else None
        if ek.noise == 0.0 and tau == alpha:
            nl = self
        else:
            # one noiseless regressor per GP, refitted in place: b200bo_gp_fit on the same handle reuses its device
            # buffers, so at most two N^2 handles (this GP's and the noiseless one) are ever live for NEI
            nl = self.__dict__.get("_b200_noiseless")
            handle = nl._handle() if nl is not None and nl.device == self.device else _Handle(self.device)
            nl = self._bare_copy()
            nl.__dict__["_b200_handle"] = handle
            self.__dict__["_b200_noiseless"] = nl
            nl.alpha = tau
            nl.precision = "fp64"
            # kernel_ stays this GP's (its input transform is found there); the fit drops the WhiteKernel term
            ek0 = parse_kernel(self.kernel_)
            ek0.noise = 0.0
            try:
                nl._device_fit(ek0)
            except np.linalg.LinAlgError as e:
                raise np.linalg.LinAlgError(f"{e} (noiseless GP with tau = {tau!r}: raise jitter)") from None
        F = np.empty((n, S))
        best = np.empty(S)
        B.check(B.lib().b200bo_gp_set_fantasies(nl._handle().ptr, self._handle().ptr, B.as_dp(Z), B.as_dp(E), S,
                                                mask.ctypes.data_as(C.POINTER(C.c_uint8)), B.as_dp(F), B.as_dp(best)))
        fant = NoiselessFantasies(nl, F, best, tau)
        if rows:
            # the fork's X_train_ grows with the pending rows (NoiselessFantasies.condition_on_pending) while its
            # targets stay the registered ones: it holds fantasies for NEI and is never refitted
            fork = nl._bare_copy()
            fork.__dict__["_b200_handle"] = nl._fork_handle(rows)
            fork.__dict__["_b200_conditioned"] = n
            fant.gp, fant._zp, fant._next = fork, Zp, 0
            fant.condition_on_pending(P)
        return fant


class NoiselessFantasies:
    """S joint samples of the noise-free function values at the training inputs (``noiseless_fantasies``).

    gp    the noiseless regressor holding A = K0^-1 F on its device handle (the fitted GP itself when tau = sigma_n^2);
          with pending points a fork of it whose ``X_train_`` ends with the pending rows
    F     (n, S) fantasy values, data units ((n + p, S) with p pending rows)
    best  (S,) best_s, the largest fantasy value over the incumbent rows
    tau   the noiseless GP's diagonal term"""

    def __init__(self, gp, F, best, tau):
        self.gp, self.F, self.best, self.tau = gp, F, best, tau
        self._zp, self._next = None, 0  # pre-drawn z rows of pending points, and the next one to use

    def condition_on_pending(self, X):
        """Extends the fantasies in place to the pending points ``X`` ((p, d) or (d,)): their values are drawn jointly
        with the fantasies from the next p of the z rows ``noiseless_fantasies(pending=..., extra_rows=...)`` drew
        (``b200bo_gp_condition_fantasies``).  F gains p rows and best may rise: pending rows count toward the incumbent.
        More rows than were drawn raise ValueError; a non-positive pivot raises np.linalg.LinAlgError naming jitter."""
        X = B.c_f64(np.asarray(X, dtype=np.float64).reshape(-1, self.gp.X_train_.shape[1]))
        p = X.shape[0]
        if self._zp is None or self._next + p > self._zp.shape[0]:
            left = 0 if self._zp is None else self._zp.shape[0] - self._next
            raise ValueError(f"{p} pending rows, {left} pre-drawn z rows left: pass pending / extra_rows to "
                             "noiseless_fantasies")
        if not np.all(np.isfinite(X)):
            raise ValueError("Input contains NaN or infinity.")
        zp = B.c_f64(self._zp[self._next:self._next + p])
        f = np.empty((p, self.n_samples))
        best = np.empty(self.n_samples)
        rc = B.lib().b200bo_gp_condition_fantasies(self.handle.ptr, B.as_dp(X), p, B.as_dp(zp), B.as_dp(f),
                                                   B.as_dp(best))
        if rc == B.ERR_NOT_PD:
            msg = B.lib().b200bo_last_error().decode("utf-8", "replace")
            raise np.linalg.LinAlgError(f"{msg} (noiseless GP with tau = {self.tau!r} at a pending point: raise "
                                        "jitter)")
        B.check(rc)
        self._next += p
        self.gp.X_train_ = np.vstack([self.gp.X_train_, X])
        self.F = np.vstack([self.F, f])
        self.best = best

    @property
    def n_samples(self):
        return self.best.size

    @property
    def handle(self):
        return self.gp._handle()

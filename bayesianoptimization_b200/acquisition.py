"""Acquisition seam of the drop-in boundary (SURVEY.md 8b.2).

The reference's plugin point is ``BayesianOptimization(acquisition_function=...)``: a subclass of
``bayes_opt.acquisition.AcquisitionFunction`` controls ``_get_acq``, ``_random_sample_minimize`` and
``_smart_minimize`` (R/bayes_opt/acquisition.py:171-219, :274-320, :322-420).  This module plugs the device
engine in at exactly those three hooks and nothing else: the classes below ARE the reference's classes
(``bayes_opt`` is imported, not restated - constructors, ``suggest``, decay schedules, parameter
get/set, ConstantLiar's dummy bookkeeping, GPHedge's portfolio logic and every error message are
inherited), with ``DeviceHooks`` mixed in:

  _get_acq                 -> FusedAcquisition: the whole closure is ONE fused kernel launch
  _random_sample_minimize  -> candidates from the caller's RandomState exactly as the reference draws
                              them, evaluation + argmin + top-n_smart selection on the device(s)
  _smart_minimize          -> the n_smart L-BFGS-B runs advanced in lockstep, one device call per round
                              (mixed-integer spaces: the reference's own DE branch, unchanged, calling
                              the device closure)

``ThompsonSampling`` is a policy defined here rather than inherited: a posterior sample path per ``suggest()``,
ranked and refined through the same three hooks.  ``ConstrainedThompsonSampling`` extends it to constrained problems
(the paths of the target and the constraint GPs, ranked feasible-first); ``suggest_batch`` proposes q points at once
from q paths (batch Thompson sampling).  ``MaxValueEntropySearch`` is the
information-based policy: samples of the maximum from posterior paths, then a fused-kernel epilogue of mu and sigma.
``KrigingBeliever`` gives UCB / EI / PoI / MES pending points and batches: the fitted GP is conditioned on the points in
flight on the device, with its own mean as their targets; ``PendingNEI`` does the same for noisy EI by drawing the
pending values jointly with its fantasies; ``ConstrainedNoisyExpectedImprovement`` adds fantasies of noisy constraints
and a sampled-feasibility incumbent.  ``LogExpectedImprovement`` and
``LogProbabilityOfImprovement`` are EI and PoI in log space, finite and well scaled where EI and PoI underflow.

``bayes_opt`` must be importable (this package is a plug-in for it).  The GP seam
(gpr.B200GaussianProcessRegressor), ``fused.FusedAcquisition`` and the C ABI do not need it.
"""
from __future__ import annotations

import abc
import ctypes as C
import warnings

import numpy as np
from scipy.special import erfcx as _erfcx
from scipy.special import log_ndtr as _log_ndtr
from scipy.special import ndtr as _ndtr

try:
    from bayes_opt import acquisition as _ref
    from bayes_opt.exception import ConstraintNotSupportedError as _ConstraintNotSupportedError
    from bayes_opt.exception import TargetSpaceEmptyError as _TargetSpaceEmptyError
    from bayes_opt.util import ensure_rng as _ensure_rng
except ImportError as e:  # pragma: no cover - depends on the environment
    raise ImportError(
        "bayesianoptimization_b200.acquisition plugs into the bayes_opt package "
        "(bayesian-optimization >= 3.0), which is not importable here: install it, or use "
        "B200GaussianProcessRegressor / FusedAcquisition / the C ABI directly") from e

from . import _lib as B
from .fused import FusedAcquisition, _as_b200_gp, lockstep_lbfgsb

_STOCK = {
    _ref.UpperConfidenceBound: B.ACQ_UCB,
    _ref.ExpectedImprovement: B.ACQ_EI,
    _ref.ProbabilityOfImprovement: B.ACQ_POI,
}


def _device_kind(obj):
    """Device epilogue code if ``obj.base_acq`` is one of the reference's three formulas, else None
    (a user subclass that overrides base_acq keeps its override: mu/sigma come from the device, the
    formula runs where the user wrote it)."""
    for cls, kind in _STOCK.items():
        if isinstance(obj, cls) and type(obj).base_acq is cls.base_acq:
            return kind
    return None


def _philox_seed(random_state):
    """The ONE 64-bit Philox key a device-generated candidate batch takes from the caller's RandomState: two 32-bit
    draws, the first the high word."""
    hi = int(random_state.randint(0, 2**32, dtype=np.uint64))
    return hi << 32 | int(random_state.randint(0, 2**32, dtype=np.uint64))


def _device_closure(acq):
    """True for closures that select and refine on the device: they map (M,d) -> (M,) and offer
    ``argmin_topk`` and ``argmin_topk_philox`` (optionally ``refine_mode``) - FusedAcquisition and the
    Thompson-sampling path closure (paths.PathAcquisition)."""
    return callable(getattr(acq, "argmin_topk", None)) and callable(getattr(acq, "argmin_topk_philox", None))


def _offers_grad(acq):
    """True for device closures with an analytic gradient: ``value_and_grad(x[, path_idx]) -> (values, gradients)``
    on one device (FusedAcquisition, the closures over unconstrained sample paths)."""
    return callable(getattr(acq, "value_and_grad", None)) and len(getattr(acq, "devices", [0])) == 1


class DeviceHooks(abc.ABC):
    """Mixin: the three hooks of the acquisition seam on the GPU.  Must precede the reference class in
    the MRO.  (Derives from abc.ABC like bayes_opt's AcquisitionFunction so that both have the same
    instance layout: a live reference object can then be re-classed in place, see ``accelerate``.)"""

    def _get_acq(self, gp, constraint=None):
        _as_b200_gp(gp)
        kind = _device_kind(self)
        if kind is None:
            acq = super()._get_acq(gp=gp, constraint=constraint)  # gp.predict / constraint.predict on device
            acq.b200_vectorized = True  # maps (M,d) -> (M,): lockstep batching is safe
            return acq
        return FusedAcquisition(kind, gp, constraint, owner=self)

    # "host_rng": the candidates are TargetSpace.random_sample's MT19937 stream (parity with the reference);
    # "device_philox": throughput mode - they are generated inside the fused kernel (continuous spaces only;
    # ONE 64-bit seed is drawn from the caller's RandomState per call).  Set by enable(candidate_source=...).
    b200_candidate_source = "host_rng"

    # "stencil": the L-BFGS-B refinement differentiates the closure by SciPy's 2-point scheme, d + 1 rows per
    # evaluation (parity with the reference); "analytic": it takes the gradient from the device, one row per
    # evaluation (continuous spaces, closures that offer value_and_grad; anything else stays on the stencil).
    # Set by enable(refine=...).
    b200_refine = "stencil"

    def _refine_grad(self, acq, space):
        return self.b200_refine == "analytic" and all(space.continuous_dimensions) and _offers_grad(acq)

    def _candidate_rows(self, space, n, random_state):
        """The host_rng candidates of the random stage: the reference's RNG stream (TrustRegionThompsonSampling: its
        trust-region source)."""
        return space.random_sample(n, random_state=random_state)

    def _select_philox(self, sel, seed, space, n, k):
        """The device_philox random stage of a closure or of q paths: ``argmin_topk_philox`` over the space's bounds
        (TrustRegionThompsonSampling: over its trust-region source)."""
        return sel.argmin_topk_philox(seed, space.bounds, n, k)

    def _random_sample_minimize(self, acq, space, random_state, n_random, n_x_seeds=0):
        if n_random == 0 or not _device_closure(acq):
            return super()._random_sample_minimize(acq, space, random_state, n_random, n_x_seeds)
        if (n_x_seeds <= B.MAX_TOPK and self.b200_candidate_source == "device_philox"
                and all(space.continuous_dimensions)):
            seed = _philox_seed(random_state)
            _, min_acq, x_min, _, x_seeds = self._select_philox(acq, seed, space, n_random, n_x_seeds)
            return x_min, min_acq, (x_seeds if n_x_seeds != 0 else [])
        x_tries = self._candidate_rows(space, n_random, random_state)
        if n_x_seeds > B.MAX_TOPK:
            # n_smart beyond the device's top-k capacity: evaluate on the device, select with numpy as the reference
            ys = acq(x_tries)
            return x_tries[ys.argmin()], ys.min(), x_tries[np.argsort(ys)[:n_x_seeds]]
        idx, min_acq, top = acq.argmin_topk(x_tries, n_x_seeds)
        return x_tries[idx], min_acq, (x_tries[top] if n_x_seeds != 0 else [])

    def _refine_bounds(self, space):
        """(d, 2) bounds of the L-BFGS-B refinement and of its clip: the space's (TrustRegionThompsonSampling: its
        trust region)."""
        return space.bounds

    def _smart_minimize(self, acq, space, x_seeds, random_state):
        bounds = self._refine_bounds(space)
        if len(x_seeds) != 0 and self._refine_grad(acq, space):
            runs = [r for r in lockstep_lbfgsb(acq, x_seeds, bounds, grad=True) if r.success]
            return self._best_run(runs, bounds)
        batched = _device_closure(acq) or getattr(acq, "b200_vectorized", False)
        refine = acq.refine_mode() if _device_closure(acq) and hasattr(acq, "refine_mode") else _null()
        with refine:
            if not batched or len(x_seeds) == 0 or not all(space.continuous_dimensions):
                return super()._smart_minimize(acq, space, x_seeds, random_state)
            runs = [r for r in lockstep_lbfgsb(acq, x_seeds, bounds) if r.success]
        return self._best_run(runs, bounds)

    @staticmethod
    def _best_run(runs, bounds):
        if not runs:
            return np.full(bounds.shape[0], np.nan), np.inf
        best = min(runs, key=lambda r: float(np.squeeze(r.fun)))  # first of equal minima, like the loop
        return np.clip(best.x, bounds[:, 0], bounds[:, 1]), np.squeeze(best.fun)


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


class AcquisitionFunction(DeviceHooks, _ref.AcquisitionFunction):
    """Base for user-defined acquisitions on the device GP: implement ``base_acq(mean, std)``."""


class UpperConfidenceBound(DeviceHooks, _ref.UpperConfidenceBound):
    """bayes_opt.acquisition.UpperConfidenceBound with the device hooks."""


class ProbabilityOfImprovement(DeviceHooks, _ref.ProbabilityOfImprovement):
    """bayes_opt.acquisition.ProbabilityOfImprovement with the device hooks."""


class ExpectedImprovement(DeviceHooks, _ref.ExpectedImprovement):
    """bayes_opt.acquisition.ExpectedImprovement with the device hooks."""


class PosteriorMean(DeviceHooks, _ref.AcquisitionFunction):
    """Maximise the posterior mean: the point a noisy run should recommend (Letham et al., Bayesian Analysis 2019),
    not a rule for what to evaluate next.  ``recommend(optimizer)`` uses it; it also works as an acquisition function.

    The closure is ``FusedAcquisition(ACQ_MEAN, gp, constraint)`` (include/b200bo.h, DESIGN.md 4.17): -mu of the target
    GP, and with constraints the merit "mu where every constraint's mean lies within its bounds, else -T (1 + the
    summed violation of the means)", so every mean-feasible point ranks above every infeasible one.  It is not a product
    of probabilities and needs no sigma: one mean-only kernel, without the L^-1 product the other kinds run.

    ``suggest`` is the reference's base ``suggest`` (random stage plus L-BFGS-B, the RandomState used as UCB uses it);
    it suggests before any feasible point is registered and never raises NoValidPointRegisteredError.  The acquisition
    params are empty, so ``save_state`` carries nothing extra.  A subclass that overrides ``base_acq(mean, std)`` gets
    the reference's closure on the device predict, as for the other classes.  ConstantLiar, GPHedge, KrigingBeliever and
    PendingNEI refuse it (TypeError)."""

    def base_acq(self, mean, std):
        return mean

    def _get_acq(self, gp, constraint=None):
        _as_b200_gp(gp)
        if type(self).base_acq is not PosteriorMean.base_acq:  # a host formula: the reference's closure
            acq = _ref.AcquisitionFunction._get_acq(self, gp=gp, constraint=constraint)
            acq.b200_vectorized = True
            return acq
        return FusedAcquisition(B.ACQ_MEAN, gp, constraint)

    def get_acquisition_params(self):
        return {}

    def set_acquisition_params(self, params):
        pass


# ---- log-space acquisitions (DESIGN.md 4.12) ------------------------------------------------------------------
# numpy forms of the device epilogue (csrc/common.cuh log_h, csrc/predict_kernels.cuh log_acq_term / log_cfactor),
# for user subclasses that override base_acq and for calls outside the fused kernel.
_LOG_H_TAIL = -(2.0**26)  # -1/sqrt(eps)
_HALF_LOG_2PI = 0.91893853320467274178
_HALF_LOG_PI_2 = 0.22579135264472743236


def log1mexp(x):
    """log(1 - exp(x)) for x <= 0: log(-expm1(x)) above -ln 2, log1p(-exp(x)) below."""
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(all="ignore"):
        return np.where(x > -np.log(2.0), np.log(-np.expm1(x)), np.log1p(-np.exp(x)))


def log_h(z):
    """log(phi(z) + z Phi(z)), the log of EI in units of sigma, in the three branches of Ament et al. (2023):
    direct above z = -1, through erfcx and log1mexp down to -1/sqrt(eps), the asymptote -z^2/2 - log(2 pi)/2 - 2 log|z|
    below."""
    z = np.asarray(z, dtype=np.float64)
    out = np.full(z.shape, np.nan)
    with np.errstate(all="ignore"):
        hi = z > -1.0
        mid = ~hi & (z > _LOG_H_TAIL)
        lo = ~hi & ~mid & ~np.isnan(z)
        t = z[hi]
        out[hi] = np.log(np.exp(-(t * t) / 2.0) / 2.50662827463100050242 + t * _ndtr(t))
        t = z[mid]
        out[mid] = (-0.5 * (t * t) - _HALF_LOG_2PI) + log1mexp(np.log(_erfcx(-t * np.sqrt(0.5)) * -t) + _HALF_LOG_PI_2)
        t = z[lo]
        out[lo] = (-0.5 * (t * t) - _HALF_LOG_2PI) - 2.0 * np.log(-t)
    return out


def log_expected_improvement(a, std):
    """log EI at a = mean - y_max - xi: log_h(a / std) + log std; std = 0 (or an infinite a / std) gives the log of the
    EI limit max(a, 0): log a, -inf for a < 0, NaN for a = 0."""
    a, std = np.broadcast_arrays(np.asarray(a, dtype=np.float64), np.asarray(std, dtype=np.float64))
    with np.errstate(all="ignore"):
        z = a / std
        lim = np.where(a > 0.0, np.log(np.where(a > 0.0, a, 1.0)), np.where(a < 0.0, -np.inf, np.nan))
        return np.where((std == 0.0) | np.isinf(z), lim, log_h(z) + np.log(std))


def log_constraint_factor(mean, std, lb, ub):
    """log P(lb <= c <= ub) for c ~ N(mean, std^2): one-sided bounds through log_ndtr, a pair of bounds in one tail
    reflected to the lower tail and combined through log1mexp, a straddling pair directly.  NaN where std <= 0 and a
    bound is finite (scipy's frozen norm), 0 when both bounds are infinite."""
    mean, std = np.broadcast_arrays(np.asarray(mean, dtype=np.float64), np.asarray(std, dtype=np.float64))
    lb, ub = float(lb), float(ub)
    if lb == -np.inf and ub == np.inf:
        return np.zeros(mean.shape)
    with np.errstate(all="ignore"):
        u, l = (ub - mean) / std, (lb - mean) / std
        if lb == -np.inf:
            out = _log_ndtr(u)
        elif ub == np.inf:
            out = _log_ndtr(-l)
        else:
            refl = l >= 0.0
            a, b = np.where(refl, -u, l), np.where(refl, -l, u)
            lpb = _log_ndtr(b)
            out = np.where((l < 0.0) & (u > 0.0), np.log(_ndtr(u) - _ndtr(l)), lpb + log1mexp(_log_ndtr(a) - lpb))
        return np.where((std > 0.0) & ~np.isnan(mean), out, np.nan)


class _LogSpace:
    """Mixin of the log-space acquisitions: the closure is -(base_acq(mean, std) + sum_j log p_j(x)), the constraint
    factors added in log space in constraint order (DeviceHooks runs the stock formulas in the fused kernel; this
    host closure serves a subclass that overrides base_acq)."""

    def _get_acq(self, gp, constraint=None):
        dim = gp.X_train_.shape[1]

        def acq(x):
            x = np.asarray(x, dtype=np.float64).reshape(-1, dim)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                mean, std = gp.predict(x, return_std=True)
                v = np.asarray(self.base_acq(mean, std), dtype=np.float64)
                if constraint is not None:
                    for j, m in enumerate(constraint.model):
                        cm, cs = m.predict(x, return_std=True)
                        v = v + log_constraint_factor(cm, cs, constraint.lb[j], constraint.ub[j])
            return -1 * v

        return acq


class LogExpectedImprovement(DeviceHooks, _LogSpace, _ref.ExpectedImprovement):
    """Log expected improvement (Ament et al., "Unexpected Improvements to Expected Improvement for Bayesian
    Optimization", NeurIPS 2023): log EI(x), evaluated so that it stays finite, smooth and well scaled where EI itself
    underflows to 0 - late in a run, when most candidates lie many sigma below the incumbent and EI's gradient is
    below any optimiser's tolerance.  Same maximiser as EI wherever EI is representable.

    Parameters, y_max, the xi decay, NoValidPointRegisteredError under constraints and get/set of the acquisition
    parameters are bayes_opt.acquisition.ExpectedImprovement's.  Constraints enter as sum_j log p_j."""

    def base_acq(self, mean, std):
        if self.y_max is None:
            return super().base_acq(mean, std)  # the reference's "y_max is not set" ValueError
        return log_expected_improvement(np.asarray(mean, dtype=np.float64) - self.y_max - self.xi, std)


class LogProbabilityOfImprovement(DeviceHooks, _LogSpace, _ref.ProbabilityOfImprovement):
    """Log probability of improvement: log PoI(x) = log Phi((mean - y_max - xi) / std) through a tail-safe log_ndtr,
    finite where PoI underflows to 0.  Everything else is bayes_opt.acquisition.ProbabilityOfImprovement's;
    constraints enter as sum_j log p_j."""

    def base_acq(self, mean, std):
        if self.y_max is None:
            return super().base_acq(mean, std)  # the reference's "y_max is not set" ValueError
        with np.errstate(all="ignore"):
            return _log_ndtr((np.asarray(mean, dtype=np.float64) - self.y_max - self.xi) / std)


# before the EI / PoI entries: the log classes are subclasses of them
_STOCK = {LogExpectedImprovement: B.ACQ_LOGEI, LogProbabilityOfImprovement: B.ACQ_LOGPOI, **_STOCK}


class _SuggestStream:
    """Mixin for policies whose closure draws random numbers: ``suggest`` keeps its RandomState (and target space)
    for ``_get_acq``, which the reference's suggest calls before the random candidates are drawn from that same
    stream.  Outside suggest(), ``_get_acq`` gets a fresh unseeded stream and no space."""

    _path_rng = None
    _suggest_space = None

    def suggest(self, gp, target_space, n_random=10_000, n_smart=10, fit_gp=True, random_state=None):
        self._path_rng = _ensure_rng(random_state)
        self._suggest_space = target_space
        try:
            return super().suggest(gp, target_space, n_random=n_random, n_smart=n_smart, fit_gp=fit_gp,
                                   random_state=self._path_rng)
        finally:
            self._path_rng = None
            self._suggest_space = None

    def _suggest_rng(self):
        return self._path_rng if self._path_rng is not None else _ensure_rng(None)


def _check_int(name, v, lo, hi=None):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < lo or (hi is not None and v > hi):
        rng = f"an integer in [{lo}, {hi}]" if hi is not None else f"an integer >= {lo}"
        raise ValueError(f"{name} must be {rng}, got {v!r}")
    return int(v)


class ThompsonSampling(_SuggestStream, DeviceHooks, _ref.AcquisitionFunction):
    """Thompson sampling: every ``suggest()`` draws ONE function from the GP posterior and proposes its maximiser.

    The function is a posterior sample path (``B200GaussianProcessRegressor.sample_paths``, n_paths=1) drawn from
    the RandomState ``suggest`` receives, before the random candidates are drawn from it.  A path is a fixed smooth
    function, so the random stage ranks it on the device and the L-BFGS-B refinement runs on it like on any other
    closure.  The reference ships no such class (its tutorial's version samples multivariate_normal(mean, cov) on
    the host, which is O(M^3) in the candidates and drops the refinement).

    n_features  random Fourier features of the prior part of each path (the data update is exact).
    Constraints are not supported (ConstraintNotSupportedError).

    ``suggest_batch(..., q)`` proposes q points per call for parallel evaluation: q paths, one maximiser each
    (batch Thompson sampling, DESIGN.md 4.7)."""

    _batch_q = None  # inside suggest_batch: the number of paths the closure draws

    def __init__(self, n_features=4096, random_state=None):
        super().__init__(random_state=random_state)
        if isinstance(n_features, bool) or not isinstance(n_features, (int, np.integer)) or n_features < 1:
            raise ValueError(f"n_features must be a positive integer, got {n_features!r}")
        self.n_features = int(n_features)

    def base_acq(self, *args, **kwargs):
        raise NotImplementedError(
            "ThompsonSampling has no base_acq(mean, std): it ranks candidates by one posterior sample path drawn "
            "per suggest() (B200GaussianProcessRegressor.sample_paths), not by a formula of mean and std")

    def suggest_batch(self, gp, target_space, q, n_random=10_000, n_smart=10, fit_gp=True, random_state=None):
        """q points to probe next, as a (q, dim) array: the maximisers of q posterior sample paths drawn together.

        Runs the reference's ``suggest`` (its TargetSpaceEmptyError, one ``self.i += 1``, the GP fit), with a
        closure of q paths instead of one, and from the RandomState draws in this order:
          1. the q target paths (one ``sample_paths(q, n_features, rs)``), then q paths of each constraint GP;
          2. ONE candidate set shared by every path: ``space.random_sample(max(n_random, n_smart), rs)``, or one
             Philox seed in device_philox mode, ranked per path in one device pass (top n_smart per path);
          3. the refinement: the q x n_smart L-BFGS-B runs in lockstep, every round one device call in which each row
             is evaluated on its own path only (mixed-integer spaces: the reference's differential evolution per
             path, in path order, on that path's closure).
        Per path the reference's rule picks between the random-stage best and the refined best.  Then, in path order,
        a point bit-equal to an earlier path's is replaced by the best row of its own top-n_smart not yet taken (kept
        when there is none).  q = 1 returns ``suggest``'s point and leaves the RandomState as ``suggest`` does.
        1 <= q <= 16, an integer."""
        q = _check_int("q", q, 1, B.MAX_PATHS)
        self._batch_q = q
        try:
            return self.suggest(gp, target_space, n_random=n_random, n_smart=n_smart, fit_gp=fit_gp,
                                random_state=random_state)
        finally:
            self._batch_q = None

    def _closure(self, paths):
        from .paths import PathAcquisition, PathBatchAcquisition

        return PathAcquisition(paths) if self._batch_q is None else PathBatchAcquisition(paths)

    def _get_acq(self, gp, constraint=None):
        if constraint is not None:
            raise _ConstraintNotSupportedError(
                f"{type(self).__name__} does not support constrained optimization: a constraint model was given")
        rs = self._suggest_rng()  # the path of this call is drawn from the caller's stream
        return self._closure(_as_b200_gp(gp).sample_paths(self._batch_q or 1, self.n_features, random_state=rs))

    def _acq_min(self, acq, space, random_state, n_random=10_000, n_smart=10):
        from .paths import PathBatchAcquisition

        if not isinstance(acq, PathBatchAcquisition):
            return super()._acq_min(acq, space, random_state, n_random=n_random, n_smart=n_smart)
        if n_random == 0 and n_smart == 0:
            raise ValueError("n_random and n_smart cannot both be 0")
        x_r, min_r, tops = self._batch_random_stage(acq.paths, space, random_state, max(n_random, n_smart), n_smart)
        picks = list(x_r)
        if n_smart:
            for p, (x_s, min_s) in enumerate(self._batch_smart_stage(acq, space, tops, random_state)):
                if min_r[p] > min_s:  # the reference's choice (R/bayes_opt/acquisition.py:267-272), per path
                    picks[p] = x_s
        return np.asarray(distinct_picks(picks, tops), dtype=np.float64)

    def _batch_random_stage(self, paths, space, random_state, n, k):
        """The random stage of DeviceHooks._random_sample_minimize for q paths over ONE candidate set.
        Returns (q, d) random-stage winners, (q,) their -path values, and per path its top-k rows, best first."""
        q = paths.n_paths
        if self.b200_candidate_source == "device_philox" and all(space.continuous_dimensions) and k <= B.MAX_TOPK:
            _, vals, x_r, _, tx = self._select_philox(paths, _philox_seed(random_state), space, n, k)
            return x_r, vals, (tx if k else [[]] * q)
        x_tries = self._candidate_rows(space, n, random_state)
        if k <= B.MAX_TOPK:
            idx, vals, ti = paths.argmin_topk(x_tries, k)
            tops = [x_tries[t] for t in ti]
        else:  # more seeds than the device selection holds: numpy selection on the device values, as the reference's
            ys = -paths(x_tries)
            idx, vals = ys.argmin(axis=0), ys.min(axis=0)
            tops = [x_tries[np.argsort(ys[:, p])[:k]] for p in range(q)]
        return x_tries[idx], vals, (tops if k else [[]] * q)

    def _batch_smart_stage(self, acq, space, tops, random_state):
        """Per path (x_s, min_s) of DeviceHooks._smart_minimize from that path's seeds: continuous spaces run every
        path's L-BFGS-B runs in one lockstep; mixed-integer spaces run the reference's branch path by path."""
        q = acq.n_paths
        if not all(space.continuous_dimensions):
            return [self._smart_minimize(acq.path(p), space, tops[p], random_state) for p in range(q)]
        seeds = [s for p in range(q) for s in tops[p]]
        owner = [p for p in range(q) for _ in tops[p]]
        bounds = self._refine_bounds(space)
        runs = lockstep_lbfgsb(acq, seeds, bounds, run_paths=owner,
                               grad=self._refine_grad(acq, space)) if seeds else []
        return [self._best_run([r for r, o in zip(runs, owner) if o == p and r.success], bounds) for p in range(q)]

    def get_acquisition_params(self):
        return {"n_features": self.n_features}

    def set_acquisition_params(self, params):
        self.n_features = int(params["n_features"])


class ConstrainedThompsonSampling(ThompsonSampling):
    """Thompson sampling that also serves constrained problems (the SCBO rule: Eriksson & Poloczek, "Scalable
    Constrained Bayesian Optimization", AISTATS 2021).

    Every ``suggest()`` draws one posterior path of the target GP and one of each constraint GP, in that order, from
    the RandomState ``suggest`` receives (each with ``draw_path_inputs`` of its own GP and the same n_features).
    Among the candidates the sampled constraints call feasible it proposes the one with the largest sampled target;
    when none is feasible, the one with the smallest total violation (``paths.ConstrainedPaths``).  Unlike EI / PoI
    it needs no feasible registered point, so it does not raise NoValidPointRegisteredError.  Without a constraint
    it is ThompsonSampling.  The constraint GPs must be device GPs (``enable(optimizer)`` makes them so)."""

    def _get_acq(self, gp, constraint=None):
        if constraint is None:
            return super()._get_acq(gp, constraint=None)
        from .paths import ConstrainedPaths

        gp = _as_b200_gp(gp)
        models = [_as_b200_gp(m) for m in constraint.model]  # before any draw: a refusal consumes no random numbers
        if len(models) + 1 > B.MAX_GPS:
            raise NotImplementedError(f"at most {B.MAX_GPS - 1} constraint GPs are supported")
        rs = self._suggest_rng()
        q = self._batch_q or 1
        target = gp.sample_paths(q, self.n_features, random_state=rs)
        paths = [m.sample_paths(q, self.n_features, random_state=rs) for m in models]
        return self._closure(ConstrainedPaths(target, paths, constraint.lb, constraint.ub))


class TrustRegionThompsonSampling(ConstrainedThompsonSampling):
    """Thompson sampling inside a trust region: TuRBO-1 (Eriksson et al., NeurIPS 2019) over the global GP, and with a
    ConstraintModel SCBO (Eriksson & Poloczek, AISTATS 2021).  DESIGN.md 4.18.

    A box around the best registered row of the current run, shaped by the fitted GP's length scales, grows after
    ``success_tolerance`` successful batches, shrinks after ``failure_tolerance`` failed ones (None:
    ceil(max(4, d) / q), q the size of the batch just evaluated) and restarts when its length falls below ``length_min``
    (``trust_region.TrustRegionState``).  Each ``suggest`` / ``suggest_batch(q <= 16)``:
      1. folds the rows registered since the last call into the state and picks the centre: the best row of the run
         inside the space's current bounds (with none inside, the run's best clipped into them);
      2. when the current run has no row yet (after a restart) returns ``space.random_sample(q, rs)`` and draws nothing
         else;
      3. otherwise runs (Constrained)ThompsonSampling's suggest with three changes: the random-stage candidates are the
         centre with a random subset of coordinates redrawn in the box (about min(d, 20) of them;
         ``trust_region.host_candidates`` from the RandomState in host_rng mode, ``argmin_topk_philox_tr`` from one
         Philox seed in device_philox mode), the L-BFGS-B refinement runs inside the box, and the result is clipped to
         it.
    Continuous spaces only (NotImplementedError otherwise).  ConstantLiar, GPHedge and KrigingBeliever refuse it
    (TypeError): their dummy rows would count as observations.  The state travels in get/set_acquisition_params, so
    ``save_state`` / ``load_state`` resume the run.  ``last_box`` is the (lo, hi) of the latest call, None after a
    random call."""

    def __init__(self, n_features=4096, length_init=0.8, length_min=2**-7, length_max=1.6, success_tolerance=3,
                 failure_tolerance=None, random_state=None):
        from .trust_region import TrustRegionConfig, TrustRegionState

        super().__init__(n_features=n_features, random_state=random_state)
        self.tr_config = TrustRegionConfig(length_init, length_min, length_max, success_tolerance, failure_tolerance)
        self.tr_state = TrustRegionState(length=self.tr_config.length_init)
        self.last_box = None
        self._tr_center = None  # inside suggest: the centre row, then (lo, hi, center, p) once the GP is fitted
        self._tr_box = None

    @staticmethod
    def _tr_rows(space):
        """(targets, total violations or None) of every registered row."""
        from .trust_region import total_violation

        if space.constraint is None:
            return space.target, None
        return space.target, total_violation(space.constraint_values, space.constraint.lb, space.constraint.ub)

    def suggest(self, gp, target_space, n_random=10_000, n_smart=10, fit_gp=True, random_state=None):
        if len(target_space) == 0:  # the reference's TargetSpaceEmptyError
            return super().suggest(gp, target_space, n_random=n_random, n_smart=n_smart, fit_gp=fit_gp,
                                   random_state=random_state)
        if not all(target_space.continuous_dimensions):
            raise NotImplementedError(f"{type(self).__name__} supports continuous spaces only: its trust region is a "
                                      "box of the continuous coordinates")
        y, viol = self._tr_rows(target_space)
        self.tr_state = self.tr_state.update(y, viol, target_space.dim, self.tr_config)
        if self.tr_state.run_empty:  # a restart: the new run begins at random points
            self.i += 1
            self.last_box = None
            X = target_space.random_sample(self._batch_q or 1, random_state=_ensure_rng(random_state))
            return X if self._batch_q is not None else X[0]
        # the best row of the run inside the current bounds; with none inside, the run's best (box() clips it in)
        idx = self.tr_state.center_index(y, viol, target_space.params, target_space.bounds)
        if idx is None:
            idx = self.tr_state.center_index(y, viol)
        self._tr_center = np.array(target_space.params[idx], dtype=np.float64)
        try:
            x = super().suggest(gp, target_space, n_random=n_random, n_smart=n_smart, fit_gp=fit_gp,
                                random_state=random_state)
            lo, hi = self.last_box
            return np.clip(x, lo, hi)
        finally:
            self._tr_center = self._tr_box = None

    def _get_acq(self, gp, constraint=None):
        if self._tr_center is not None:  # the fitted GP's length scales shape this call's box
            from .gpr import parse_kernel
            from .trust_region import box, perturb_probability

            space = self._suggest_space
            ls = parse_kernel(_as_b200_gp(gp).kernel_).length_scale
            lo, hi, center = box(self._tr_center, self.tr_state.length, ls, space.bounds)
            self._tr_box = (lo, hi, center, perturb_probability(space.dim))
            self.last_box = (lo, hi)
        return super()._get_acq(gp, constraint=constraint)

    def _refine_bounds(self, space):
        if self._tr_box is None:
            return space.bounds
        return np.stack(self._tr_box[:2], axis=1)

    def _candidate_rows(self, space, n, random_state):
        if self._tr_box is None:
            return super()._candidate_rows(space, n, random_state)
        from .trust_region import host_candidates

        lo, hi, center, p = self._tr_box
        return host_candidates(random_state, n, lo, hi, center, p)

    def _select_philox(self, sel, seed, space, n, k):
        if self._tr_box is None:
            return super()._select_philox(sel, seed, space, n, k)
        lo, hi, center, p = self._tr_box
        return sel.argmin_topk_philox_tr(seed, lo, hi, center, p, n, k)

    def get_acquisition_params(self):
        from dataclasses import asdict

        return {**super().get_acquisition_params(), "trust_region_config": asdict(self.tr_config),
                "trust_region": self.tr_state.to_dict()}

    def set_acquisition_params(self, params):
        from .trust_region import TrustRegionConfig, TrustRegionState

        super().set_acquisition_params(params)
        self.tr_config = TrustRegionConfig(**params["trust_region_config"])
        self.tr_state = TrustRegionState.from_dict(params["trust_region"])


def distinct_picks(picks, tops):
    """The duplicate rule of batch Thompson sampling: in path order p = 0..q-1, a pick bit-equal to an earlier pick is
    replaced by the first row of tops[p] (path p's top-k, best first) that is bit-equal to no pick so far; with none
    left the duplicate stays.  Late in a run several paths can share their random-stage winner."""
    out, taken = [], set()
    for p, x in enumerate(picks):
        x = np.asarray(x, dtype=np.float64)
        if x.tobytes() in taken:
            for t in tops[p]:
                t = np.asarray(t, dtype=np.float64)
                if t.tobytes() not in taken:
                    x = t
                    break
        out.append(x)
        taken.add(x.tobytes())
    return out


def suggest_batch(optimizer, q):
    """q parameter dicts to probe next from a ``bayes_opt.BayesianOptimization`` whose acquisition function is a
    (Constrained)ThompsonSampling, a TrustRegionThompsonSampling, a KrigingBeliever or a PendingNEI:
    ``BayesianOptimization.suggest`` for a batch (R/bayes_opt/bayesian_optimization.py:323-333).  With no registered
    point it returns ``optimizer.random_sample(q)``; otherwise the acquisition's ``suggest_batch`` with the optimizer's
    GP, target space and RandomState, each row converted with ``array_to_params``.  For Thompson sampling nothing new
    enters ``save_state`` (q is an argument, not state); a KrigingBeliever or PendingNEI records the q points as
    dummies, which ``save_state`` carries."""
    acq = optimizer._acquisition_function
    if isinstance(acq, _PendingBatch):
        q = _check_int("q", q, 1)
    elif isinstance(acq, ThompsonSampling):
        q = _check_int("q", q, 1, B.MAX_PATHS)
    else:
        raise TypeError(f"suggest_batch needs a ThompsonSampling, ConstrainedThompsonSampling, KrigingBeliever or "
                        f"PendingNEI acquisition function, got {type(acq).__name__}; for a batch of other acquisition "
                        f"functions use ConstantLiar")
    space = optimizer._space
    if len(space) == 0:
        return optimizer.random_sample(q)
    X = acq.suggest_batch(gp=optimizer._gp, target_space=space, q=q, fit_gp=True, random_state=optimizer._random_state)
    return [space.array_to_params(x) for x in X]


# Default size of the candidate set over which the maxima of the MES sample paths are taken (DESIGN.md 4.8).
MES_MAX_CANDIDATES = 2**16


def mes_max_values(gp, paths, space, random_state, n_candidates, candidate_source="host_rng"):
    """Samples y*_k of the maximum of the target: per path k of ``paths`` (a PosteriorPaths of ``gp``),
    y*_k = max(max of path k over n_candidates random points and X_train_, the largest registered target) - on a GP
    conditioned on pending points (``condition_on_pending``), over its registered rows only.
    The floor keeps every sample consistent with the data: the maximum is at least what has been observed.
    The candidates are ``space.random_sample(n_candidates, random_state)``, or in device_philox mode on a continuous
    space one 64-bit seed drawn as DeviceHooks._random_sample_minimize draws it (rows generated in the kernel)."""
    if candidate_source == "device_philox" and all(space.continuous_dimensions):
        _, neg_max, *_ = paths.argmin_topk_philox(_philox_seed(random_state), space.bounds, n_candidates, 0)
    else:
        _, neg_max, _ = paths.argmin_topk(space.random_sample(n_candidates, random_state=random_state), 0)
    n_reg = gp.__dict__.get("_b200_conditioned")  # a GP conditioned on pending points: its registered rows only
    best = np.maximum(-np.asarray(neg_max, dtype=np.float64), paths(gp.X_train_[:n_reg]).max(axis=0))
    return np.maximum(best, float(np.max(gp._y_raw[:n_reg])))


class MaxValueEntropySearch(_SuggestStream, DeviceHooks, _ref.AcquisitionFunction):
    """Max-value entropy search (MES: Wang & Jegelka, "Max-value Entropy Search for Efficient Bayesian
    Optimization", ICML 2017): proposes the point whose observation is expected to tell the most about the value of
    the maximum, y*.  With K samples y*_k and the GP's posterior mean mu(x) and standard deviation sigma(x),

        alpha(x) = (1/K) sum_k [ g_k psi(g_k) / (2 Psi(g_k)) - log Psi(g_k) ],    g_k = (y*_k - mu(x)) / sigma(x)

    (psi, Psi: standard normal pdf and cdf; alpha = 0 where sigma = 0), evaluated in the epilogue of the fused
    predict kernel like EI.  Every ``suggest()`` draws from the RandomState it receives, in this order:

      1. ``draw_path_inputs`` of n_samples posterior sample paths of the target GP (``sample_paths``);
      2. the candidate set of the maxima: ``space.random_sample(n_max_candidates, rs)``, or with
         candidate_source="device_philox" on a continuous space one 64-bit Philox seed (``mes_max_values``);
      3. then the reference's random stage and L-BFGS-B refinement, as for every acquisition.

    y*_k is path k's maximum over those candidates and the training inputs, floored at the largest registered
    target.  With a constraint the closure is MES times the probability of feasibility; y* is sampled from the
    unconstrained target, and no feasible registered point is needed (EI / PoI raise NoValidPointRegisteredError).

    n_samples         K, 1..16 sample paths (one per y* sample)
    n_features        random Fourier features of each path's prior part
    n_max_candidates  size of the candidate set of step 2 (default MES_MAX_CANDIDATES)"""

    def __init__(self, n_samples=10, n_features=4096, n_max_candidates=MES_MAX_CANDIDATES, random_state=None):
        super().__init__(random_state=random_state)
        self.n_samples = _check_int("n_samples", n_samples, 1, B.MAX_PATHS)
        self.n_features = _check_int("n_features", n_features, 1)
        self.n_max_candidates = _check_int("n_max_candidates", n_max_candidates, 1)
        self.max_values = None  # the y* samples of the latest closure

    def base_acq(self, *args, **kwargs):
        raise NotImplementedError(
            "MaxValueEntropySearch has no base_acq(mean, std): its formula also needs the samples of the maximum "
            "drawn per suggest(), and it runs in the fused device kernel")

    def _get_acq(self, gp, constraint=None):
        gp = _as_b200_gp(gp)
        if constraint is not None:  # before any draw: a refusal consumes no random numbers
            models = [_as_b200_gp(m) for m in constraint.model]
            if len(models) + 1 > B.MAX_GPS:
                raise NotImplementedError(f"at most {B.MAX_GPS - 1} constraint GPs are supported")
        space = self._suggest_space
        if space is None:
            raise RuntimeError("MaxValueEntropySearch samples the maximum over the target space of suggest(): "
                               "build its closure through suggest()")
        rs = self._suggest_rng()
        paths = gp.sample_paths(self.n_samples, self.n_features, random_state=rs)
        ystar = mes_max_values(gp, paths, space, rs, self.n_max_candidates, self.b200_candidate_source)
        self.max_values = ystar
        return FusedAcquisition(B.ACQ_MES, gp, constraint, owner=self, max_values=ystar)

    def get_acquisition_params(self):
        return {"n_samples": self.n_samples, "n_features": self.n_features,
                "n_max_candidates": self.n_max_candidates}

    def set_acquisition_params(self, params):
        self.n_samples = _check_int("n_samples", params["n_samples"], 1, B.MAX_PATHS)
        self.n_features = _check_int("n_features", params["n_features"], 1)
        self.n_max_candidates = _check_int("n_max_candidates", params["n_max_candidates"], 1)


class _NoisyEI(_SuggestStream, DeviceHooks, _ref.ExpectedImprovement):
    """Noisy expected improvement (Letham, Karrer, Ottoni & Bakshy, "Constrained Bayesian Optimization with Noisy
    Experiments", Bayesian Analysis 2019; DESIGN.md 4.13): EI averaged over S joint samples of the noise-free function
    values at the registered points, each conditioned on as if observed exactly.  Under observation noise the largest
    registered target is the luckiest draw, not the best point, and EI against it scores little near the real optimum;
    NEI measures each fantasy against its own incumbent best_s.

    Every ``suggest()`` refuses before any draw (TargetSpaceEmptyError, NoValidPointRegisteredError without a feasible
    registered point, as EI), then draws from the RandomState it receives, in this order:
      1. Z = standard_normal((n, S)), 2. E = standard_normal((n, S))  (``noiseless_fantasies``);
      3. the reference's random stage and L-BFGS-B refinement (refine="analytic": the device gradient of NEI).
    The incumbent of each fantasy is its largest value over ``target_space.mask`` (the rows ``_target_max`` uses).
    Parameters, y_max, the xi decay and saved state are ExpectedImprovement's, plus ``n_samples`` (S, 1..16) and
    ``jitter`` (tau = min(alpha, jitter) on the noiseless GP's diagonal).  Constraints enter as for EI / LogEI.
    Not inside KrigingBeliever, ConstantLiar or GPHedge (pending points and batches: ``PendingNEI``); one device."""

    _nei_kind = None

    def __init__(self, xi=0.0, n_samples=16, jitter=1e-6, exploration_decay=None, exploration_decay_delay=None,
                 random_state=None):
        super().__init__(xi, exploration_decay=exploration_decay, exploration_decay_delay=exploration_decay_delay,
                         random_state=random_state)
        self.n_samples = _check_int("n_samples", n_samples, 1, B.MAX_PATHS)
        self.jitter = _check_jitter(jitter)
        self.fantasies = None  # the NoiselessFantasies of the latest closure

    def base_acq(self, *args, **kwargs):
        raise NotImplementedError(
            f"{type(self).__name__} has no base_acq(mean, std): it averages over fantasies of the noise-free values "
            "drawn per suggest(), and it runs in the fused device kernel")

    def _get_acq(self, gp, constraint=None):
        gp = _as_b200_gp(gp)
        if constraint is not None:  # before any draw: a refusal consumes no random numbers
            models = [_as_b200_gp(m) for m in constraint.model]
            if len(models) + 1 > B.MAX_GPS:
                raise NotImplementedError(f"at most {B.MAX_GPS - 1} constraint GPs are supported")
        space = self._suggest_space
        if space is None:
            raise RuntimeError(f"{type(self).__name__} draws its fantasies against the target space of suggest(): "
                               "build its closure through suggest()")
        return self._closure(gp, constraint, space)

    def _closure(self, gp, constraint, space, pending=None, extra_rows=0):
        """The closure over fantasies drawn from the suggest() stream; ``pending`` / ``extra_rows`` as in
        ``noiseless_fantasies`` (PendingNEI)."""
        self.fantasies = None  # the previous closure's fantasies are not needed past this point
        fant = gp.noiseless_fantasies(self.n_samples, self.jitter, incumbent=np.asarray(space.mask, dtype=bool),
                                      random_state=self._suggest_rng(), pending=pending, extra_rows=extra_rows)
        self.fantasies = fant
        return FusedAcquisition(self._nei_kind, gp, constraint, owner=self, fantasies=fant)

    def _extender(self, constraint):
        """PendingNEI's round step for the latest closure: extends its fantasies in place to a pick (d,)."""
        return self.fantasies.condition_on_pending

    def get_acquisition_params(self):
        return {**super().get_acquisition_params(), "n_samples": self.n_samples, "jitter": self.jitter}

    def set_acquisition_params(self, params):
        super().set_acquisition_params(params)
        self.n_samples = _check_int("n_samples", params["n_samples"], 1, B.MAX_PATHS)
        self.jitter = _check_jitter(params["jitter"])


def _check_jitter(v):
    if isinstance(v, bool) or not isinstance(v, (int, float, np.floating, np.integer)) or not 0.0 < float(v) < np.inf:
        raise ValueError(f"jitter must be a positive float, got {v!r}")
    return float(v)


class NoisyExpectedImprovement(_NoisyEI):
    __doc__ = _NoisyEI.__doc__
    _nei_kind = B.ACQ_NEI


class LogNoisyExpectedImprovement(_NoisyEI):
    """Log noisy expected improvement: log NEI(x) = log of the mean over the fantasies of EI, formed from LogEI's
    tail-safe terms (Ament et al. 2023), finite where NEI underflows.  Otherwise NoisyExpectedImprovement; constraints
    enter as sum_j log p_j."""

    _nei_kind = B.ACQ_LOGNEI


def cnei_eligible(space_in_bounds, constraint_fantasies, lb, ub):
    """The (n, S) incumbent mask of constrained NEI (DESIGN.md 4.15): row i may be sample s's incumbent when it lies
    within the bounds (``space_in_bounds``, (n,)) and lb_j <= F_j[i, s] <= ub_j for every constraint j."""
    ok = np.asarray(space_in_bounds, dtype=bool)[:, None]
    for j, F in enumerate(constraint_fantasies):
        ok = ok & (lb[j] <= F) & (F <= ub[j])
    return ok


def _in_bounds(space):
    """The bounds part of ``target_space.mask``: the registered rows inside the parameter bounds."""
    return _rows_in_bounds(space.params, space.bounds)


def _rows_in_bounds(rows, bounds):
    p, b = np.asarray(rows), np.asarray(bounds)
    return np.all((b[:, 0] <= p) & (p <= b[:, 1]), axis=1)


def _which_gp(j):
    return "the target GP" if j == 0 else f"constraint GP {j - 1} (constraint.model[{j - 1}])"


class _ConstrainedNoisyEI(_NoisyEI):
    """Constrained noisy expected improvement (Letham, Karrer, Ottoni & Bakshy, "Constrained Bayesian Optimization with
    Noisy Experiments", Bayesian Analysis 2019; DESIGN.md 4.15): NEI whose constraints are noisy too.  Each constraint
    GP gets fantasies of its own, and per sample s

        CNEI(x) = (1/S) sum_s EI(mu_s(x) - best_s - xi, sigma0(x)) * prod_j P_js(x),

    with P_js the probability that constraint j lies in [lb_j, ub_j] under its noiseless GP conditioned on sample s of
    its fantasies, and best_s the largest target fantasy over the rows that lie within the bounds and that sample s
    calls feasible.  A sample with no such row takes the smallest target fantasy over all registered rows as its
    incumbent: a floor, against which EI still rewards objective value and feasibility together.  So the class ranks
    candidates before any feasible point is registered and never raises NoValidPointRegisteredError (it still raises
    TargetSpaceEmptyError on an empty space).

    Every ``suggest()`` refuses before any draw (more than 7 constraints, multi-device GPs, a GP conditioned on pending
    points), then draws from the RandomState it receives: the target's Z, E, then per constraint j in order its Z_j,
    E_j (``noiseless_fantasies``), then the reference's random stage and refinement (refine="analytic": the device
    gradient of CNEI).  Parameters, get/set_acquisition_params and saved state are NoisyExpectedImprovement's.
    Without a constraint it is NoisyExpectedImprovement (LogNoisyExpectedImprovement), the same draws and values.  With
    constraint GPs fitted as the reference fits them (alpha = 1e-6, no WhiteKernel term) the constraint fantasies are
    the observed values and the value is NEI times the probability of feasibility; make the constraint GPs noisy, for
    example ``m.set_params(kernel=Matern(nu=2.5) + WhiteKernel())`` for each ``m`` in ``optimizer.constraint.model``,
    to model constraint noise.  The incumbents are formed on the device (``b200bo_gp_set_constrained_incumbent``).

    ``PendingNEI`` gives it pending points and batches with constraints (DESIGN.md 4.16): the target's and every
    constraint's fantasies are drawn jointly with their values at the pending points (per GP in order: Z, E, then
    ``standard_normal((p + q - 1, S))``), a pending row counts toward sample s's incumbent only where sample s's
    constraint fantasies call it feasible (and it lies within the bounds), and each round extends every GP to the pick
    (``condition_on_pending``).  A batch built round by round is greedy sequential constrained qNEI."""

    _cnei_kind = None

    def suggest(self, gp, target_space, n_random=10_000, n_smart=10, fit_gp=True, random_state=None):
        # ExpectedImprovement.suggest without its NoValidPointRegisteredError: y_max is not used by (C)NEI
        self._path_rng = _ensure_rng(random_state)
        self._suggest_space = target_space
        try:
            self.y_max = target_space._target_max()
            x = _ref.AcquisitionFunction.suggest(self, gp, target_space, n_random=n_random, n_smart=n_smart,
                                                 fit_gp=fit_gp, random_state=self._path_rng)
            self.decay_exploration()
            return x
        finally:
            self._path_rng = None
            self._suggest_space = None

    def _closure(self, gp, constraint, space, pending=None, extra_rows=0):
        """The closure over the fantasies of the target and of every constraint GP; ``pending`` ((p, d)) and
        ``extra_rows`` as in ``noiseless_fantasies``, for every GP (PendingNEI, DESIGN.md 4.16)."""
        if constraint is None:
            return super()._closure(gp, constraint, space, pending=pending, extra_rows=extra_rows)
        models = [_as_b200_gp(m) for m in constraint.model]
        box = np.asarray(space.bounds, dtype=np.float64)
        P = np.empty((0, box.shape[0])) if pending is None else np.asarray(pending, dtype=np.float64)
        P = P.reshape(-1, box.shape[0])
        rows = P.shape[0] + int(extra_rows)
        # before any draw: a refusal consumes no random numbers
        if len(models) + 1 > B.MAX_GPS:
            raise NotImplementedError(f"at most {B.MAX_GPS - 1} constraint GPs are supported")
        for g in [gp, *models]:
            if len(g.device_list()) > 1:
                raise NotImplementedError("constrained noisy expected improvement runs on one device: a GP is "
                                          "multi-device")
            if g.__dict__.get("_b200_conditioned") is not None:
                raise NotImplementedError("constrained noisy expected improvement on a GP conditioned on pending "
                                          "points")
        for g in [gp, *models] if rows else []:
            g._ensure_device_fit()
            if g.__dict__.get("_b200_xform", ("device", None))[0] == "host":
                raise NotImplementedError("pending points for constrained noisy expected improvement with a host-side "
                                          "(categorical) kernel transform")
        self.fantasies = self.constraint_fantasies = None
        rs = self._suggest_rng()
        kw = {"pending": P, "extra_rows": extra_rows} if rows else {}
        fants = []
        for j, g in enumerate([gp, *models]):  # the target's draws, then each constraint's, in order
            try:
                fants.append(g.noiseless_fantasies(self.n_samples, self.jitter, random_state=rs, **kw))
            except np.linalg.LinAlgError as e:
                raise np.linalg.LinAlgError(f"{e} [{_which_gp(j)}]") from None
        self.fantasies, self.constraint_fantasies = fants[0], fants[1:]
        self._bounds_box = box
        self._in_bounds_mask = np.concatenate([_in_bounds(space), _rows_in_bounds(P, box)])
        self._lb = B.c_f64(np.atleast_1d(constraint.lb))
        self._ub = B.c_f64(np.atleast_1d(constraint.ub))
        self._set_incumbent()
        return FusedAcquisition(self._cnei_kind, gp, constraint, owner=self, fantasies=self.fantasies,
                                constraint_fantasies=self.constraint_fantasies)

    def _set_incumbent(self):
        """best_s over the rows the fantasies hold, on the device (``b200bo_gp_set_constrained_incumbent``)."""
        fant, cfant = self.fantasies, self.constraint_fantasies
        handles = (C.c_void_p * len(cfant))(*[f.handle.ptr.value for f in cfant])
        inb = np.ascontiguousarray(self._in_bounds_mask, dtype=np.uint8)
        best = np.empty(self.n_samples)
        B.check(B.lib().b200bo_gp_set_constrained_incumbent(
            fant.handle.ptr, handles, len(cfant), B.as_dp(self._lb), B.as_dp(self._ub),
            inb.ctypes.data_as(C.POINTER(C.c_uint8)), B.as_dp(best)))
        fant.best = best

    def condition_on_pending(self, X):
        """Extends the latest closure in place to the pending points ``X`` ((p, d) or (d,)): the target's fantasies,
        then each constraint's in ``constraint.model`` order (``NoiselessFantasies.condition_on_pending``, each from
        its own pre-drawn z rows), then the incumbents over the grown rows.  A non-positive pivot raises
        np.linalg.LinAlgError naming jitter and the GP."""
        X = np.asarray(X, dtype=np.float64).reshape(-1, self._bounds_box.shape[0])
        for j, f in enumerate([self.fantasies, *self.constraint_fantasies]):
            try:
                f.condition_on_pending(X)
            except np.linalg.LinAlgError as e:
                raise np.linalg.LinAlgError(f"{e} [{_which_gp(j)}]") from None
        self._in_bounds_mask = np.concatenate([self._in_bounds_mask, _rows_in_bounds(X, self._bounds_box)])
        self._set_incumbent()

    def _extender(self, constraint):
        return super()._extender(constraint) if constraint is None else self.condition_on_pending


class ConstrainedNoisyExpectedImprovement(_ConstrainedNoisyEI):
    __doc__ = _ConstrainedNoisyEI.__doc__
    _nei_kind = B.ACQ_NEI
    _cnei_kind = B.ACQ_CNEI


class LogConstrainedNoisyExpectedImprovement(_ConstrainedNoisyEI):
    """Log constrained noisy expected improvement: log CNEI(x) = log of the mean over the samples of
    EI_s * prod_j P_js, formed from LogEI's tail-safe terms plus sum_j log P_js (Ament et al. 2023), finite where CNEI
    underflows.  Otherwise ConstrainedNoisyExpectedImprovement; without a constraint it is LogNoisyExpectedImprovement."""

    _nei_kind = B.ACQ_LOGNEI
    _cnei_kind = B.ACQ_LOGCNEI


def _refuse_nei(acq, where):
    if isinstance(acq, _NoisyEI):
        raise TypeError(f"{where} does not support {type(acq).__name__}: its fantasies are drawn per suggest() against "
                        "the registered data")
    if isinstance(acq, PosteriorMean):
        raise TypeError(f"{where} does not support {type(acq).__name__}: it recommends the best posterior mean and "
                        "does not choose points to evaluate")
    if isinstance(acq, TrustRegionThompsonSampling):
        raise TypeError(f"{where} does not support {type(acq).__name__}: its trust region would count the dummy rows "
                        "as observations")


_HOOKED = {
    _ref.UpperConfidenceBound: UpperConfidenceBound,
    _ref.ProbabilityOfImprovement: ProbabilityOfImprovement,
    _ref.ExpectedImprovement: ExpectedImprovement,
}


def accelerate(acq, candidate_source=None, refine=None):
    """Give an existing reference acquisition object the device hooks IN PLACE (all state kept: kappa/xi,
    decay counters, dummies, gains).  ConstantLiar / GPHedge only orchestrate: their base acquisitions are
    accelerated, the wrappers stay what they are.  candidate_source / refine: None leaves the object's setting."""
    if candidate_source not in (None, "host_rng", "device_philox"):
        raise ValueError("candidate_source must be 'host_rng' or 'device_philox'")
    if refine not in (None, "stencil", "analytic"):
        raise ValueError("refine must be 'stencil' or 'analytic'")
    if isinstance(acq, _ref.ConstantLiar):
        if not isinstance(acq, PendingNEI):
            _refuse_nei(acq.base_acquisition, type(acq).__name__)
        acq.base_acquisition = accelerate(acq.base_acquisition, candidate_source, refine)
        return acq
    if isinstance(acq, _ref.GPHedge):
        for a in acq.base_acquisitions:
            _refuse_nei(a, type(acq).__name__)
        acq.base_acquisitions = [accelerate(a, candidate_source, refine) for a in acq.base_acquisitions]
        return acq
    if candidate_source is not None:
        acq.b200_candidate_source = candidate_source
    if refine is not None:
        acq.b200_refine = refine
    if isinstance(acq, DeviceHooks):
        return acq
    cls = type(acq)
    hooked = _HOOKED.get(cls)
    if hooked is None:  # user subclass (possibly of UCB/EI/PoI, possibly with its own base_acq)
        hooked = type("B200" + cls.__name__, (DeviceHooks, cls), {"__module__": __name__})
    acq.__class__ = hooked
    return acq


class ConstantLiar(_ref.ConstantLiar):
    """bayes_opt.acquisition.ConstantLiar whose base acquisition runs on the device."""

    def __init__(self, base_acquisition, *args, **kwargs):
        _refuse_nei(base_acquisition, "ConstantLiar")
        super().__init__(accelerate(base_acquisition), *args, **kwargs)


class GPHedge(_ref.GPHedge):
    """bayes_opt.acquisition.GPHedge over device base acquisitions."""

    def __init__(self, base_acquisitions, *args, **kwargs):
        for a in base_acquisitions:
            _refuse_nei(a, "GPHedge")
        super().__init__([accelerate(a) for a in base_acquisitions], *args, **kwargs)


class _PendingBatch(_ref.ConstantLiar):
    """ConstantLiar's dummy bookkeeping (``dummies``, their expiry within atol / rtol of a registered point, and
    get/set_acquisition_params, so ``save_state`` carries them) with the base acquisition's own ``suggest`` and greedy
    batch rounds on one candidate set.  Subclasses say how the dummies and the picks enter the closure
    (``_round_closure``); KrigingBeliever conditions the GP, PendingNEI the NEI fantasies."""

    def suggest(self, gp, target_space, n_random=10_000, n_smart=10, fit_gp=True, random_state=None):
        return self._believe(gp, target_space, None, n_random, n_smart, fit_gp, random_state)

    def _round_closure(self, gp, constraint, pending, q):
        """(closure of round 0 over the dummies ``pending``, callable that extends it in place by one pick (d,))."""
        raise NotImplementedError

    def _serves_constraints(self):
        return False

    def _believe(self, gp, target_space, q, n_random, n_smart, fit_gp, random_state):
        if len(target_space) == 0:
            raise _TargetSpaceEmptyError("Cannot suggest a point without previous samples: register a point first "
                                         "(target_space.random_sample() / target_space.probe()).")
        if target_space.constraint is not None and not self._serves_constraints():
            raise _ConstraintNotSupportedError(f"{type(self).__name__} does not support constrained optimization: "
                                               "the target space has a constraint")
        self._remove_expired_dummies(target_space)
        base = self.base_acquisition
        pending = np.asarray(self.dummies, dtype=np.float64).reshape(len(self.dummies), target_space.dim)
        extend = []

        def get_acq(gp, constraint=None):  # between the base's fit and its closure
            acq, ext = self._round_closure(_as_b200_gp(gp), constraint, pending, q)
            extend.append(ext)
            return acq

        def acq_min(acq, space, random_state, n_random=10_000, n_smart=10):
            return self._rounds(acq, extend[0], space, random_state, n_random, n_smart, q)

        base._get_acq = get_acq
        if q is not None:
            base._acq_min = acq_min
        try:
            x = base.suggest(gp, target_space, n_random=n_random, n_smart=n_smart, fit_gp=fit_gp,
                             random_state=_ensure_rng(random_state))
        finally:
            base.__dict__.pop("_get_acq", None)
            base.__dict__.pop("_acq_min", None)
        if q is None:
            self.dummies.append(x)
        else:
            self.dummies.extend(np.array(r) for r in x)
        return x

    def _rounds(self, acq, extend, space, random_state, n_random, n_smart, q):
        if n_random == 0 and n_smart == 0:
            raise ValueError("Either n_random or n_smart needs to be greater than 0.")
        base = self.base_acquisition
        n = max(n_random, n_smart)
        philox = base.b200_candidate_source == "device_philox" and all(space.continuous_dimensions)
        philox = philox and n_smart <= B.MAX_TOPK
        if philox:
            seed = _philox_seed(random_state)
        else:
            x_tries = space.random_sample(n, random_state=random_state)  # the reference's RNG stream
        picks = []
        for j in range(q):
            # the random stage of DeviceHooks._random_sample_minimize on the shared set
            if philox:
                _, min_r, x_r, _, tops = acq.argmin_topk_philox(seed, space.bounds, n, n_smart)
            elif n_smart <= B.MAX_TOPK:
                idx, min_r, top = acq.argmin_topk(x_tries, n_smart)
                x_r, tops = x_tries[idx], x_tries[top]
            else:  # more seeds than the device selection holds: numpy selection on the device values
                ys = acq(x_tries)
                x_r, min_r, tops = x_tries[ys.argmin()], ys.min(), x_tries[np.argsort(ys)[:n_smart]]
            x = x_r
            if n_smart:
                x_s, min_s = base._smart_minimize(acq, space, x_seeds=tops, random_state=random_state)
                if min_r > min_s:  # the reference's choice (R/bayes_opt/acquisition.py:267-272)
                    x = x_s
            x = distinct_picks(picks + [x], [[]] * len(picks) + [tops])[-1]
            picks.append(np.asarray(x, dtype=np.float64))
            if j < q - 1:
                extend(picks[-1])  # in place: the closure has room for the batch
        return np.asarray(picks, dtype=np.float64)


class KrigingBeliever(_PendingBatch):
    """Batches and asynchronous suggestions for UCB, EI, PoI and MES: the fixed-hyper-parameter counterpart of
    ``ConstantLiar`` (Kriging believer: Ginsbourger, Le Riche & Carraro, "Kriging is well-suited to parallelize
    optimization", 2010; DESIGN.md 4.11).

    A pending point - suggested, not yet registered - is a dummy, with ConstantLiar's bookkeeping (inherited:
    ``dummies``, their expiry once a registered point is within atol / rtol, and get/set_acquisition_params, so
    ``save_state`` carries them).  Where ConstantLiar registers the dummies with a made-up target and refits the GP on
    that space, this class fits the hyper-parameters on the registered data only and then conditions the fitted GP on
    the dummies with the GP's own posterior mean as their targets (``condition_on_pending``: one O(N^2) row update per
    point on the device).  The mean is unchanged; the standard deviation shrinks near the dummies, so the base
    acquisition turns away from them.  ``strategy`` is accepted for ConstantLiar's parameter layout and not used.

    ``suggest()``: the base acquisition's own ``suggest`` (its empty-space error, one ``i += 1``, its y_max, its
    kappa / xi decay) with the GP conditioned on the unexpired dummies between the fit and the closure; the pick
    becomes a dummy.  ``suggest_batch(..., q)``: q points from one call by greedy rounds on one candidate set.
    Constraints raise ConstraintNotSupportedError, as ConstantLiar does.  Noisy EI: ``PendingNEI``."""

    def __init__(self, base_acquisition, strategy="max", random_state=None, atol=1e-5, rtol=1e-8):
        _refuse_nei(base_acquisition, "KrigingBeliever")
        if _device_kind(base_acquisition) is None and not isinstance(base_acquisition, MaxValueEntropySearch):
            raise TypeError(f"KrigingBeliever needs an UpperConfidenceBound, ExpectedImprovement, "
                            f"ProbabilityOfImprovement, LogExpectedImprovement, LogProbabilityOfImprovement or "
                            f"MaxValueEntropySearch base acquisition, got {type(base_acquisition).__name__}")
        super().__init__(accelerate(base_acquisition), strategy, random_state, atol, rtol)

    def suggest_batch(self, gp, target_space, q, n_random=10_000, n_smart=10, fit_gp=True, random_state=None):
        """q points to probe next, as a (q, dim) array.  In this order:
          1. the base acquisition's ``suggest`` accounting, once for the batch (one ``i += 1``, one kappa / xi decay;
             y_max is the registered data's for every round), the hyper-parameter fit on the registered data, then
             the conditioning on the unexpired dummies, on a fork of the GP with room for the batch;
          2. the base closure on that GP - MES draws its y* samples here, once per batch;
          3. ONE candidate set shared by every round: ``space.random_sample(max(n_random, n_smart), rs)``, or one
             Philox seed in device_philox mode;
          4. per round j = 0..q-1: the fused selection over that set on round j's GP, the refinement of its top
             n_smart (the L-BFGS-B runs in lockstep; mixed-integer spaces: the reference's DE branch), the reference's
             random-vs-refined rule, the duplicate rule of ``distinct_picks`` against the earlier picks, then the GP
             is conditioned in place on the pick;
          5. the q picks become dummies.
        q = 1 without dummies returns the base acquisition's ``suggest`` point and leaves the RandomState as it does.
        q is an integer >= 1."""
        q = _check_int("q", q, 1)
        return self._believe(gp, target_space, q, n_random, n_smart, fit_gp, random_state)

    def _round_closure(self, gp, constraint, pending, q):
        if len(pending) or (q or 1) > 1:
            gp = gp.condition_on_pending(pending, extra_rows=q or 0)
        base = self.base_acquisition
        return type(base)._get_acq(base, gp=gp, constraint=constraint), lambda x: gp.condition_on_pending(x[None])


class PendingNEI(_PendingBatch):
    """Pending points and batches for noisy EI (``NoisyExpectedImprovement`` / ``LogNoisyExpectedImprovement``): the
    unknown values at the points in flight are drawn jointly with NEI's fantasies of the registered values (Letham et
    al., Bayesian Analysis 2019, section 5; DESIGN.md 4.14), not believed as in ``KrigingBeliever``.  Each candidate is
    scored by NEI on the noiseless GP conditioned on the pending points, against incumbents that count the pending
    fantasies, so a batch built round by round is greedy sequential qNEI (qLogNEI with the log base).

    Dummies, their expiry, ``save_state``, ``suggest()``, ``suggest_batch(..., q)``, one ``i += 1`` and one xi decay
    per call, the shared candidate set and the rounds are KrigingBeliever's.  The differences: per call the base draws
    its fantasies once (Z, E, then ``standard_normal((p + q - 1, S))`` for the p unexpired dummies and the q - 1 later
    picks; ``noiseless_fantasies(pending=..., extra_rows=...)``) on a fork of the noiseless GP, and each round extends
    those fantasies to the previous pick (``NoiselessFantasies.condition_on_pending``); the fitted GP is never
    conditioned or modified.  q = 1 without dummies returns the base's ``suggest`` point and leaves the RandomState as
    it does.  With a ``ConstrainedNoisyExpectedImprovement`` / ``LogConstrainedNoisyExpectedImprovement`` base it
    serves constrained target spaces (DESIGN.md 4.16): every constraint GP gets fantasies at the pending points too,
    after the target's, and a pending row counts toward a sample's incumbent only where that sample calls it feasible;
    with an NEI / LogNEI base a constraint raises ConstraintNotSupportedError.  Multi-device GPs and host-side
    (categorical) transforms raise NotImplementedError; a non-positive pivot raises np.linalg.LinAlgError naming jitter
    (and, with constraints, the GP).  ``strategy`` is accepted for ConstantLiar's parameter layout and not used."""

    def __init__(self, base_acquisition, strategy="max", random_state=None, atol=1e-5, rtol=1e-8):
        if not isinstance(base_acquisition, _NoisyEI):
            raise TypeError(f"PendingNEI needs a NoisyExpectedImprovement or LogNoisyExpectedImprovement base "
                            f"acquisition, got {type(base_acquisition).__name__}")
        super().__init__(base_acquisition, strategy, random_state, atol, rtol)

    def suggest_batch(self, gp, target_space, q, n_random=10_000, n_smart=10, fit_gp=True, random_state=None):
        """q points to probe next, as a (q, dim) array: KrigingBeliever.suggest_batch's steps, with the fantasies of
        step 2 drawn for the dummies and q - 1 later picks, and each round extending them to the previous pick.
        q is an integer >= 1."""
        q = _check_int("q", q, 1)
        return self._believe(gp, target_space, q, n_random, n_smart, fit_gp, random_state)

    def _serves_constraints(self):
        return isinstance(self.base_acquisition, _ConstrainedNoisyEI)

    def _round_closure(self, gp, constraint, pending, q):
        base = self.base_acquisition
        acq = base._closure(gp, constraint, base._suggest_space, pending=pending, extra_rows=(q or 1) - 1)
        return acq, base._extender(constraint)


# isinstance(x, b200.AcquisitionFunction) holds for every acquisition of this module, as
# isinstance(x, bayes_opt.acquisition.AcquisitionFunction) does in the reference (abc virtual subclasses:
# the concrete classes keep the reference's MRO).
for _cls in (UpperConfidenceBound, ProbabilityOfImprovement, ExpectedImprovement, LogExpectedImprovement,
             LogProbabilityOfImprovement, ConstantLiar, GPHedge, ThompsonSampling, ConstrainedThompsonSampling,
             MaxValueEntropySearch, KrigingBeliever, NoisyExpectedImprovement, LogNoisyExpectedImprovement,
             ConstrainedNoisyExpectedImprovement, LogConstrainedNoisyExpectedImprovement, PendingNEI, PosteriorMean):
    AcquisitionFunction.register(_cls)
del _cls

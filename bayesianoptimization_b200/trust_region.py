"""Trust region of TuRBO (Eriksson et al., "Scalable Global Optimization via Local Bayesian Optimization", NeurIPS 2019)
and of SCBO (Eriksson & Poloczek, "Scalable Constrained Bayesian Optimization", AISTATS 2021): the state machine, the
box and the host candidate sampler behind ``acquisition.TrustRegionThompsonSampling`` (DESIGN.md 4.18).

Numpy only, no ``bayes_opt`` import.  The state is a pure function of the registered rows and of how many of them were
registered before each ``suggest``: ``TrustRegionState.update`` folds the rows registered since the last call into it.

Ranking of rows (``best_index``).  Without constraints the largest target wins.  With constraints a row is feasible when
its total violation ``sum_j max(0, lb_j - c_j) + max(0, c_j - ub_j)`` is 0 (``total_violation``, the ``viol`` of
``paths.ConstrainedPaths``); feasible rows rank first by target, infeasible rows by the smallest violation.  The first
of equal rows wins.

Success of a batch (``improves``): its best row beats the run's best so far -
  feasible vs feasible:      y_new > y_best + 1e-3 |y_best|
  feasible vs infeasible:    always
  infeasible vs infeasible:  viol_new < viol_best            (SCBO's rule: a strict decrease, no relative margin)
  infeasible vs feasible:    never
The state counts every registered row.  The centre is the best row of the current run among those inside the space's
current bounds (``center_index``), as ``TargetSpace.mask`` counts them; when none is inside (bounds shrunk past the
whole run) it is the run's best row clipped into the bounds (``box``).
"""
from __future__ import annotations

import math
from dataclasses import asdict, dataclass

import numpy as np

LENGTH_INIT, LENGTH_MIN, LENGTH_MAX = 0.8, 2.0**-7, 1.6
SUCCESS_TOLERANCE = 3
MAX_PERTURBED = 20  # expected number of perturbed coordinates per candidate (TuRBO's min(d, 20))
IMPROVEMENT = 1e-3  # relative margin of a success


def perturb_probability(d):
    """p of the trust-region source: (min(d, 20) - 1) / (d - 1), 1 for d <= 20.  With the forced column every row
    perturbs 1 + p (d - 1) = min(d, 20) coordinates in expectation, at least one."""
    d = int(d)
    return 1.0 if d <= MAX_PERTURBED else (MAX_PERTURBED - 1) / (d - 1)


def failure_tolerance(d, q):
    """tau_fail = ceil(max(4, d) / q): q the size of the batch just evaluated."""
    return math.ceil(max(4, int(d)) / max(1, int(q)))


def total_violation(c, lb, ub):
    """(n,) sum over constraints j, in j order, of max(0, lb_j - c_j) + max(0, c_j - ub_j); c: (n,) or (n, J)."""
    c = np.asarray(c, dtype=np.float64)
    c = c.reshape(c.shape[0], -1)
    lb = np.broadcast_to(np.asarray(lb, dtype=np.float64).reshape(-1), (c.shape[1],))
    ub = np.broadcast_to(np.asarray(ub, dtype=np.float64).reshape(-1), (c.shape[1],))
    v = np.zeros(c.shape[0])
    for j in range(c.shape[1]):
        v = v + (np.maximum(0.0, lb[j] - c[:, j]) + np.maximum(0.0, c[:, j] - ub[j]))
    return v


def best_index(y, viol=None):
    """Index of the best row: the largest y, or with violations the feasible row with the largest y, else the row
    with the smallest violation.  The first of equal rows."""
    y = np.asarray(y, dtype=np.float64)
    if viol is None:
        return int(np.argmax(y))
    viol = np.asarray(viol, dtype=np.float64)
    feas = viol == 0.0
    if feas.any():
        idx = np.flatnonzero(feas)
        return int(idx[np.argmax(y[idx])])
    return int(np.argmin(viol))


def improves(y_new, v_new, y_best, v_best):
    """True when a batch whose best row is (y_new, v_new) is a success against the run's best (y_best, v_best);
    v_* None without constraints (module docstring)."""
    if v_new is None or (v_new == 0.0 and v_best == 0.0):
        return bool(y_new > y_best + IMPROVEMENT * abs(y_best))
    if v_new == 0.0:
        return True
    if v_best == 0.0:
        return False
    return bool(v_new < v_best)


@dataclass
class TrustRegionConfig:
    length_init: float = LENGTH_INIT
    length_min: float = LENGTH_MIN
    length_max: float = LENGTH_MAX
    success_tolerance: int = SUCCESS_TOLERANCE
    failure_tolerance: int | None = None  # None: ceil(max(4, d) / q) per batch

    def __post_init__(self):
        vals = (self.length_init, self.length_min, self.length_max)
        if not all(isinstance(v, (int, float, np.floating)) and not isinstance(v, bool) and math.isfinite(v)
                   for v in vals):
            raise ValueError(f"trust-region lengths must be finite numbers, got {vals!r}")
        if not 0.0 < self.length_min <= self.length_init <= self.length_max:
            raise ValueError(f"need 0 < length_min <= length_init <= length_max, got {vals!r}")
        self.length_init, self.length_min, self.length_max = (float(v) for v in vals)
        for name in ("success_tolerance", "failure_tolerance"):
            v = getattr(self, name)
            if v is None and name == "failure_tolerance":
                continue
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
                raise ValueError(f"{name} must be a positive integer, got {v!r}")
            setattr(self, name, int(v))


@dataclass
class TrustRegionState:
    """length: side of the box in units of the bounds' spans (before the length-scale shaping); n_success /
    n_failure: consecutive successful / failed batches; run_start: index of the first registered row of the current
    run; n_seen: rows already folded in; n_restarts: runs abandoned because the box collapsed."""

    length: float = LENGTH_INIT
    n_success: int = 0
    n_failure: int = 0
    run_start: int = 0
    n_seen: int = 0
    n_restarts: int = 0

    @property
    def run_empty(self):
        """True when no registered row belongs to the current run (after a restart): the next call samples the
        whole space."""
        return self.run_start >= self.n_seen

    def update(self, y, viol, d, config):
        """The state after folding in rows n_seen..len(y)-1 (y: every registered target, viol: their total
        violations or None).  The first batch of a run only starts it; each later batch is a success or a failure
        (``improves``).  tau_succ successes double the length (up to length_max), tau_fail failures halve it; below
        length_min the run restarts at the next registered row."""
        y = np.asarray(y, dtype=np.float64).reshape(-1)
        n = y.shape[0]
        if n < self.n_seen:
            raise ValueError(f"{n} registered rows, but the trust region has already seen {self.n_seen}")
        s = TrustRegionState(**asdict(self))
        if n == self.n_seen:
            return s
        if s.run_start < s.n_seen:
            v = None if viol is None else np.asarray(viol, dtype=np.float64).reshape(-1)
            old = slice(s.run_start, s.n_seen)
            new = slice(s.n_seen, n)
            bo = s.run_start + best_index(y[old], None if v is None else v[old])
            bn = s.n_seen + best_index(y[new], None if v is None else v[new])
            ok = improves(y[bn], None if v is None else v[bn], y[bo], None if v is None else v[bo])
            tau_fail = config.failure_tolerance or failure_tolerance(d, n - s.n_seen)
            if ok:
                s.n_success, s.n_failure = s.n_success + 1, 0
            else:
                s.n_success, s.n_failure = 0, s.n_failure + 1
            if s.n_success >= config.success_tolerance:
                s.length, s.n_success = min(2.0 * s.length, config.length_max), 0
            elif s.n_failure >= tau_fail:
                s.length, s.n_failure = s.length / 2.0, 0
            if s.length < config.length_min:
                s.length, s.n_success, s.n_failure = config.length_init, 0, 0
                s.run_start = n
                s.n_restarts += 1
        s.n_seen = n
        return s

    def center_index(self, y, viol, X=None, bounds=None):
        """Index (into the registered rows) of the best row of the current run.  With X (the registered rows) and
        bounds (d, 2), only rows inside the bounds compete, as ``TargetSpace.mask`` counts them (bounds shrunk by a
        bounds transformer or ``set_bounds``, points registered outside them); None when no row of the run is inside."""
        r = np.arange(self.run_start, self.n_seen)
        if X is not None:
            b = np.asarray(bounds, dtype=np.float64)
            Xr = np.asarray(X, dtype=np.float64)[r]
            r = r[np.all((b[:, 0] <= Xr) & (Xr <= b[:, 1]), axis=1)]
            if r.size == 0:
                return None
        return int(r[best_index(np.asarray(y)[r], None if viol is None else np.asarray(viol)[r])])

    def to_dict(self):
        return {k: (float(v) if k == "length" else int(v)) for k, v in asdict(self).items()}

    @classmethod
    def from_dict(cls, d):
        return cls(length=float(d["length"]), **{k: int(d[k]) for k in
                                                 ("n_success", "n_failure", "run_start", "n_seen", "n_restarts")})


def box(center, length, length_scales, bounds):
    """(lo, hi, center) of the trust region: center_j -+ length w_j span_j / 2, intersected with bounds (d, 2).
    l~_j = l_j / span_j are the fitted length scales in units of the spans (an isotropic one broadcast), and
    w = l~ / geomean(l~), so the box has the volume of a cube of side length (before the intersection).  A centre
    outside the bounds is clipped into them first, so lo <= center <= hi always holds."""
    bounds = np.asarray(bounds, dtype=np.float64)
    lo, hi = bounds[:, 0], bounds[:, 1]
    span = hi - lo
    d = lo.shape[0]
    ls = np.broadcast_to(np.asarray(length_scales, dtype=np.float64).reshape(-1), (d,))
    lt = ls / span
    w = lt / np.exp(np.mean(np.log(lt)))
    half = length * w * span / 2.0
    center = np.clip(np.asarray(center, dtype=np.float64), lo, hi)
    return np.maximum(center - half, lo), np.minimum(center + half, hi), center


def host_candidates(rs, n, lo, hi, center, p):
    """n candidates of the trust-region source from a RandomState, in this order:
        U = rs.random_sample((n, d)); x = lo + span U        (two roundings, as on the device)
        V = rs.random_sample((n, d))
        f = rs.randint(0, d, n)                            (the column every row perturbs)
        row i: x_ij where j == f_i or V_ij < p, center_j elsewhere
    The RandomState advances by the same amount whatever p, lo, hi and center are."""
    lo, hi, center = (np.asarray(a, dtype=np.float64) for a in (lo, hi, center))
    d = lo.shape[0]
    U = rs.random_sample((n, d))
    x = lo + (hi - lo) * U
    V = rs.random_sample((n, d))
    f = rs.randint(0, d, n)
    mask = (V < p) | (np.arange(d)[None, :] == f[:, None])
    return np.where(mask, x, center[None, :])

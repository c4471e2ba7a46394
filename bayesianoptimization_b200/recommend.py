"""``recommend(optimizer)``: the point a run should report, by the posterior mean rather than the luckiest draw.

``optimizer.max`` is the reference's ``TargetSpace.max()``: the largest noisy observation among the rows observed
feasible.  Under noise that overstates the target, and under noisy constraints it may be infeasible in truth.  NEI's
paper (Letham et al., Bayesian Analysis 2019) recommends the best posterior mean instead; this module does that on the
device with the ``B200BO_ACQ_MEAN`` merit (include/b200bo.h, DESIGN.md 4.17), and leaves the optimizer as it was.
"""
from __future__ import annotations

import numpy as np
from sklearn.base import clone

from . import _lib as B
from .gpr import B200GaussianProcessRegressor, to_b200_gp


class _Constraint:
    """What FusedAcquisition reads of a ConstraintModel: its GPs and bounds."""

    def __init__(self, model, lb, ub):
        self.model, self.lb, self.ub = model, lb, ub


def _fitted_on(gp, X, y):
    """True when ``gp`` is a device GP fitted on exactly the rows (X, y): no conditioning on pending points."""
    if not isinstance(gp, B200GaussianProcessRegressor) or not hasattr(gp, "X_train_"):
        return False
    if gp.__dict__.get("_b200_conditioned") is not None or not hasattr(gp, "_y_raw"):
        return False
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    return (gp.X_train_.shape == X.shape and np.array_equal(gp.X_train_, X) and gp._y_raw.shape == y.shape
            and np.array_equal(gp._y_raw, y))


def _model_on(gp, X, y, rng):
    """``gp`` itself, read-only, when it is fitted on (X, y); otherwise a device clone fitted there whose restarts
    draw from ``rng`` - never ``gp`` or its RandomState."""
    if _fitted_on(gp, X, y):
        return gp
    c = to_b200_gp(clone(gp))
    c.set_params(random_state=rng)
    c.fit(X, np.asarray(y, dtype=np.float64).reshape(-1))
    return c


def _violation(means, lb, ub):
    """The summed violation of the constraint means, as the device forms it (infinite bounds contribute 0)."""
    v = 0.0
    for m, lo, hi in zip(means, lb, ub):
        a = 0.0 if lo == -np.inf else max(0.0, lo - m)
        b = 0.0 if hi == np.inf else max(0.0, m - hi)
        v = v + (a + b)
    return v


def recommend(optimizer, in_sample=True, n_random=10_000, n_smart=10, random_state=None):
    """The point to report at the end of a (noisy) run, as a dict shaped like ``optimizer.max``.

    ``target`` is the posterior mean of the target GP there and ``params`` the point; ``std`` is the posterior standard
    deviation there; with constraints, ``constraint`` holds the constraint GPs' means (a float for one constraint) and
    ``allowed`` whether each lies within its bounds.  The ranking is the ``PosteriorMean`` merit: the best mean among
    the mean-feasible points, else the least summed violation of the constraint means.

    in_sample=True   the registered point with the best merit (the choice of Letham et al. and BoTorch): always a
                     point that was evaluated.
    in_sample=False  the best merit over the whole domain: the reference's random stage and L-BFGS-B (n_random,
                     n_smart) on a ``PosteriorMean`` closure, the candidates and seeds drawn from ``random_state``.

    The optimizer is left exactly as it was: its GPs are used read-only when they are fitted on the registered rows,
    and otherwise clones are fitted on the device, their restarts drawing from ``random_state``; no RandomState of the
    optimizer, no model and no dummy is touched, so a call in the middle of a run changes no later suggestion.
    Raises the package's no-device error without a device, and TargetSpaceEmptyError without a registered point."""
    if B.lib().b200bo_device_count() < 1:
        raise B.B200Error(f"b200bo error {B.ERR_CUDA}: no CUDA device available; this engine has no CPU fallback")
    from bayes_opt.exception import TargetSpaceEmptyError
    from bayes_opt.util import ensure_rng

    from .acquisition import PosteriorMean
    from .fused import FusedAcquisition

    space = optimizer.space
    if len(space) == 0:
        raise TargetSpaceEmptyError("Cannot recommend a point without registered samples: probe or register a "
                                    "point first.")
    rng = ensure_rng(random_state)
    X = np.asarray(space.params, dtype=np.float64)
    gp = _model_on(optimizer._gp, X, space.target, rng)
    cm = space.constraint
    constraint = None
    if cm is not None:
        Y = np.asarray(space.constraint_values, dtype=np.float64).reshape(X.shape[0], -1)
        models = [_model_on(g, X, Y[:, j], rng) for j, g in enumerate(cm.model)]
        constraint = _Constraint(models, np.atleast_1d(cm.lb), np.atleast_1d(cm.ub))
    acq = FusedAcquisition(B.ACQ_MEAN, gp, constraint)
    if in_sample:
        x = X[int(np.argsort(acq(X), kind="stable")[0])]
    else:
        pm = PosteriorMean()
        own = optimizer.acquisition_function
        pm.b200_candidate_source = getattr(own, "b200_candidate_source", pm.b200_candidate_source)
        pm.b200_refine = getattr(own, "b200_refine", pm.b200_refine)
        x = np.asarray(pm._acq_min(acq, space, random_state=rng, n_random=n_random, n_smart=n_smart),
                       dtype=np.float64)
    mu, sd = gp.predict(x[None, :], return_std=True)
    res = {"target": float(mu[0]), "params": space.array_to_params(x), "std": float(sd[0])}
    if constraint is not None:
        means = np.array([float(g.predict(x[None, :])[0]) for g in constraint.model])
        res["constraint"] = float(means[0]) if means.size == 1 else means
        res["allowed"] = bool(_violation(means, constraint.lb, constraint.ub) == 0.0)
    return res

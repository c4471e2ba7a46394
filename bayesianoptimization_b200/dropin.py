"""``enable(optimizer)``: switch an existing ``bayes_opt.BayesianOptimization`` onto the device engine.
The reference constructs its GP objects privately (R/bayes_opt/bayesian_optimization.py:124-130,
R/bayes_opt/constraint.py:72-81) and offers no constructor injection, so the swap happens on the three
attributes the hot path reads:

  optimizer._gp                       -> B200GaussianProcessRegressor (same kernel / params / RandomState)
  optimizer._space._constraint._model -> list of B200GaussianProcessRegressor
  optimizer._acquisition_function     -> same object, given the device hooks in place (acquisition.accelerate)

``devices=[0, 1, ...]`` additionally shards every acquisition batch and the L-BFGS-B seeds over several
GPUs of the box (SURVEY.md 8e).
"""
from __future__ import annotations

from .gpr import to_b200_gp


def accelerate_acquisition(acq, candidate_source=None, refine=None):
    from .acquisition import accelerate

    return accelerate(acq, candidate_source, refine)


def enable(optimizer, device=0, devices=None, precision="fp64", candidate_source="host_rng", refine="stencil"):
    """Make ``optimizer.suggest()`` / ``maximize()`` / ``predict()`` run on the GPU.

    candidate_source  "host_rng" (default): the random candidates of every suggest() are the reference's own
                      MT19937 stream (parity mode); "device_philox": generated inside the fused kernel
                      (throughput mode, continuous spaces; results are valid but differ from the reference's run).
    refine            "stencil" (default): the L-BFGS-B refinement of every suggest() differentiates the acquisition
                      by the reference's 2-point finite differences, d + 1 rows per evaluation (parity mode);
                      "analytic": it takes the gradient from the device, one row per evaluation (continuous spaces
                      and the built-in acquisitions; one device; iterates differ from the reference's run)."""
    if refine not in ("stencil", "analytic"):
        raise ValueError(f"refine must be 'stencil' or 'analytic', got {refine!r}")
    if refine == "analytic" and devices is not None and len(devices) > 1:
        raise NotImplementedError("refine='analytic' runs on one device: multi-device gradient sharding is not built")
    optimizer._gp = to_b200_gp(optimizer._gp, device, devices, precision)
    cm = getattr(optimizer._space, "_constraint", None)
    if cm is not None:
        cm._model = [to_b200_gp(g, device, devices, precision) for g in cm._model]
    optimizer._acquisition_function = accelerate_acquisition(optimizer._acquisition_function, candidate_source, refine)
    return optimizer

"""bayesianoptimization_b200 - a H100-native GP-surrogate + acquisition engine that drops in
behind ``bayes_opt.BayesianOptimization.suggest()`` and the ``bayes_opt.acquisition`` classes.

Hot path: GP fit -> batched posterior predict -> UCB/EI/PoI/MES/LogEI/LogPoI/NEI/LogNEI (x constraint probability)
or CNEI/LogCNEI -> argmin/top-k, in hand-written sm_90a CUDA behind the C ABI declared in include/b200bo.h.
No CPU fallback: importing the compute classes without the built library raises ImportError.

Two layers:
  * GP seam / C ABI (needs numpy, scipy, sklearn):  B200GaussianProcessRegressor, FusedAcquisition,
    PosteriorPaths, ConstrainedPaths (posterior sample paths, resolved lazily)
  * acquisition seam (a plug-in for the ``bayes_opt`` package, which must be importable):
    UpperConfidenceBound, ExpectedImprovement, ProbabilityOfImprovement, LogExpectedImprovement,
    LogProbabilityOfImprovement, NoisyExpectedImprovement, LogNoisyExpectedImprovement,
    ConstrainedNoisyExpectedImprovement, LogConstrainedNoisyExpectedImprovement, ThompsonSampling,
    ConstrainedThompsonSampling, TrustRegionThompsonSampling, MaxValueEntropySearch, PosteriorMean, ConstantLiar,
    KrigingBeliever, PendingNEI, GPHedge,
    AcquisitionFunction, ConstraintModel, enable(optimizer), suggest_batch(optimizer, q) - resolved lazily on first access.
  * recommend(optimizer): the point a run should report, by the posterior mean (bayes_opt is imported when called).
"""
from . import _lib
from ._build import build_library
from .dropin import accelerate_acquisition, enable
from .fused import FusedAcquisition
from .gpr import B200GaussianProcessRegressor, to_b200_gp
from .recommend import recommend

__version__ = "0.2.0"

_PLUGIN = {
    "AcquisitionFunction": "acquisition", "UpperConfidenceBound": "acquisition",
    "ExpectedImprovement": "acquisition", "ProbabilityOfImprovement": "acquisition",
    "LogExpectedImprovement": "acquisition", "LogProbabilityOfImprovement": "acquisition",
    "ConstantLiar": "acquisition", "GPHedge": "acquisition", "DeviceHooks": "acquisition",
    "ThompsonSampling": "acquisition", "ConstrainedThompsonSampling": "acquisition",
    "MaxValueEntropySearch": "acquisition", "suggest_batch": "acquisition", "KrigingBeliever": "acquisition",
    "NoisyExpectedImprovement": "acquisition", "LogNoisyExpectedImprovement": "acquisition",
    "PendingNEI": "acquisition", "ConstrainedNoisyExpectedImprovement": "acquisition",
    "LogConstrainedNoisyExpectedImprovement": "acquisition", "ConstraintModel": "constraint", "PosteriorPaths": "paths",
    "ConstrainedPaths": "paths", "PosteriorMean": "acquisition", "TrustRegionThompsonSampling": "acquisition",
}


def __getattr__(name):
    mod = _PLUGIN.get(name)
    if mod is None:
        raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
    import importlib

    return getattr(importlib.import_module(f"{__name__}.{mod}"), name)


__all__ = [
    "B200GaussianProcessRegressor", "FusedAcquisition", "enable", "accelerate_acquisition", "to_b200_gp",
    "build_library", "recommend", "__version__", *_PLUGIN,
]

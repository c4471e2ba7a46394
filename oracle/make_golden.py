#!/usr/bin/env python
"""Generate tests/golden/*.npz from the UNMODIFIED reference + the live sklearn/scipy stack.

Run in the build container only (needs the reference checkout):

    PYTHONPATH=oracle/shims:the reference checkout python oracle/make_golden.py

The fixtures pin the oracle (oracle/gp_oracle.py) and, through it, the CUDA path.  Every value
below comes out of reference code paths:
  bayes_opt.BayesianOptimization / TargetSpace.random_sample / acquisition.*._get_acq /
  constraint.ConstraintModel.predict  and  sklearn GaussianProcessRegressor.fit / predict /
  log_marginal_likelihood.
Library versions are recorded inside each file.
"""
import os
import sys
import warnings

import numpy as np
import scipy
import sklearn
from numpy.random import RandomState
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern

import bayes_opt
from bayes_opt import BayesianOptimization, acquisition
from bayes_opt.constraint import ConstraintModel
from bayes_opt.parameter import wrap_kernel
from bayes_opt.target_space import TargetSpace
from scipy.optimize import NonlinearConstraint

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
VERS = dict(
    bayes_opt=bayes_opt.__version__, sklearn=sklearn.__version__, scipy=scipy.__version__,
    numpy=np.__version__,
)


def save(name, **arrs):
    arrs["versions"] = np.array(repr(VERS))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **arrs)
    print("wrote", name, {k: getattr(v, "shape", None) for k, v in arrs.items()})


def unit_space(d):
    return TargetSpace(None, {f"x{i:02d}": (0.0, 1.0) for i in range(d)})


def synth(d, N, seed=0):
    """BASELINE.md section 3.2 inputs."""
    space = unit_space(d)
    X = space.random_sample(N, RandomState(seed))
    y = np.sin(X.sum(1)) + 0.1 * RandomState(seed).randn(N)
    return space, X, y


def fixed_gp(space, ls, nu=2.5):
    return GaussianProcessRegressor(
        kernel=wrap_kernel(Matern(nu=nu, length_scale=ls), space.kernel_transform),
        alpha=1e-6, normalize_y=True, optimizer=None,
    )


def case_readme():
    """C1: README 2-D function, N=25, UCB kappa=2.576 (R/README.md:66-91)."""

    def black_box_function(x, y):
        return -(x**2) - (y - 1) ** 2 + 1

    opt = BayesianOptimization(f=black_box_function, pbounds={"x": (2, 4), "y": (-3, 3)},
                               random_state=1, verbose=0)
    opt.maximize(init_points=5, n_iter=20)
    assert len(opt.space) == 25
    acq = opt._acquisition_function
    rs_before = opt._random_state.get_state()
    acq._fit_gp(opt._gp, opt._space)           # consumes 5 restart draws from opt._random_state
    gp = opt._gp
    xt = opt._space.random_sample(10_000, RandomState(7))
    f = acq._get_acq(gp=gp)
    ys = f(xt)
    mu, sd = gp.predict(xt, return_std=True)
    # single-row calls as L-BFGS-B makes them
    ys_single = np.array([f(xt[i])[0] for i in range(16)])
    # one full end-to-end suggest() from a known RNG state
    opt._random_state.set_state(rs_before)
    sugg = opt.suggest()
    save("c1_readme_ucb",
         X=opt._space.params, y=opt._space.target, bounds=opt._space.bounds,
         length_scale=np.float64(gp.kernel_.length_scale), L=gp.L_, alpha_=gp.alpha_,
         y_mean=gp._y_train_mean, y_std=gp._y_train_std, lml=gp.log_marginal_likelihood_value_,
         xt=xt, mu=mu, sd=sd, acq=ys, acq_single=ys_single, kappa=np.float64(acq.kappa),
         suggestion=np.array([sugg["x"], sugg["y"]]),
         rs_keys=rs_before[1], rs_pos=np.int64(rs_before[2]))


def case_ei(d=8, N=128, M=4096, ls=0.7, name="c2s_ei"):
    space, X, y = synth(d, N)
    gp = fixed_gp(space, ls)
    gp.fit(X, y)
    xt = space.random_sample(M, RandomState(1))
    ei = acquisition.ExpectedImprovement(xi=0.01)
    ei.y_max = y.max()
    ys = ei._get_acq(gp=gp)(xt)
    poi = acquisition.ProbabilityOfImprovement(xi=0.01)
    poi.y_max = y.max()
    ys_poi = poi._get_acq(gp=gp)(xt)
    ucb = acquisition.UpperConfidenceBound(kappa=2.576)
    ys_ucb = ucb._get_acq(gp=gp)(xt)
    mu, sd = gp.predict(xt, return_std=True)
    K = gp.kernel_(X)
    # LML + gradient at a few thetas (sklearn: SK/_gpr.py:541-656)
    thetas = np.log(np.array([0.05, 0.3, 0.7, 2.0, 30.0]))
    lml = np.array([gp.log_marginal_likelihood(np.array([t]), eval_gradient=True) for t in thetas],
                   dtype=object)
    lml_v = np.array([float(v[0]) for v in lml])
    lml_g = np.array([float(v[1][0]) for v in lml])
    idx = np.argsort(ys)[:10]
    # near-duplicate candidates (sigma -> ~0) : the EI/PoI edge semantics
    xe = np.vstack([X[:8], X[:8] + 1e-9, X[8:16] + 1e-4])
    mu_e, sd_e = gp.predict(xe, return_std=True)
    ys_e = ei._get_acq(gp=gp)(xe)
    ysp_e = poi._get_acq(gp=gp)(xe)
    save(name, X=X, y=y, length_scale=np.float64(ls), K=K, L=gp.L_, alpha_=gp.alpha_,
         y_mean=gp._y_train_mean, y_std=gp._y_train_std, xt=xt, mu=mu, sd=sd, acq_ei=ys,
         acq_poi=ys_poi, acq_ucb=ys_ucb, y_max=np.float64(y.max()), xi=np.float64(0.01),
         kappa=np.float64(2.576), argmin=np.int64(ys.argmin()), top10=idx,
         thetas=thetas, lml=lml_v, lml_grad=lml_g,
         xe=xe, mu_e=mu_e, sd_e=sd_e, acq_ei_e=ys_e, acq_poi_e=ysp_e)


def case_kernels():
    """Other supported kernels: Matern nu in {0.5,1.5,inf}, anisotropic Matern-2.5, and sklearn's
    default ConstantKernel*RBF used by R/tests/test_acquisition.py:50-52."""
    space, X, y = synth(4, 48)
    xt = space.random_sample(512, RandomState(1))
    out = dict(X=X, y=y, xt=xt)
    for tag, kern in [
        ("m05", Matern(nu=0.5, length_scale=0.6)),
        ("m15", Matern(nu=1.5, length_scale=0.6)),
        ("rbf", RBF(length_scale=0.6)),
        ("m25aniso", Matern(nu=2.5, length_scale=[0.3, 0.6, 1.2, 2.4])),
        ("crbf", ConstantKernel(2.0) * RBF(length_scale=0.8)),
        ("cm25", ConstantKernel(0.5) * Matern(nu=2.5, length_scale=0.5)),
    ]:
        gp = GaussianProcessRegressor(kernel=kern, alpha=1e-6, normalize_y=True, optimizer=None)
        gp.fit(X, y)
        mu, sd = gp.predict(xt, return_std=True)
        v, g = gp.log_marginal_likelihood(gp.kernel_.theta, eval_gradient=True)
        out.update({f"{tag}_mu": mu, f"{tag}_sd": sd, f"{tag}_L": gp.L_, f"{tag}_alpha_": gp.alpha_,
                    f"{tag}_lml": np.float64(v), f"{tag}_lml_grad": g,
                    f"{tag}_theta": gp.kernel_.theta})
    save("kernels_small", **out)


def case_constrained(d=4, N=96, M=2048):
    """C4-style: target GP + ConstraintModel with 2 constraint GPs, PoI and EI x p_constraint
    (R/bayes_opt/acquisition.py:199-207, R/bayes_opt/constraint.py:153-221)."""
    space, X, y = synth(d, N)
    c = np.column_stack([np.cos(X.sum(1)), np.sin(2 * X.sum(1))])
    lb = np.array([-np.inf, -0.5])
    ub = np.array([0.6, 0.5])
    cm = ConstraintModel(None, lb, ub)
    ls_c = [0.9, 0.5]
    for g, l in zip(cm._model, ls_c):
        g.set_params(kernel=Matern(nu=2.5, length_scale=l), optimizer=None)
    cm.fit(X, c)
    gp = fixed_gp(space, 0.7)
    gp.fit(X, y)
    xt = space.random_sample(M, RandomState(1))
    allowed = cm.allowed(c)
    y_max = y[allowed].max()
    p = cm.predict(xt)
    poi = acquisition.ProbabilityOfImprovement(xi=0.01)
    poi.y_max = y_max
    ys_poi = poi._get_acq(gp=gp, constraint=cm)(xt)
    ei = acquisition.ExpectedImprovement(xi=0.01)
    ei.y_max = y_max
    ys_ei = ei._get_acq(gp=gp, constraint=cm)(xt)
    # two-sided single constraint (J=1 branch, constraint.py:199-209)
    cm1 = ConstraintModel(None, -0.5, 0.5)
    cm1._model[0].set_params(kernel=Matern(nu=2.5, length_scale=0.5), optimizer=None)
    cm1.fit(X, c[:, 1])
    p1 = cm1.predict(xt)
    save("c4s_constrained", X=X, y=y, c=c, lb=lb, ub=ub, ls=np.float64(0.7), ls_c=np.array(ls_c),
         xt=xt, p=p, p1=p1, acq_poi=ys_poi, acq_ei=ys_ei, y_max=np.float64(y_max),
         xi=np.float64(0.01), approx=cm.approx(xt))


def case_fit_full(d=3, N=40):
    """Full hyper-parameter fit (SK/_gpr.py:302-340): theta*, LML*, and how far the optimizer's
    RandomState advanced (5 restart draws of size 1)."""
    space, X, y = synth(d, N)
    rs = RandomState(3)
    gp = GaussianProcessRegressor(
        kernel=wrap_kernel(Matern(nu=2.5), space.kernel_transform), alpha=1e-6, normalize_y=True,
        n_restarts_optimizer=5, random_state=rs,
    )
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gp.fit(X, y)
    nxt = rs.uniform(size=3)   # what the NEXT consumer of the shared RNG would see
    xt = space.random_sample(256, RandomState(1))
    mu, sd = gp.predict(xt, return_std=True)
    save("fit_full_small", X=X, y=y, theta=gp.kernel_.theta, lml=np.float64(gp.log_marginal_likelihood_value_),
         next_uniform=nxt, xt=xt, mu=mu, sd=sd)


def case_constant_liar():
    """ConstantLiar over UCB on the 2-D test space of R/tests/test_acquisition.py:55-57,258-286."""
    space = TargetSpace(lambda x, y: -((x - 3) ** 2) - (y - 1) ** 2, {"x": (1, 4), "y": (0, 3.0)})
    rs = RandomState(0)
    for _ in range(6):
        space.probe(space.random_sample(random_state=rs))
    gp = GaussianProcessRegressor(kernel=Matern(nu=2.5), alpha=1e-6, normalize_y=True,
                                  n_restarts_optimizer=5, random_state=RandomState(0))
    cl = acquisition.ConstantLiar(acquisition.UpperConfidenceBound(kappa=2.576), strategy="max")
    sug = []
    rng = RandomState(5)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for _ in range(4):
            sug.append(cl.suggest(gp=gp, target_space=space, random_state=rng))
    save("constant_liar_small", X=space.params, y=space.target, bounds=space.bounds,
         suggestions=np.array(sug))


def case_mixed_int():
    """Float + int parameters: np.round kernel transform (R/bayes_opt/parameter.py:308-320) and the
    DifferentialEvolution branch of _smart_minimize (R/bayes_opt/acquisition.py:376-412)."""
    def f(x, k):
        return -((x - 2.2) ** 2) - 0.3 * (k - 4) ** 2

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        space = TargetSpace(f, {"x": (0.0, 5.0), "k": (0, 6, int)})
        rs = RandomState(2)
        for _ in range(12):
            space.probe(space.random_sample(random_state=rs))
        gp = GaussianProcessRegressor(
            kernel=wrap_kernel(Matern(nu=2.5, length_scale=1.3), space.kernel_transform), alpha=1e-6,
            normalize_y=True, optimizer=None)
        gp.fit(space.params, space.target)
        ei = acquisition.ExpectedImprovement(xi=0.01)
        ei.y_max = space.target.max()
        xt = np.column_stack([RandomState(5).uniform(0, 5, 600), RandomState(6).uniform(-0.49, 6.49, 600)])
        ys = ei._get_acq(gp=gp)(xt)
        mu, sd = gp.predict(xt, return_std=True)
        rng = RandomState(11)
        sug = ei.suggest(gp, space, n_random=2000, n_smart=4, fit_gp=False, random_state=rng)
    save("mixed_int_small", X=space.params, y=space.target, xt=xt, acq_ei=ys, mu=mu, sd=sd,
         y_max=np.float64(space.target.max()), suggestion=sug, rand_draw=space.random_sample(50, RandomState(9)))


def case_categorical():
    """Float + categorical parameter: the one-hot kernel transform of R/bayes_opt/parameter.py:434-449
    (batch-dependent as written in the reference) through wrap_kernel."""
    def f(x, c):
        return -((x - 2.0) ** 2) + {"a": 0.0, "b": 1.0, "c": -0.5}[c]

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        space = TargetSpace(f, {"x": (0.0, 5.0), "c": ["a", "b", "c"]})
        rs = RandomState(4)
        for _ in range(14):
            space.probe(space.random_sample(random_state=rs))
        gp = GaussianProcessRegressor(
            kernel=wrap_kernel(Matern(nu=2.5, length_scale=1.1), space.kernel_transform), alpha=1e-6,
            normalize_y=True, optimizer=None)
        gp.fit(space.params, space.target)
        xt = space.random_sample(300, RandomState(8))
        xt[:, 0] = RandomState(9).uniform(0, 5, 300)
        xt[:, 1:] = RandomState(10).uniform(0, 1, (300, 3))
        ucb = acquisition.UpperConfidenceBound(kappa=2.0)
        ys = ucb._get_acq(gp=gp)(xt)
        ys_single = np.array([ucb._get_acq(gp=gp)(xt[i])[0] for i in range(12)])
        mu, sd = gp.predict(xt, return_std=True)
    save("categorical_small", X=space.params, y=space.target, xt=xt, acq_ucb=ys, acq_single=ys_single,
         mu=mu, sd=sd, X_transformed=space.kernel_transform(space.params))


def case_gphedge():
    """GPHedge (R/bayes_opt/acquisition.py:1181-1360) over UCB / EI / PoI: four suggest() calls at fixed
    hyper-parameters (fit_gp=False on a GP re-fitted with optimizer=None before every call), so that the
    gains (cumulative posterior means of the previous candidates, :1236-1252), the softmax draw (:1222-1234)
    and the three base suggestions are pinned tightly."""
    def f(x, y):
        return -((x - 3) ** 2) - (y - 1) ** 2 + 0.3 * np.sin(3 * x)

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        space = TargetSpace(f, {"x": (1, 4), "y": (0, 3.0)})
        rs = RandomState(2)
        for _ in range(7):
            space.probe(space.random_sample(random_state=rs))
        X0, y0 = space.params.copy(), space.target.copy()
        gp = GaussianProcessRegressor(
            kernel=wrap_kernel(Matern(nu=2.5, length_scale=0.9), space.kernel_transform), alpha=1e-6,
            normalize_y=True, optimizer=None)
        hedge = acquisition.GPHedge([acquisition.UpperConfidenceBound(kappa=2.0),
                                     acquisition.ExpectedImprovement(xi=0.01),
                                     acquisition.ProbabilityOfImprovement(xi=0.01)])
        rng = RandomState(13)
        sugg, gains, cands = [], [], []
        for _ in range(4):
            gp.fit(space.params, space.target)
            x = hedge.suggest(gp, space, n_random=3000, n_smart=3, fit_gp=False, random_state=rng)
            sugg.append(x)
            gains.append(hedge.gains.copy())
            cands.append(hedge.previous_candidates.copy())
            space.probe(x)
    save("gphedge_small", X=X0, y=y0, suggestions=np.array(sugg), gains=np.array(gains), candidates=np.array(cands),
         next_rand=np.float64(rng.rand()))


CASES = dict(readme=case_readme, ei=case_ei, kernels=case_kernels, constrained=case_constrained,
             fit_full=case_fit_full, constant_liar=case_constant_liar, mixed_int=case_mixed_int,
             categorical=case_categorical, gphedge=case_gphedge)

if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for name in (sys.argv[1:] or list(CASES)):  # no arguments: regenerate everything
        CASES[name]()

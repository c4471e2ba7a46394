"""Numpy restatement of the posterior-mean merit B200BO_ACQ_MEAN (include/b200bo.h, DESIGN.md 4.17), shared by
tests/test_mean_cpu.py (which pins it against sklearn and central differences) and tests/test_gpu_mean.py (which holds
the device to it).

With mu_j the posterior mean of GP j (data units), A1 = sum |alpha_| of the target GP (normalised units):
    viol  = sum_{j=1..J}, in j order, (max(0, lb_j - mu_j) + max(0, mu_j - ub_j))     (an infinite bound adds 0)
    merit = mu_0 where viol = 0, else -T (1 + viol),   T = 2 B + 1,  B = |y_mean| + y_std c A1
    value = -merit
The sums, max (NaN-propagating, np.maximum) and the product are the device's operations in its order, so on the
device's own means the value is reproduced bit for bit.  Gradient: -d mu_0 where viol = 0; T sum_j s_j d mu_j
elsewhere, s_j = -1 below lb_j, +1 above ub_j, 0 within.
"""
import numpy as np


def bound_T(y_mean, y_std, const, alpha_):
    """T = 2 B + 1, B = |y_mean| + y_std c sum |alpha_| >= |mu_0(x)| for every x (0 <= c k <= c)."""
    return 2.0 * (abs(float(y_mean)) + float(y_std) * float(const) * float(np.sum(np.abs(alpha_)))) + 1.0


def violation(cmeans, lb, ub, m):
    """Summed violation of the constraint means cmeans[j] (each (m,)) against [lb[j], ub[j]]."""
    v = np.zeros(m)
    for mu, lo, hi in zip(cmeans, lb, ub):
        a = np.zeros(m) if lo == -np.inf else np.maximum(0.0, lo - np.asarray(mu))
        b = np.zeros(m) if hi == np.inf else np.maximum(0.0, np.asarray(mu) - hi)
        v = v + (a + b)
    return v


def merit(mu0, viol, T):
    return np.where(viol == 0.0, mu0, -T * (1.0 + viol))


def value(mu0, cmeans=(), lb=(), ub=(), T=1.0):
    """The closure value -merit (m,)."""
    mu0 = np.asarray(mu0, dtype=float)
    return -merit(mu0, violation(cmeans, lb, ub, mu0.shape[0]), T)


def value_grad(target, x, constraints=()):
    """(value (m,), gradient (m, d)) over grad_oracle.GradGP models: target, constraints = [(GradGP, lb, ub)]."""
    x = np.asarray(x, dtype=float).reshape(-1, target.d)
    mu0, _, dmu0, _ = target.predict_grad(x)
    T = bound_T(target.y_mean, target.y_std, target.const, target.alpha_)
    cs = [(gp.predict_grad(x), lo, hi) for gp, lo, hi in constraints]
    viol = violation([c[0][0] for c in cs], [c[1] for c in cs], [c[2] for c in cs], len(x))
    val = -merit(mu0, viol, T)
    grad = np.zeros_like(dmu0)
    for (mu, _, dmu, _), lo, hi in cs:
        s = np.where((lo != -np.inf) & (mu < lo), -1.0, np.where((hi != np.inf) & (mu > hi), 1.0, 0.0))
        grad += T * s[:, None] * dmu
    feasible = viol == 0.0
    grad[feasible] = -dmu0[feasible]
    grad[np.isnan(val)] = np.nan
    return val, grad

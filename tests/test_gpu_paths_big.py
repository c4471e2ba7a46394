"""Posterior sample paths (DESIGN.md 4.7) at production sizes on ill-conditioned training sets, against a double-double
reference.

The fixtures (oracle/make_paths_big.py, tests/golden/pathbig_*.npz) hold the true path values, input gradients, sums
sum_i |V_pi| and bounds B_p of four draw sets (q16: QT = 16; q4; q1; q5_L1000: q < QT and L ragged against 64 and 256)
on the four problems of tests/test_gpu_illcond_big.py (N = 1000 .. 4096, cond(K) 6.5e6 .. 1.8e11) and at bench.py's C5
shape (b_m25_c5: N = 8192, d = 32), and the errors of the fp64 referee (tests/thompson_oracle.make_paths and
tests/grad_oracle.path_value_grad: Cholesky solves on the same draws) against them.

Rules, as in the other ill-conditioned suites: the device within max(C_REF * the referee's error, FLOOR) of the truth,
per row class; at the training rows, where a path's error is s_y times the residual of the V solve (apart from a
sigma_n^2 dV term), within 2x the larger of the referee's and the fp64 evaluation floor (TRAIN_REF).  Each
(problem, set) is also held to a pin at about 10x its own error measured on an H100 80GB HBM3 at a 700 W power
limit (in the comments).  Metrics: values |d| / (|f| + s_y); gradients
max_j |d g_j| / (max_j |g_j| + |value| / l_min + 1e-6) per row (DESIGN.md 4.10).  Every case prints the device's and
the referee's errors (pytest -s).
"""
import ctypes as C

import numpy as np
import pytest

from oracle import dd
from oracle import make_acq_big as AB
from oracle import make_illcond as MI
from oracle import make_paths_big as PB

pytestmark = pytest.mark.gpu

PROBLEMS = PB.PROBLEMS
SETS = tuple(PB.SETS)
C_REF = 10.0
# The training rows: within TRAIN_REF x the larger of the referee's error and train_eval_<s>, the error an fp64
# sequential evaluation of c k*^T V leaves with the TRUE V (oracle/make_paths_big.train_eval).  At a training row the
# feature error cancels (r carries the same Phi w), so a path's error there is the residual of K V = r as the evaluator's
# own sum of N terms c k_i V_i forms it; with |V_i| toward 1/alpha that sum's rounding, not the solve, dominates: the
# floor reaches 3e-11 on b_m15_d17 where the device measures 2.6e-11 (DESIGN.md section 2).
TRAIN_REF = 2.0
FLOOR = 1e-13
# Pins per (problem, set) at about 10x the H100 measurement (comments): values over every row, gradients over the 64
# grad rows, and the relative difference of paths.bound() from the truth's B_p (sum |v| carries V's error).
def _table(rows):
    """{(problem, set): pin} from one tuple per problem in the order of make_paths_big.SETS."""
    return {(name, s): v for name, vals in rows.items() for s, v in zip(PB.SETS, vals)}


PIN = _table({  # q16, q4, q1, q5_L1000
    "b_m05_ard": (2.1e-11, 2.4e-11, 1.3e-11, 4.9e-11),  # 2.05e-12 2.32e-12 1.21e-12 4.81e-12
    "b_m15_d17": (1.3e-9, 7.8e-10, 6e-10, 1.2e-9),  # 1.24e-10 7.78e-11 5.95e-11 1.13e-10
    "b_m25_c3": (3.1e-9, 1.4e-9, 1.1e-9, 1.7e-9),  # 3.08e-10 1.39e-10 1.09e-10 1.69e-10
    "b_m25_c5": (3.3e-9, 3.1e-9, 1.5e-9, 2.5e-9),  # 3.27e-10 3.10e-10 1.43e-10 2.50e-10
    "b_rbf_long": (9.8e-6, 7.5e-6, 5.5e-6, 7.2e-6),  # 9.77e-7 7.45e-7 5.44e-7 7.18e-7
})
PIN_GRAD = _table({
    "b_m05_ard": (2.8e-10, 1.2e-10, 2.7e-10, 9.1e-10),  # 2.8e-11 1.2e-11 2.7e-11 9.1e-11
    "b_m15_d17": (8.4e-9, 6.3e-9, 4.8e-9, 6.9e-9),  # 8.4e-10 6.3e-10 4.8e-10 6.9e-10
    "b_m25_c3": (1.1e-8, 5.4e-9, 4.4e-9, 8.6e-9),  # 1.1e-9 5.4e-10 4.4e-10 8.6e-10
    "b_m25_c5": (1.1e-8, 1.3e-8, 1.1e-8, 1.1e-8),  # 1.1e-9 1.3e-9 1.1e-9 1.1e-9
    "b_rbf_long": (9.3e-6, 4.3e-6, 3.5e-6, 4.3e-6),  # 9.3e-7 4.3e-7 3.5e-7 4.3e-7
})
PIN_BOUND = _table({
    "b_m05_ard": (1.3e-11, 1.7e-11, 2e-12, 1e-11),  # 1.3e-12 1.7e-12 2.0e-13 9.9e-13
    "b_m15_d17": (7.9e-9, 4.1e-9, 1e-9, 3.5e-9),  # 7.9e-10 4.1e-10 1.0e-10 3.5e-10
    "b_m25_c3": (1.4e-8, 9.9e-9, 7.6e-9, 8.5e-9),  # 1.4e-9 9.9e-10 7.6e-10 8.5e-10
    "b_m25_c5": (1.1e-8, 1.3e-8, 1.9e-9, 1.4e-8),  # 1.1e-9 1.3e-9 1.9e-10 1.4e-9
    "b_rbf_long": (6.9e-7, 4.5e-7, 5.8e-7, 5.2e-7),  # 6.9e-8 4.5e-8 5.8e-8 5.2e-8
})
CLASSES = {MI.GROUP_NAMES[g]: g for g in range(len(MI.GROUP_NAMES))}
ROW_COPIES = 8  # 8 x 4296 = 34 368 rows > 2 x 132 x 128: every CTA of the persistent grid takes two tiles

_FIX, _GP = {}, {}


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def fixture(name):
    if name not in _FIX:
        _FIX[name] = PB.load(name)
    return _FIX[name]


def _gp(bo, name, precision="fp64"):
    if (name, precision) not in _GP:
        c, r = AB.case(name), fixture(name)
        _GP[name, precision] = bo.B200GaussianProcessRegressor(
            kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True, optimizer=None,
            precision=precision).fit(r["X"], r["y"])
    return _GP[name, precision]


def _paths(bo, name, s, precision="fp64"):
    q, L = PB.SETS[s]
    return _gp(bo, name, precision).sample_paths(q, L, random_state=PB.seed(name, s))


def _verr(v, want, s_y):
    return PB.value_metric(v, want, s_y).max(axis=1)


@pytest.mark.parametrize("s", SETS)
@pytest.mark.parametrize("name", PROBLEMS)
def test_values_against_truth(bo, name, s):
    """Full evaluation per row class; eval_rows bit-equal to the full column for a random path mix, on the rows and
    on eight copies of every candidate; grad_rows' values bit-equal to eval_rows."""
    r = fixture(name)
    q = PB.SETS[s][0]
    rows = PB.rows_of(s, r["group"])
    xt, want, ref = r["xt"][rows], r[f"val_{s}"], r[f"ref_err_{s}"]
    paths = _paths(bo, name, s)
    full = paths(xt)
    dev = _verr(full, want, float(r["y_std"]))
    group = r["group"][rows]
    out = []
    for cname, g in CLASSES.items():
        sel = group == g
        if not np.any(sel):
            continue
        d, f = float(np.max(dev[sel])), float(np.max(ref[sel]))
        out.append(f"{cname} {d:.1e}/{f:.1e}")
        if g == MI.G_TRAIN:
            fl = float(np.max(r[f"train_eval_{s}"]))
            out.append(f"(evaluation floor {fl:.1e})")
            assert d <= max(TRAIN_REF * max(f, fl), FLOOR), (cname, d, f, fl)
        else:
            assert d <= max(C_REF * f, FLOOR), (cname, d, f)
    worst = float(np.max(dev))
    print(f"\n{name} {s} values device/referee: " + " ".join(out) + f" | all {worst:.2e}")
    assert worst <= PIN[name, s]
    rs = np.random.RandomState(PB.seed(name, s))
    pidx = rs.randint(q, size=len(xt))
    ev = paths.eval_rows(xt, pidx)
    assert np.array_equal(ev, full[np.arange(len(xt)), pidx])
    big = np.tile(r["xt"], (ROW_COPIES, 1))
    bidx = rs.randint(q, size=len(big))
    eb = paths.eval_rows(big, bidx)
    gv, _ = paths.grad_rows(big, bidx)
    assert np.array_equal(gv, eb)
    fb = np.tile(paths(r["xt"]), (ROW_COPIES, 1))
    assert np.array_equal(eb, fb[np.arange(len(big)), bidx])


@pytest.mark.parametrize("s", SETS)
@pytest.mark.parametrize("name", PROBLEMS)
def test_gradients_against_truth(bo, name, s):
    """grad_rows on the 64 grad rows, path row mod q: values and gradients against the truth."""
    r = fixture(name)
    q = PB.SETS[s][0]
    gi = r["grad_rows"]
    paths = _paths(bo, name, s)
    val, grad = paths.grad_rows(r["xt"][gi], gi % q)
    assert np.all(np.isfinite(grad))
    ls = dd.ls_vec(AB.case(name))
    dv = float(np.max(PB.value_metric(val, r[f"gval_{s}"], float(r["y_std"]))))
    dg = PB.grad_metric(grad, r[f"grad_{s}"], r[f"gval_{s}"], ls)
    ref = r[f"ref_gerr_{s}"]
    group = r["group"][gi]
    out = []
    for cname, g in CLASSES.items():
        sel = group == g
        if np.any(sel):
            d, f = float(np.max(dg[sel])), float(np.max(ref[sel]))
            out.append(f"{cname} {d:.1e}/{f:.1e}")
            assert d <= max(C_REF * f, FLOOR), (cname, d, f)
    print(f"\n{name} {s} gradients device/referee: " + " ".join(out) + f" | value {dv:.1e}")
    assert float(np.max(dg)) <= PIN_GRAD[name, s]
    assert dv <= PIN[name, s]


@pytest.mark.parametrize("s", SETS)
@pytest.mark.parametrize("name", PROBLEMS)
def test_bound_and_selection(bo, name, s):
    """paths.bound() >= max |f| of the truth and equal to the truth's B_p within its pin; argmin_topk(X, 64) per
    path in the truth's order, two rows trading places only when their true values are within twice the pin of each
    other in the value metric; the selected maximum equals the truth's."""
    r = fixture(name)
    q = PB.SETS[s][0]
    rows = PB.rows_of(s, r["group"])
    want = r[f"val_{s}"]
    paths = _paths(bo, name, s)
    bound = paths.bound()
    assert np.all(bound >= np.max(np.abs(want), axis=0))
    eb = float(np.max(np.abs(bound - r[f"bound_{s}"]) / r[f"bound_{s}"]))
    print(f"\n{name} {s} bound: rel. difference {eb:.1e}, B_p / max|f| "
          f"{float(np.min(r[f'bound_{s}'] / np.max(np.abs(want), axis=0))):.1f}")
    assert eb <= PIN_BOUND[name, s]
    bi, bv, tops = paths.argmin_topk(r["xt"][rows], 64)
    pin, s_y = PIN[name, s], float(r["y_std"])
    for p in range(q):
        f = want[:, p]
        order = np.argsort(-f, kind="stable")
        got = [int(bi[p])] + [int(t) for t in tops[p]]  # the argmin, then the top-k from the first place again
        truth = [int(order[0])] + [int(t) for t in order[:len(tops[p])]]
        for g, w in zip(got, truth):  # a swap only between values within twice the pin, in the value metric
            if g != w:
                assert abs(f[g] - f[w]) <= 2 * pin * (max(abs(f[g]), abs(f[w])) + s_y), (p, g, w, f[g], f[w])
        m = float(np.max(f))
        assert abs(-bv[p] - m) <= 2 * pin * (abs(m) + s_y), (p, -bv[p], m)


def test_philox_source_at_d32_equals_the_host_evaluation(bo):
    """argmin_topk_philox over 2^20 Philox rows on the C5 shape (d = 32, QT = 16) against the host evaluation of the
    same rows (b200bo_philox_rows), bit for bit."""
    from bayesianoptimization_b200 import _lib as B

    name = "b_m25_c5"
    paths = _paths(bo, name, "q16")
    d = fixture(name)["X"].shape[1]
    lo, hi = np.zeros(d), np.ones(d)
    m, k, seed = 1 << 20, 8, 0x5EED_C5
    rows = np.empty((m, d))
    gidx = np.arange(m, dtype=np.int64)
    B.check(B.lib().b200bo_philox_rows(0, seed, B.as_dp(lo), B.as_dp(hi), d, gidx.ctypes.data_as(C.POINTER(C.c_int64)),
                                       m, B.as_dp(rows)))
    bi, bv, bx, ti, tx = paths.argmin_topk_philox(seed, np.stack([lo, hi], axis=1), m, k)
    host = -paths(rows)
    for p in range(paths.n_paths):
        order = np.lexsort((np.arange(m), host[:, p]))
        assert bi[p] == order[0] and bv[p] == host[order[0], p] and np.array_equal(bx[p], rows[order[0]])
        assert list(ti[p]) == list(order[:k]) and np.array_equal(tx[p], rows[order[:k]])


@pytest.mark.parametrize("s", ("q16", "q4"))
def test_fp32_gp_gives_the_fp64_paths(bo, s):
    """Paths are fp64 throughout: on b_m25_c3 a GP with precision="fp32" gives the fp64 GP's paths bit for bit."""
    name = "b_m25_c3"
    r = fixture(name)
    a, b = _paths(bo, name, s), _paths(bo, name, s, "fp32")
    assert np.array_equal(a(r["xt"]), b(r["xt"]))
    assert np.array_equal(a.bound(), b.bound())
    gi = r["grad_rows"]
    q = PB.SETS[s][0]
    ga, gb = a.grad_rows(r["xt"][gi], gi % q), b.grad_rows(r["xt"][gi], gi % q)
    assert np.array_equal(ga[0], gb[0]) and np.array_equal(ga[1], gb[1])

"""Noisy expected improvement (DESIGN.md 4.13) at production sizes and on ill-conditioned noiseless factors, against a
double-double reference.

tests/test_gpu_nei.py holds the device to tests/nei_oracle.py, an fp64 restatement, at N = 300 on well-conditioned
sets.  The fixtures here (oracle/make_nei_big.py, tests/golden/neibig_*.npz) take the ill-conditioned problems of
oracle/make_illcond_big.py (N = 1000 .. 4096, 4296 candidates: 34 tiles) and of make_illcond.py (N = 121 .. 200) with
a WhiteKernel noise term, so that K0 = c k + tau I of the noiseless GP has cond(K0) from 1e6 to 1e11, and hold the
double-double truth of every quantity of the definition and the restatement's fp64 results on the same draws as the
referee.  At these sizes the fantasy solves run over 32 row blocks, nei_term's loop over 4096 rows of the K* column,
and the small-batch gradient's S + 1 lists per row block over 32 row blocks.

The rules are those of tests/test_gpu_illcond.py: device error <= max(C_REF * the referee's error, FLOOR), the 1e-5 bar
wherever the referee meets it, and per-case bars pinned at about 10x the error measured on an H100 80GB HBM3 at a
700 W power limit (in the comments).  Every case prints the device's and the referee's errors (pytest -s).  Metrics:
F and best_s relative to |value| + s_y; sigma0 relative; NEI relative to the batch's largest value (underflowed tails
do not dominate); LogNEI |d| / (1 + |v|) as in tests/test_gpu_logei.py; gradients relative to the largest entry.
"""
import ctypes as C
import warnings

import numpy as np
import pytest

from oracle import make_illcond as MI
from oracle import make_nei_big as NB
from test_gpu_illcond import RTOL
from test_gpu_illcond_ext import _order_ok
from test_gpu_mes import _ENV

pytestmark = pytest.mark.gpu

CASES = sorted(c for c in NB.CASES if "jitter" not in NB.CASES[c])
SMALL_ROWS = 256  # the small-batch path runs on the first rows only
KINDS = ("nei", "lognei")
# The fantasies, best_s, NEI's means and the gradients' mean part come from solves with the explicit inverse factors
# plus one refinement step, held to 10x; sigma0 (and through it every value and gradient) is the residue
# c - sum V^2 of the product with the explicit inverse, held to 100x as sigma is in tests/test_gpu_illcond.py.
C_REF = dict(F=10.0, best=10.0, sd0=100.0, nei=100.0, lognei=100.0, gnei=100.0, glognei=100.0)
FLOOR = dict(F=1e-13, best=1e-13, sd0=1e-11, nei=1e-12, lognei=1e-12, gnei=1e-10, glognei=1e-10)
# Per-case bars at about 10x the measurement (comments), over every metric of the case: LogNEI or sigma0 sets each.
PIN = {
    "b_m05_ard": 3.1e-7,  # 3.1e-8 LogNEI
    "b_m15_d17": 1.1e-6,  # 1.1e-7 LogNEI
    "b_m25_c3": 4.5e-6,  # 4.5e-7 LogNEI gradient
    "b_m25_c3_j27": 4.4e-4,  # 4.4e-5 LogNEI
    "b_rbf_long": 1.3e-4,  # 1.3e-5 LogNEI
    "c_m15_d17": 8.4e-6,  # 8.4e-7 LogNEI gradient
    "c_m25_d3": 5.3e-7,  # 5.3e-8 LogNEI gradient
    "l_m25_d4": 5.3e-7,  # 5.3e-8 LogNEI gradient
}
# Findings (DESIGN.md section 2), held to their pin instead of C_REF x the referee and the 1e-5 bar.  sigma0 is the
# residue c - sum V^2 of the product with the explicit inverse: at cond(K0) ~ 1e11 it is 8x further from the truth than
# the referee's triangular solve (6.5e-6 against 7.7e-7 on b_rbf_long), and LogNEI, whose log sigma0 term carries that
# error whole, misses 1e-5 where the referee meets it; on c_m25_d3 the NEI gradient at the training rows and their
# 1e-7 neighbours follows the value there (8.0e-9 against the referee's 4.0e-11, relative to the largest gradient).
FINDINGS = {("b_rbf_long", "lognei"), ("b_m25_c3_j27", "lognei"), ("c_m25_d3", "gnei")}
PIPES = {"bulk": {"B200BO_SMALL_PATH": "0", "B200BO_PREDICT_PIPE": "bulk"},
         "bulk_nomc": {"B200BO_SMALL_PATH": "0", "B200BO_PREDICT_PIPE": "bulk_nomc"},
         "small": {"B200BO_SMALL_PATH": "1"}}

_FIX, _GP = {}, {}


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def fixture(name):
    if name not in _FIX:
        _FIX[name] = NB.load(name)
    return _FIX[name]


def _gp(bo, name, precision="fp64"):
    if (name, precision) not in _GP:
        noisy, _, _ = NB.gp_cases(name)
        r = fixture(name)
        _GP[name, precision] = bo.B200GaussianProcessRegressor(
            kernel=MI.sk_kernel(noisy), alpha=noisy["alpha"], normalize_y=True, optimizer=None,
            precision=precision).fit(r["X"], r["y"])
    return _GP[name, precision]


def _fant(gp, name, run):
    S, masked = NB.RUNS[run]
    return gp.noiseless_fantasies(S, jitter=NB.CASES[name].get("jitter", NB.JITTER),
                                  incumbent=NB.incumbent_mask(fixture(name)["y"], masked), random_state=NB.SEEDS[S])


def _acq(bo, gp, kind, fant):
    code = bo._lib.ACQ_NEI if kind == "nei" else bo._lib.ACQ_LOGNEI
    return bo.FusedAcquisition(code, gp, xi=NB.XI, fantasies=fant)


def _pin(monkeypatch, env):
    for k in _ENV + ("B200BO_PRUNE",):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _fmt(e):
    return " ".join(f"{k} {v:.1e}" for k, v in e.items())


def _hold(name, dev, ref, dev_all=None):
    """The rule on the rows where the referee forms a value (dev), the pin on every row (dev_all, default dev)."""
    for k in dev:
        if (name, k) in FINDINGS:
            continue
        assert dev[k] <= max(C_REF[k] * ref[k], FLOOR[k]), (k, dev[k], ref[k])
        if ref[k] <= RTOL:
            assert dev[k] <= RTOL, (k, dev[k], ref[k])
    if name in PIN:
        assert max((dev_all or dev).values()) <= PIN[name], (name, dev_all or dev)


TINY = np.finfo(np.float64).tiny


def _err(e):
    """The largest entry; a non-finite one is an infinite error.  The rule compares the device with the referee on the
    rows where the referee forms a value (its LogNEI and LogNEI gradient are the log and ratio of an NEI that
    underflows far out); the pin holds the device on every row."""
    return float(np.max(np.where(np.isfinite(e), e, np.inf), initial=0.0))


def _value_err(kind, got, want):
    """NEI relative to the batch's largest value (absolute when every value underflows); LogNEI |d| / (1 + |v|)."""
    with np.errstate(all="ignore"):
        if kind == "nei":
            e = np.abs(got - want) / max(float(np.max(np.abs(want), initial=0.0)), TINY)
        else:
            e = np.abs(got - want) / (1.0 + np.abs(want))
    return _err(e)


def _grad_err(got, want):
    with np.errstate(all="ignore"):
        e = np.abs(got - want) / max(float(np.max(np.abs(want), initial=0.0)), TINY)
    return _err(e)


# ---------------------------------------------------------------------------------------------------------------
# fantasies and sigma0
# ---------------------------------------------------------------------------------------------------------------
def _f_errors(r, run, F, best):
    ys, rows = float(r["y_std"]), r["F_rows"]
    t, tb = r[f"{run}_F"], r[f"{run}_best"]
    return dict(F=float(np.max(np.abs(F[rows] - t) / (np.abs(t) + ys))),
                best=float(np.max(np.abs(best - tb) / (np.abs(tb) + ys))))


@pytest.mark.parametrize("name", CASES)
def test_fantasies_against_truth(bo, name):
    r = fixture(name)
    gp = _gp(bo, name)
    for run in NB.RUNS:
        fant = _fant(gp, name, run)
        assert fant.F.shape == (len(r["X"]), NB.RUNS[run][0])
        dev = _f_errors(r, run, fant.F, fant.best)
        ref = dict(F=float(np.max(np.abs(r[f"sk_{run}_F"] - r[f"{run}_F"]) / (np.abs(r[f"{run}_F"]) + r["y_std"]))),
                   best=float(np.max(np.abs(r[f"sk_{run}_best"] - r[f"{run}_best"]) /
                                     (np.abs(r[f"{run}_best"]) + r["y_std"]))))
        print(f"\n{name} {run} cond(K0) {float(r['cond0']):.1e}\n  device  {_fmt(dev)}\n  referee {_fmt(ref)}")
        _hold(name, dev, ref)
    # the masked run leaves the rows of largest y out of best_s: its incumbents differ from the all-rows run's
    assert not np.array_equal(r["s4m_best"], r["s4_best"])


@pytest.mark.parametrize("pipe", list(PIPES))
@pytest.mark.parametrize("name", CASES)
def test_sigma0_against_truth(bo, monkeypatch, name, pipe):
    r = fixture(name)
    fant = _fant(_gp(bo, name), name, "s4")
    m = SMALL_ROWS if pipe == "small" else len(r["xt"])
    _pin(monkeypatch, PIPES[pipe])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, sd = fant.gp.predict(r["xt"][:m], return_std=True)
    t = r["sd0"][:m]
    dev = dict(sd0=float(np.max(np.abs(sd - t) / t)))
    ref = dict(sd0=float(np.max(np.abs(r["sk_sd0"][:m] - t) / t)))
    print(f"\n{name} sigma0 {pipe} cond(K0) {float(r['cond0']):.1e}\n  device  {_fmt(dev)}\n  referee {_fmt(ref)}")
    _hold(name, dev, ref)


# ---------------------------------------------------------------------------------------------------------------
# values at every candidate, selection
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pipe", list(PIPES))
@pytest.mark.parametrize("name", CASES)
def test_values_against_truth(bo, monkeypatch, name, pipe):
    r = fixture(name)
    gp = _gp(bo, name)
    m = SMALL_ROWS if pipe == "small" else len(r["xt"])
    _pin(monkeypatch, PIPES[pipe])
    for run in NB.RUNS:
        fant = _fant(gp, name, run)
        for kind in KINDS:
            got = -_acq(bo, gp, kind, fant)(r["xt"][:m])
            want, sk = r[f"{run}_{kind}"][:m], r[f"sk_{run}_{kind}"][:m]
            ok = np.isfinite(sk)
            dev_all = {kind: _value_err(kind, got, want)}
            dev = {kind: _value_err(kind, got[ok], want[ok])}
            ref = {kind: _value_err(kind, sk[ok], want[ok])}
            print(f"\n{name} {pipe} {run}: device {_fmt(dev_all)} | referee {_fmt(ref)} on {ok.sum()} rows")
            _hold(name, dev, ref, dev_all)


@pytest.mark.parametrize("name", CASES)
def test_selection_against_truth_and_pruning(bo, monkeypatch, name):
    from bayesianoptimization_b200 import _lib as B

    r = fixture(name)
    gp = _gp(bo, name)
    x = r["xt"]
    for run in ("s4", "s4m"):
        fant = _fant(gp, name, run)
        for kind in KINDS:
            f = _acq(bo, gp, kind, fant)
            ref = -r[f"{run}_{kind}"]
            out = []
            for prune in ("0", "1"):
                _pin(monkeypatch, {"B200BO_PRUNE": prune})
                i, v, t = f.argmin_topk(x, 10)
                out.append((i, np.float64(v).view(np.int64), list(t)))
                ev, tot = C.c_int64(), C.c_int64()
                B.check(B.lib().b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
                assert ev.value == tot.value == len(x), (prune, ev.value, tot.value)  # NEI is never pruned
            assert out[0] == out[1], out
            tol = 2 * PIN.get(name, RTOL) if kind == "nei" else 2 * PIN.get(name, RTOL) * (1 + np.max(np.abs(ref)))
            _order_ok([int(out[0][0])] + [int(k) for k in out[0][2]], ref, tol)


def test_philox_candidates_match_the_host_evaluation(bo):
    """The Philox candidate source on the C3 handle gives the values and order of the host evaluation of the same rows
    (b200bo_philox_rows), bit for bit."""
    from bayesianoptimization_b200 import _lib as B

    name = "b_m25_c3"
    gp = _gp(bo, name)
    fant = _fant(gp, name, "s4")
    d = fixture(name)["X"].shape[1]
    lo, hi = np.zeros(d), np.ones(d)
    m, k, seed = 8192, 8, 91
    rows = np.empty((m, d))
    gidx = np.arange(m, dtype=np.int64)
    B.check(B.lib().b200bo_philox_rows(0, seed, B.as_dp(lo), B.as_dp(hi), d, gidx.ctypes.data_as(C.POINTER(C.c_int64)),
                                       m, B.as_dp(rows)))
    for kind in KINDS:
        f = _acq(bo, gp, kind, fant)
        idx, val, bx, ti, tx = f.argmin_topk_philox(seed, np.stack([lo, hi], axis=1), m, k)
        host = f(rows)
        order = np.lexsort((np.arange(m), host))
        assert idx == order[0] and val == host[order[0]] and np.array_equal(bx, rows[order[0]])
        assert list(ti) == list(order[:k]) and np.array_equal(tx, rows[order[:k]])
        ih, vh, th = f.argmin_topk(rows, k)
        assert (ih, vh, list(th)) == (idx, val, list(ti))


# ---------------------------------------------------------------------------------------------------------------
# gradients
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_gradient_against_truth(bo, name):
    r = fixture(name)
    gp = _gp(bo, name)
    rows = r["xt"][r["grad_rows"]]
    for run in NB.RUNS:
        fant = _fant(gp, name, run)
        for kind in KINDS:
            val, grad = _acq(bo, gp, kind, fant).value_and_grad(rows)
            want, sk = r[f"{run}_g_{kind}"], r[f"sk_{run}_g_{kind}"]
            ok = np.all(np.isfinite(sk), axis=1)
            dev_all = {f"g{kind}": _grad_err(-grad, want)}
            dev = {f"g{kind}": _grad_err(-grad[ok], want[ok])}
            ref = {f"g{kind}": _grad_err(sk[ok], want[ok])}
            vdev = _value_err(kind, -val, r[f"{run}_{kind}"][r["grad_rows"]])
            print(f"\n{name} grad {run}: device {_fmt(dev_all)} (value {vdev:.1e}) | referee {_fmt(ref)} on "
                  f"{ok.sum()} rows")
            _hold(name, dev, ref, dev_all)
            assert vdev <= max(PIN.get(name, RTOL), FLOOR[kind])


# ---------------------------------------------------------------------------------------------------------------
# tau < alpha, handle precision, refit across a capacity change
# ---------------------------------------------------------------------------------------------------------------
def test_small_jitter_matches_truth_or_names_jitter(bo, monkeypatch):
    """jitter = 2^-27 < alpha on the C3 set: tau = 7.5e-9 and cond(K0) near 1e11.  Either the device holds the rules or
    it raises the LinAlgError that names jitter - and then the referee's fp64 Cholesky of the same K0 must have
    failed too (its values are not finite), or the refusal is a finding."""
    name = "b_m25_c3_j27"
    r = fixture(name)
    gp = _gp(bo, name)
    try:
        fant = _fant(gp, name, "s4")
    except np.linalg.LinAlgError as e:
        assert "jitter" in str(e)
        assert not np.all(np.isfinite(r["sk_s4_nei"])), "the device refuses a K0 that fp64 Cholesky factors"
        return
    assert fant.tau == 2.0 ** -27
    for run in NB.RUNS:
        fant = _fant(gp, name, run)
        dev, ref = _f_errors(r, run, fant.F, fant.best), {}
        for k in ("F", "best"):
            t = r[f"{run}_{k}"]
            ref[k] = float(np.max(np.abs(r[f"sk_{run}_{k}"] - t) / (np.abs(t) + r["y_std"])))
        for kind in KINDS:
            _pin(monkeypatch, PIPES["bulk"])
            ok = np.isfinite(r[f"sk_{run}_{kind}"])
            dev[kind] = _value_err(kind, -_acq(bo, gp, kind, fant)(r["xt"])[ok], r[f"{run}_{kind}"][ok])
            ref[kind] = _value_err(kind, r[f"sk_{run}_{kind}"][ok], r[f"{run}_{kind}"][ok])
        print(f"\n{name} {run} cond(K0) {float(r['cond0']):.1e}\n  device  {_fmt(dev)}\n  referee {_fmt(ref)}")
        _hold(name, dev, ref)


def test_nei_ignores_the_handle_precision(bo):
    """NEI on a noisy GP fitted with precision="fp32" gives the fp64 handle's values bit for bit: the noiseless handle
    is always fp64 and an NEI call evaluates it alone."""
    name = "b_m15_d17"
    r = fixture(name)
    for kind in KINDS:
        a = _acq(bo, _gp(bo, name), kind, _fant(_gp(bo, name), name, "s4"))(r["xt"])
        g32 = _gp(bo, name, "fp32")
        b = _acq(bo, g32, kind, _fant(g32, name, "s4"))(r["xt"])
        assert np.array_equal(a.view(np.int64), b.view(np.int64)), kind


def test_refit_across_a_capacity_change(bo):
    """noiseless_fantasies refits one noiseless handle in place.  Growing the GP through 255, 256 and 257 rows
    re-pitches every N^2 buffer of that handle from np = 256 to np = 384 at the last step; shrinking it back re-pitches
    them again.  At every step the handle is the same object and the values match the restatement."""
    from test_gpu_nei import C0, _fit, _oracle

    import nei_oracle as NO

    rs = np.random.RandomState(12)
    Xc = rs.uniform(size=(1500, 3))
    gp, X, y = _fit(bo, 257, 3)
    first = None
    for n in (255, 256, 257, 256, 255):
        gp.fit(X[:n], y[:n])
        fant = gp.noiseless_fantasies(4, random_state=n)
        first = fant.handle if first is None else first
        assert fant.handle is first, n
        kc, Kc, tau, ym, ys, F, A, best = _oracle(gp, X[:n], 4, n)
        np.testing.assert_allclose(fant.F, ys * F + ym, rtol=1e-8, atol=1e-8 * ys)
        for kind in KINDS:
            Ks = kc(Xc, X[:n])
            want = -NO.nei(Ks, A, best, NO.noiseless_sd(Kc, tau, Ks, C0, ys), 0.01, ym, ys, log=(kind == "lognei"))
            code = bo._lib.ACQ_NEI if kind == "nei" else bo._lib.ACQ_LOGNEI
            got = bo.FusedAcquisition(code, gp, xi=0.01, fantasies=fant)(Xc)
            np.testing.assert_allclose(got, want, rtol=1e-7, atol=1e-10)

"""Constrained noisy expected improvement (DESIGN.md 4.15), alone and with pending points (4.16), at production sizes
and on ill-conditioned noiseless factors, against a double-double reference.

tests/test_gpu_cnei.py and tests/test_gpu_cnei_batch.py hold the device to the fp64 restatements tests/cnei_oracle.py and
tests/cnei_batch_oracle.py.  The fixtures here (oracle/make_cnei_big.py, tests/golden/cneibig_*.npz) take four cases of
oracle/make_nei_big.py (N = 121 .. 4096, cond(K0) to about 1e11) with J = 1, 2, 3 and 7 constraint GPs of mixed
covariance families, noisy and noiseless, and every bound shape, and hold the double-double truth of every GP's
fantasies, the eligibility mask, best_s, CNEI / LogCNEI at every candidate and the input gradients, with the
restatements' fp64 results on the same draws as the referee.  The handles are built as the class builds them: each GP's
noiseless_fantasies from one RandomState in order, the incumbents through b200bo_gp_set_constrained_incumbent.

The rules are tests/test_gpu_nei_big.py's: device error <= max(C_REF * the referee's error, FLOOR) (C_REF_P for the
pending fantasies), the 1e-5 bar wherever the referee meets it, and per-case bars pinned at about 10x the error measured
on an H100 80GB HBM3 at a 700 W power limit (in the comments).  Every case prints the device's and the referee's errors
(pytest -s).  Metrics: F (every GP) and best_s relative to |value| + s_y; CNEI relative to the batch's largest value;
"tail": CNEI relative to its own value over the candidates below 1e-3 of the largest where the referee forms it to 1e-5;
LogCNEI |d| / (1 + |v|); gradients relative to the largest entry.  The eligibility mask must equal the truth's exactly
(the generator keeps every constraint fantasy 1e-6 s_y away from every bound).
"""
import types

import numpy as np
import pytest

from oracle import make_cnei_big as CB
from oracle import make_illcond as MI
from test_gpu_cnei_batch import _closure, _entry
from test_gpu_illcond import RTOL
from test_gpu_illcond_ext import _order_ok
from test_gpu_nei_big import PIPES, SMALL_ROWS, _err, _fmt, _grad_err, _pin, _value_err

import cnei_oracle as CO

pytestmark = pytest.mark.gpu

CASES = list(CB.CASES)
KINDS = ("cnei", "logcnei")
C_REF = dict(F=10.0, best=10.0, cnei=100.0, tail=100.0, logcnei=100.0)
# The pending rows' fantasies come from the explicit-inverse row update, held to 100x as in tests/test_gpu_nei_batch_big.py;
# a pending row may be a sample's incumbent, so best_s is held as they are.
C_REF_P = dict(C_REF, F=100.0, best=100.0)
FLOOR = dict(F=1e-13, best=1e-13, cnei=1e-12, tail=1e-12, logcnei=1e-12, gcnei=1e-10, glogcnei=1e-10)
# Per-case bars at about 10x the measurement (comments), over every metric, run and path of the case.
PIN = {
    "b_m25_c3": 4.7e-5,  # 4.7e-6 LogCNEI gradient, s4f
    "b_m15_d17": 1.0e-5,  # 1.0e-6 CNEI tail, p7
    "b_rbf_long": 1.3e-4,  # 1.3e-5 LogCNEI, p15
    "c_m25_d3": 4.7e-6,  # 4.7e-7 CNEI tail, p15
}
# Findings (DESIGN.md section 2), held to their pin instead of C_REF x the referee and the 1e-5 bar.  best_s is the
# fantasy of one row; on c_m25_d3 the floor's row in s4f (the smallest fantasy over every row) is 3.0e-12 from the
# truth against the referee's 1.9e-13 there, 16x, while F over all rows stays within 2.3x of the referee.
# On b_rbf_long (the target's cond(K0) about 1e11) LogCNEI and its gradient carry the error of sigma0, the residue
# c - sum V^2 of the product with the explicit inverse, whole: test_gpu_nei_big.py's LogNEI finding on the same target.
FINDINGS = {("c_m25_d3", "best"), ("b_rbf_long", "logcnei"), ("b_rbf_long", "glogcnei")}

_FIX, _GPS = {}, {}


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def fixture(name):
    if name not in _FIX:
        _FIX[name] = CB.load(name)
    return _FIX[name]


def _gps(bo, name):
    """The target GP and the J constraint GPs, fitted on the fixture's inputs."""
    if name not in _GPS:
        r = fixture(name)
        ys = [r["y"]] + list(r["Yc"])
        gps = []
        for (noisy, _, _), y in zip(CB.gp_specs(name, r["X"].shape[1]), ys):
            gps.append(bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(noisy), alpha=noisy["alpha"],
                                                       normalize_y=True, optimizer=None).fit(r["X"], y))
        _GPS[name] = gps
    return _GPS[name]


def _con(bo, name, run):
    r = fixture(name)
    lb, ub = (r["lb_f"], r["ub_f"]) if run == "s4f" else (r["lb"], r["ub"])
    return types.SimpleNamespace(model=_gps(bo, name)[1:], lb=lb, ub=ub)


def _fant(bo, name, run):
    """Every GP's fantasies drawn as the class draws them, the incumbents set on the device."""
    r = fixture(name)
    gps = _gps(bo, name)
    S, seed, p = CB.RUNS[run]
    rs = np.random.RandomState(seed)
    kw = dict(pending=r["P"][:p], extra_rows=CB.P_MAX - p) if p else {}
    fants = [g.noiseless_fantasies(S, jitter=CB.JITTER, random_state=rs, **kw) for g in gps]
    con = _con(bo, name, run)
    rc, best = _entry(bo, fants[0], fants[1:], con.lb, con.ub, r["inb"][:len(r["X"]) + p])
    assert rc == bo._lib.OK
    fants[0].best = best
    return fants, con


def _acq(bo, name, kind, fants, con):
    code = bo._lib.ACQ_CNEI if kind == "cnei" else bo._lib.ACQ_LOGCNEI
    return bo.FusedAcquisition(code, _gps(bo, name)[0], con, xi=CB.XI, fantasies=fants[0],
                               constraint_fantasies=fants[1:])


def _tail_err(got, want, sk):
    """CNEI relative to its own value over the candidates below 1e-3 of the largest where the referee is within 1e-5 of
    the truth (further out, fp64 means and sigma0 no longer fix a tail value to 1e-5 on either side); the value 0 of an
    underflowed truth is left out."""
    with np.errstate(all="ignore"):
        ref = np.abs(sk - want) / want
        sel = (want > 0) & (want < 1e-3 * np.max(want)) & (ref <= RTOL)
        return _err(np.abs(got[sel] - want[sel]) / want[sel]), int(sel.sum())


def _hold(name, dev, ref, c_ref=C_REF):
    for k in dev:
        if (name, k) in FINDINGS:
            continue
        assert dev[k] <= max(c_ref.get(k, 100.0) * ref.get(k, 0.0), FLOOR[k]), (k, dev[k], ref.get(k))
        if k in ref and ref[k] <= RTOL:
            assert dev[k] <= RTOL, (k, dev[k], ref[k])
    if name in PIN:
        assert max(dev.values()) <= PIN[name], (name, dev)


# ---------------------------------------------------------------------------------------------------------------
# fantasies, eligibility, incumbents
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_fantasies_eligibility_and_incumbents(bo, name):
    r = fixture(name)
    n = len(r["X"])
    ys = r["y_std"]
    for run in CB.RUNS:
        fants, con = _fant(bo, name, run)
        p = CB.RUNS[run][2]
        rows = np.concatenate([r["F_rows"], np.arange(n, n + p)])
        t, sk = r[f"{run}_F"], r[f"sk_{run}_F"]
        dev = dict(F=max(float(np.max(np.abs(f.F[rows] - t[g]) / (np.abs(t[g]) + ys[g])))
                         for g, f in enumerate(fants)),
                   best=float(np.max(np.abs(fants[0].best - r[f"{run}_best"]) / (np.abs(r[f"{run}_best"]) + ys[0]))))
        ref = dict(F=max(float(np.max(np.abs(sk[g] - t[g]) / (np.abs(t[g]) + ys[g]))) for g in range(len(fants))),
                   best=float(np.max(np.abs(r[f"sk_{run}_best"] - r[f"{run}_best"]) /
                                     (np.abs(r[f"{run}_best"]) + ys[0]))))
        ok = CO.eligible(r["inb"][:n + p], [f.F for f in fants[1:]], con.lb, con.ub)
        print(f"\n{name} {run}: eligible {ok[:n].mean():.2f}, floor {int(r[f'{run}_floor'].sum())} of "
              f"{len(ok[0])}\n  device  {_fmt(dev)}\n  referee {_fmt(ref)}")
        assert np.array_equal(ok, r[f"{run}_ok"]), run
        # best_s is the fantasy of the truth's row (or the floor, the smallest over every row)
        F0 = fants[0].F
        assert np.array_equal(fants[0].best, F0[r[f"{run}_best_row"], np.arange(F0.shape[1])]), run
        _hold(name, dev, ref, C_REF_P if p else C_REF)
    assert r["s4f_floor"].any() and not r["s4f_floor"].all()


# ---------------------------------------------------------------------------------------------------------------
# values on every path, selection
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_values_against_truth(bo, monkeypatch, name):
    r = fixture(name)
    xc = r["xc"]
    for run in CB.RUNS:
        fants, con = _fant(bo, name, run)
        for pipe, env in PIPES.items():
            m = SMALL_ROWS if pipe == "small" else len(xc)
            _pin(monkeypatch, env)
            dev, ref, rows = {}, {}, 0
            for kind in KINDS:
                got = -_acq(bo, name, kind, fants, con)(xc[:m])
                want, sk = r[f"{run}_{kind}"][:m], r[f"sk_{run}_{kind}"][:m]
                fin = np.isfinite(sk)
                dev[kind] = _value_err("nei" if kind == "cnei" else "lognei", got, want)
                ref[kind] = _value_err("nei" if kind == "cnei" else "lognei", sk[fin], want[fin])
                if kind == "cnei":
                    dev["tail"], rows = _tail_err(got, want, sk)
                    ref["tail"], _ = _tail_err(sk, want, sk)
            print(f"\n{name} {pipe} {run}: device {_fmt(dev)} | referee {_fmt(ref)} (tail over {rows} rows)")
            _hold(name, dev, ref)


@pytest.mark.parametrize("name", CASES)
def test_selection_against_truth(bo, monkeypatch, name):
    r = fixture(name)
    xc = r["xc"]
    _pin(monkeypatch, {})
    for run in ("s4", "s4f", "p7"):
        fants, con = _fant(bo, name, run)
        for kind in KINDS:
            want = -r[f"{run}_{kind}"]
            i, _, top = _acq(bo, name, kind, fants, con).argmin_topk(xc, 10)
            tol = 2 * PIN.get(name, RTOL) * (1.0 if kind == "cnei" else 1 + np.max(np.abs(want)))
            _order_ok([int(i)] + [int(k) for k in top], want, tol)


# ---------------------------------------------------------------------------------------------------------------
# gradients
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_gradient_against_truth(bo, name):
    r = fixture(name)
    gi = r["grad_rows"]
    rows = r["xc"][gi]
    for run in CB.GRAD_RUNS:
        fants, con = _fant(bo, name, run)
        dev = {}
        for kind in KINDS:
            val, grad = _acq(bo, name, kind, fants, con).value_and_grad(rows)
            dev[f"g{kind}"] = _grad_err(-grad, r[f"{run}_g_{kind}"])
            v = _value_err("nei" if kind == "cnei" else "lognei", -val, r[f"{run}_{kind}"][gi])
            assert v <= max(PIN.get(name, RTOL), FLOOR[kind]), (kind, v)
        print(f"\n{name} grad {run}: device {_fmt(dev)} (no fp64 referee)")
        for k, e in dev.items():
            if (name, k) not in FINDINGS:
                assert e <= RTOL, (k, e)
        if name in PIN:
            assert max(dev.values()) <= PIN[name], (name, dev)


# ---------------------------------------------------------------------------------------------------------------
# the class path
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log", [False, True])
def test_class_closure_is_the_direct_construction(bo, log):
    """p = 0: the class's own closure (its draws, its in-bounds mask from the parameter bounds) gives the direct
    construction's values bit for bit."""
    name = "b_m15_d17"
    r = fixture(name)
    X = r["X"]
    gps = _gps(bo, name)
    con = _con(bo, name, "s4")
    params = X.copy()
    params[int(np.argmax(r["y"])), 0] = 3.0  # the registered row of largest y outside the bounds, as r["inb"] has it
    box = np.array([[0.0, 1.0]] * X.shape[1])
    S, seed, _ = CB.RUNS["s4"]
    acq, closure, _ = _closure(bo, gps, con, params, None, S, seed, box=box, log=log)
    assert acq.xi == CB.XI
    got, best = closure(r["xc"]), acq.fantasies.best.copy()
    fants, _ = _fant(bo, name, "s4")
    direct = _acq(bo, name, "logcnei" if log else "cnei", fants, con)(r["xc"])
    assert np.array_equal(got.view(np.int64), direct.view(np.int64))
    assert np.array_equal(best, fants[0].best)

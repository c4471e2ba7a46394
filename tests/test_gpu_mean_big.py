"""The posterior-mean merit B200BO_ACQ_MEAN (DESIGN.md 4.17) at production sizes against the double-double reference
of oracle/make_mean_big.py (tests/golden/meanbig_*.npz): N = 901 .. 8192, d = 2 .. 32, target and constraint GPs at
cond(K) up to 1.8e11, A1 = sum |alpha_| up to 1e10 (b_rbf_long), means at a 1e6 offset (o_offset_d2).

  1. mu of every GP on the tile kernel (bit-equal to b200bo_gp_predict, the same bits on an fp32 handle) and on the
     small-batch path forced over every candidate (B200BO_SMALL_PATH=1: 8 and 16 k-chunks, many passes), both held
     to the truth, and the small path to the tile path within SMALL_TILE;
  2. per bound run the merit: the feasibility mask equals the truth's exactly, feasible values are -mu_0 of the
     device bit for bit, infeasible ones are held to T (1 + viol) of the truth, the device's T to the truth's T and to
     the restatement on the handle's alpha_; "inf" is the unconstrained call bit for bit;
  3. selection: argmin and top 64 in the truth's order (swaps only within twice the pin, or between candidates whose
     device values are equal: 1 + viol rounds equal in fp64 - counted and printed); the records are numpy's stable
     order of the device's values on host, device-resident and eight-copy candidates, equal under B200BO_PRUNE=0 / 1
     and every single B200BO_PRUNE_* arm ("never pruned"); the Philox records at m = 2^20 at the C3 and C5 shapes equal
     the host evaluation of b200bo_philox_rows;
  4. the gradient: value_and_grad's values bit-equal to the small path's, gradients held to the truth (per row,
     relative to s_0 = max_j |d mu_0| + y_std_0 / l_min on rows the truth calls feasible and to T max_g s_g over the
     constraint GPs elsewhere); at rows where lb_j or ub_j is the device's own mu_j, viol = 0 and the gradient is
     -d mu_0 bit for bit (the boundary is feasible);
  5. changed handles: MEAN first, then conditioning on illbig's pending rows (1 row on a fork that re-pitches np, then
     8 and 64 in place), the append path (b200bo_gp_append) and NEI fantasies set on the handle: mu stays within the
     pin of the unconditioned truth, T follows the handle's alpha_ (and keeps its bits under believer conditioning,
     which extends alpha_ by an exact 0), fantasies change no bit;
  6. recommend(in_sample=True) with every row of b_m15_d17 / o_offset_d2 registered in the reference's optimizer:
     the truth's best row, the same from stale GPs (device clones) and fitted ones, the optimizer left unchanged.

The rule is that of tests/test_gpu_illcond.py: device error <= max(C * the referee's (sklearn's) error, floor), and
per-problem pins at about 10x the error measured on an H100 80GB HBM3 at a 700 W power limit (comments).  Every case
prints its measured errors next to the pin (pytest -s).
"""
import ctypes as C
import types
import warnings

import numpy as np
import pytest

import grad_oracle as GO
import mean_oracle as MO
from oracle import dd
from oracle import make_illcond as MI
from oracle import make_illcond_big as MB
from oracle import make_mean_big as MM
from test_gpu_illcond import C_SK, FLOOR
from test_gpu_prune_matrix import SINGLE, SWITCHES

pytestmark = pytest.mark.gpu

PROBLEMS = MM.PROBLEMS
CONSTRAINED = tuple(p for p in PROBLEMS if p != "b_m25_c5")
NU = {"m05": 0.5, "m15": 1.5, "m25": 2.5, "rbf": np.inf}
C_GRAD = 10.0
FLOOR_GRAD = 1e-12
# Pins, about 10x the measurement (comments), per problem.  On o_offset_d2 every mean the device forms is the truth
# rounded to fp64 (measured 0); its pins allow two ulps of a mean near 1e6 (2.3e-16 of |mu| + y_std), as 10x of 0
# would bound nothing.
# mu: max over the GPs of |mu - truth| / (|truth| + y_std), tile and small path
PIN_MU = {
    "b_m15_d17": 8.7e-9,  # 8.7e-10 (the RBF constraint GP at cond(K) 1.7e11; sklearn 2.5e-9)
    "b_m25_c3": 5.1e-9,  # 5.1e-10 (the same GP; sklearn 1.6e-9)
    "b_rbf_long": 6.2e-6,  # 6.2e-7 (the target at cond(K) 1.8e11; sklearn 9.9e-7)
    "b_m25_c5": 5.1e-11,  # 5.1e-12
    "o_offset_d2": 2.3e-16,  # 0
}
# the small path against the tile path, the same metric
SMALL_TILE = {
    "b_m15_d17": 3.4e-10,  # 3.4e-11
    "b_m25_c3": 1.2e-9,  # 1.2e-10
    "b_rbf_long": 5.5e-6,  # 5.5e-7
    "b_m25_c5": 9.1e-12,  # 9.1e-13
    "o_offset_d2": 2.3e-16,  # 0
}
# infeasible merits: |v - T (1 + viol)| / (T (1 + viol)) of the truth's T and viol.  On o_offset_d2 it is viol's
# rounding: lb - mu cancels two numbers near 1e6 whose ulp (1.2e-10) T = 2e6 carries.
PIN_MERIT = {
    "b_m15_d17": 9.7e-9,  # 9.7e-10
    "b_m25_c3": 7.3e-9,  # 7.3e-10
    "b_rbf_long": 8.3e-8,  # 8.3e-9 (T's own error: A1 = 1.07e10 from the alpha_ of a cond(K) 1.8e11 factor)
    "o_offset_d2": 5.8e-10,  # 5.8e-11
}
# |T_dev - T| / T
PIN_T = {
    "b_m15_d17": 2.6e-9,  # 2.6e-10
    "b_m25_c3": 2.6e-9,  # 2.6e-10
    "b_rbf_long": 8.3e-8,  # 8.3e-9
    "o_offset_d2": 2.5e-13,  # 2.5e-14
}
# gradient rows (module docstring)
PIN_GRAD = {
    "b_m15_d17": 4.7e-9,  # 4.7e-10
    "b_m25_c3": 4.6e-9,  # 4.6e-10
    "b_rbf_long": 6e-6,  # 6.0e-7
    "b_m25_c5": 5.1e-10,  # 5.1e-11
    "o_offset_d2": 2.3e-9,  # 2.3e-10
}
# mu after conditioning on pending rows, against the unconditioned truth
PIN_COND = {
    "b_m15_d17": 1.1e-11,  # 1.05e-12
    "b_rbf_long": 6.2e-6,  # 6.2e-7
}
T_RESTATED = 1e-14  # the device's A1 and the restatement's sum |alpha_| add in different orders

_FIX, _GP = {}, {}


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(autouse=True)
def _defaults(monkeypatch):
    for k in ("B200BO_SMALL_PATH", "B200BO_PRUNE", "B200BO_CHUNKED", "B200BO_PREDICT_IMPL") + SWITCHES:
        monkeypatch.delenv(k, raising=False)


def fixture(name):
    if name not in _FIX:
        _FIX[name] = MM.load(name)
    return _FIX[name]


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


def _fit(bo, c, X, y, precision="fp64"):
    return bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True, optimizer=None,
                                           precision=precision).fit(X, y)


def _gp(bo, name, g, precision="fp64"):
    if (name, g, precision) not in _GP:
        r = fixture(name)
        c, y = r["spec"][g]
        _GP[name, g, precision] = _fit(bo, c, r["X"], y, precision)
    return _GP[name, g, precision]


def _con(gps, lb, ub):
    return types.SimpleNamespace(model=list(gps), lb=np.asarray(lb, float), ub=np.asarray(ub, float))


def _mean(bo, gp, con=None):
    return bo.FusedAcquisition(bo._lib.ACQ_MEAN, gp, con)


def _acq(bo, name, run=None):
    r = fixture(name)
    if run is None:
        return _mean(bo, _gp(bo, name, 0))
    J = len(r["spec"]) - 1
    return _mean(bo, _gp(bo, name, 0), _con([_gp(bo, name, j + 1) for j in range(J)], r[f"{run}_lb"], r[f"{run}_ub"]))


def _set(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _mu_err(mu, t, ys):
    return float(np.max(np.abs(mu - t) / (np.abs(t) + ys)))


def _check(what, name, e, pins):
    print(f"\n{name} {what}: device {e:.2e} | pin {pins[name]:.1e}")
    assert e <= pins[name], (name, what, e, pins[name])


def _T_dev(v, viol):
    """The device's T, read back from its infeasible values: v = T (1 + viol) rounded once."""
    bad = viol > 0
    t = v[bad] / (1.0 + viol[bad])
    return float(np.median(t))


def _T_alpha(gp, c):
    return MO.bound_T(float(np.ravel(gp._y_train_mean)[0]), float(np.ravel(gp._y_train_std)[0]),
                      float(c.get("const") or 1.0), np.asarray(gp.alpha_, dtype=float))


# ---------------------------------------------------------------------------------------------------------------
# 1. mu on the tile and the small path
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", PROBLEMS)
def test_mu_tile_and_small_path_against_truth(bo, monkeypatch, name):
    r = fixture(name)
    xt = r["xt"]
    worst, small_tile = 0.0, 0.0
    for g in range(len(r["spec"])):
        gp, ys = _gp(bo, name, g), float(r[f"y_std{g}"])
        t = r[f"mu{g}_hi"]
        _set(monkeypatch, {"B200BO_SMALL_PATH": "0"})
        tile = -_mean(bo, gp)(xt)
        assert np.array_equal(tile.view(np.int64), _quiet(gp.predict, xt).view(np.int64)), g
        if g == 0:
            tile32 = -_mean(bo, _gp(bo, name, g, "fp32"))(xt)
            assert np.array_equal(tile32.view(np.int64), tile.view(np.int64)), g
        _set(monkeypatch, {"B200BO_SMALL_PATH": "1"})
        small = -_mean(bo, gp)(xt)
        e_sk = _mu_err(r[f"sk_mu{g}"], t, ys)
        e = max(_mu_err(tile, t, ys), _mu_err(small, t, ys))
        print(f"\n{name} gp{g}: tile {_mu_err(tile, t, ys):.2e} small {_mu_err(small, t, ys):.2e} sklearn {e_sk:.2e}")
        assert e <= max(C_SK["mu"] * e_sk, FLOOR["mu"]), (g, e, e_sk)
        worst = max(worst, e)
        small_tile = max(small_tile, _mu_err(small, tile, ys))
    _check("mu", name, worst, PIN_MU)
    _check("small vs tile", name, small_tile, SMALL_TILE)


# ---------------------------------------------------------------------------------------------------------------
# 2. the merit per bound run
# ---------------------------------------------------------------------------------------------------------------
def _device_view(bo, name, run, xt):
    """The device's values of a run, its own means (b200bo_gp_predict) and its viol restated on them."""
    r = fixture(name)
    J = len(r["spec"]) - 1
    v = _acq(bo, name, run)(xt)
    mus = [_quiet(_gp(bo, name, g).predict, xt) for g in range(J + 1)]
    viol = MO.violation(mus[1:], r[f"{run}_lb"], r[f"{run}_ub"], len(xt))
    return v, mus, viol


@pytest.mark.parametrize("name", CONSTRAINED)
def test_merit_per_run_against_truth(bo, monkeypatch, name):
    r = fixture(name)
    xt, T = r["xt"], float(r["T"])
    _set(monkeypatch, {"B200BO_SMALL_PATH": "0"})
    unc = _acq(bo, name)(xt)
    worst, worst_T = 0.0, 0.0
    for run in MM.RUNS:
        v, mus, viol = _device_view(bo, name, run, xt)
        feas = r[f"{run}_feas"]
        assert np.array_equal(viol == 0, feas), (run, int(np.sum((viol == 0) != feas)))
        assert np.array_equal(v[feas].view(np.int64), (-mus[0][feas]).view(np.int64)), run
        assert np.all(v[~feas] >= T * (1 - 1e-6)) and np.all(v[feas] < 0.5 * T), run
        if run == "inf":
            assert np.array_equal(v.view(np.int64), unc.view(np.int64))
            continue
        want = -r[f"{run}_merit"]
        e = float(np.max(np.abs(v[~feas] - want[~feas]) / want[~feas]))
        T_dev = _T_dev(v, viol)
        T_res = _T_alpha(_gp(bo, name, 0), r["spec"][0][0])
        assert abs(T_dev - T_res) <= T_RESTATED * T_res, (run, T_dev, T_res)
        worst, worst_T = max(worst, e), max(worst_T, abs(T_dev - T) / T)
        print(f"\n{name} {run}: {feas.sum()} of {len(xt)} feasible, infeasible merit {e:.2e}, "
              f"T {abs(T_dev - T) / T:.2e} (T = {T:.3e})")
    _check("merit", name, worst, PIN_MERIT)
    _check("T", name, worst_T, PIN_T)


# ---------------------------------------------------------------------------------------------------------------
# 3. selection
# ---------------------------------------------------------------------------------------------------------------
def _records(f, x, k=64):
    i, v, t = f.argmin_topk(x, k)
    return int(i), np.float64(v).view(np.int64), [int(u) for u in t]


def _dev_records(bo, f, x, k=64):
    import torch

    m = len(x)
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    out = torch.empty(m, dtype=torch.float64, device="cuda")
    sel = torch.empty(2 * (k + 1), dtype=torch.float64, device="cuda")
    bo._lib.check(bo._lib.lib().b200bo_acq_eval_dev(C.byref(f.spec), xd.data_ptr(), m, out.data_ptr(), None, None, k,
                                                    sel.data_ptr(), 0, None))
    torch.cuda.synchronize()
    rec = sel.cpu().numpy().view(np.int64).reshape(-1, 2)
    return out.cpu().numpy(), int(rec[0, 1]), [int(u) for u in rec[1:, 1]]


def _order_against_truth(got, val_t, v_dev, tol):
    """got (the top list) against the truth's values val_t (closure values, smaller first): where the device's order
    differs from the truth's stable order, the two candidates' true values are within tol of each other, or the
    device cannot tell them apart (equal device values).  Returns the number of places of the second kind."""
    want = np.argsort(val_t, kind="stable")[:len(got)]
    rounded = 0
    for g, w in zip(got, want):
        if g == w:
            continue
        if v_dev[g] == v_dev[w] and val_t[g] != val_t[w]:
            rounded += 1
            continue
        assert abs(val_t[g] - val_t[w]) <= tol * max(abs(val_t[g]), abs(val_t[w])), (g, w, val_t[g], val_t[w])
    return rounded


@pytest.mark.parametrize("name", PROBLEMS)
def test_selection_against_truth_and_every_pruning_arm(bo, monkeypatch, name):
    r = fixture(name)
    xt = r["xt"]
    m = len(xt)
    x8 = np.tile(xt, (8, 1))
    runs = MM.RUNS if name in CONSTRAINED else (None,)
    for run in runs:
        f = _acq(bo, name, run)
        v = f(xt)
        rec = _records(f, xt)
        order = list(np.argsort(v, kind="stable")[:64])
        assert rec[0] == int(np.argmin(v)) and rec[1] == v[rec[0]].view(np.int64) and rec[2] == order, run
        val_t = -(r[f"{run}_merit"] if run else r["mu0_hi"])
        nr = _order_against_truth(rec[2], val_t, v, 2 * max(PIN_MERIT.get(name, 0.0), PIN_MU[name]))
        # infeasible candidates whose viol is too small for fp64 to resolve (1 + viol == 1: value T, as at viol = 0+)
        if run:
            feas = r[f"{run}_feas"]
            _, _, viol = _device_view(bo, name, run, xt)
            unres = int(np.sum(~feas & (1.0 + viol == 1.0)))
            print(f"\n{name} {run}: {nr} top-64 places decided by equal device values; {unres} infeasible "
                  f"candidates with 1 + viol == 1 in fp64")
        dv, di, dtop = _dev_records(bo, f, xt)
        assert np.array_equal(dv.view(np.int64), v.view(np.int64)) and di == rec[0] and dtop == rec[2], run
        out = []
        for prune in ("0", "1"):
            for setting in SINGLE if prune == "1" else SINGLE[:1]:
                _set(monkeypatch, {"B200BO_PRUNE": prune, **dict(zip(SWITCHES, setting))})
                out.append(_records(f, x8))
        for k in ("B200BO_PRUNE",) + SWITCHES:
            monkeypatch.delenv(k, raising=False)
        v8 = np.tile(v, 8)
        assert out[0][0] == int(np.argmin(v8)) and out[0][2] == list(np.argsort(v8, kind="stable")[:64]), run
        assert out[0][0] % m == rec[0]
        assert all(o == out[0] for o in out[1:]), run


@pytest.mark.parametrize("name", ["b_m25_c3", "b_m25_c5"])
def test_philox_records_at_c3_and_c5(bo, name):
    r = fixture(name)
    f = _acq(bo, name, "two" if name in CONSTRAINED else None)
    d = r["X"].shape[1]
    lo, hi = np.zeros(d), np.ones(d)
    m, k, seed = 1 << 20, 64, 2024
    bi, bv, bx, ti, tx = f.argmin_topk_philox(seed, np.column_stack([lo, hi]), m, k)
    rows = np.empty((m, d))
    idx = np.arange(m, dtype=np.int64)
    bo._lib.check(bo._lib.lib().b200bo_philox_rows(0, seed, bo._lib.as_dp(lo), bo._lib.as_dp(hi), d,
                                                   idx.ctypes.data_as(C.POINTER(C.c_int64)), m, bo._lib.as_dp(rows)))
    hi_i, hi_v, hi_top = f.argmin_topk(rows, k)
    assert (bi, np.float64(bv).view(np.int64), list(ti)) == (hi_i, np.float64(hi_v).view(np.int64), list(hi_top))
    assert np.array_equal(bx, rows[bi]) and np.array_equal(tx, rows[ti])


# ---------------------------------------------------------------------------------------------------------------
# 4. the gradient
# ---------------------------------------------------------------------------------------------------------------
def _referee_gp(c, X, y):
    return GO.GradGP(X, y, NU[c["kern"]], dd.ls_vec(c), const=float(c.get("const") or 1.0),
                     noise=float(c.get("white") or 0.0), alpha=c["alpha"])


def _grad_err(g, want, scale):
    return np.max(np.abs(g - want), axis=1) / scale


def _scales(r, run, gi):
    """Per gradient row: s_0 where the truth is feasible, T max_{g >= 1} s_g elsewhere, with s_g = max_j |d mu_g| +
    y_std_g / l_min,g (the gradient's natural scale keeps rows near a stationary point of mu_g meaningful)."""
    def s(g):
        return np.max(np.abs(r[f"dmu{g}"]), axis=1) + float(r[f"y_std{g}"]) / float(np.min(dd.ls_vec(r["spec"][g][0])))

    if run is None:
        return s(0)
    sc = float(r["T"]) * np.max([s(j + 1) for j in range(len(r["spec"]) - 1)], axis=0)
    return np.where(r[f"{run}_feas"][gi], s(0), sc)


@pytest.mark.parametrize("name", PROBLEMS)
def test_gradient_against_truth(bo, monkeypatch, name):
    r = fixture(name)
    gi = r["grad_rows"]
    rows = r["xt"][gi]
    refs = [_referee_gp(c, r["X"], y) for c, y in r["spec"]]
    worst = 0.0
    for run in (MM.RUNS if name in CONSTRAINED else (None,)):
        f = _acq(bo, name, run)
        val, grad = f.value_and_grad(rows)
        _set(monkeypatch, {"B200BO_SMALL_PATH": "1"})
        small = f(rows)
        monkeypatch.delenv("B200BO_SMALL_PATH")
        assert np.array_equal(val.view(np.int64), small.view(np.int64)), run
        want = -(r[f"{run}_dmerit"] if run else r["dmu0"])
        if run:
            lb, ub = r[f"{run}_lb"], r[f"{run}_ub"]
            feas_dev = val < 0.5 * float(r["T"])
            assert np.array_equal(feas_dev, r[f"{run}_feas"][gi]), run
            _, sg = MO.value_grad(refs[0], rows, [(g, lo, hi) for g, lo, hi in zip(refs[1:], lb, ub)])
        else:
            _, sg = MO.value_grad(refs[0], rows)
        sc = _scales(r, run, gi)
        e_dev, e_ref = float(np.max(_grad_err(grad, want, sc))), float(np.max(_grad_err(sg, want, sc)))
        print(f"\n{name} grad {run}: device {e_dev:.2e} | referee {e_ref:.2e}")
        assert e_dev <= max(C_GRAD * e_ref, FLOOR_GRAD), (run, e_dev, e_ref)
        worst = max(worst, e_dev)
    _check("gradient", name, worst, PIN_GRAD)


@pytest.mark.parametrize("name", CONSTRAINED)
def test_boundary_rows_are_feasible(bo, monkeypatch, name):
    """lb_j = the device's own mu_j (small path, as value_and_grad computes it) at a row: viol = 0 there, and the
    gradient is the unconstrained one, -d mu_0, bit for bit; so is ub_j = mu_j."""
    r = fixture(name)
    gi = r["grad_rows"]
    rows = r["xt"][gi[::8]]
    J = len(r["spec"]) - 1
    _set(monkeypatch, {"B200BO_SMALL_PATH": "1"})
    mus = [-_mean(bo, _gp(bo, name, j + 1))(rows) for j in range(J)]
    monkeypatch.delenv("B200BO_SMALL_PATH")
    v0, g0 = _acq(bo, name).value_and_grad(rows)
    # the unconstrained gradient these rows are held to is -d mu_0 itself (within the pin of the truth's)
    e = float(np.max(_grad_err(g0, -r["dmu0"][::8], _scales(r, None, gi)[::8])))
    assert e <= PIN_GRAD[name], e
    for j in range(J):
        for side in ("lb", "ub"):
            for i in range(len(rows)):
                lb, ub = np.full(J, -np.inf), np.full(J, np.inf)
                (lb if side == "lb" else ub)[j] = mus[j][i]
                f = _mean(bo, _gp(bo, name, 0), _con([_gp(bo, name, q + 1) for q in range(J)], lb, ub))
                v, g = f.value_and_grad(rows[i:i + 1])
                assert v[0] == v0[i] and np.array_equal(g[0].view(np.int64), g0[i].view(np.int64)), (j, side, i)


# ---------------------------------------------------------------------------------------------------------------
# 5. changed handles
# ---------------------------------------------------------------------------------------------------------------
def _changed_check(bo, name, tgt, cons, run, label, mu_truth=True, prev=None):
    r = fixture(name)
    xt = r["xt"]
    f = _mean(bo, tgt, _con(cons, r[f"{run}_lb"], r[f"{run}_ub"]))
    v = f(xt)
    mu0 = _quiet(tgt.predict, xt)
    viol = MO.violation([_quiet(g.predict, xt) for g in cons], r[f"{run}_lb"], r[f"{run}_ub"], len(xt))
    feas = viol == 0
    assert np.array_equal(v[feas].view(np.int64), (-mu0[feas]).view(np.int64)), label
    T_dev, T_res = _T_dev(v, viol), _T_alpha(tgt, r["spec"][0][0])
    e_T = abs(T_dev - T_res) / T_res
    e_mu = _mu_err(mu0, r["mu0_hi"], float(r["y_std0"]))
    print(f"\n{name} {label}: T {T_dev:.6e} against the restatement on alpha_ {e_T:.1e}; mu against the "
          f"unconditioned truth {e_mu:.2e}" + (f" | pin {PIN_COND[name]:.1e}" if mu_truth else ""))
    assert e_T <= T_RESTATED, (label, T_dev, T_res)
    if prev is not None:
        print(f"{name} {label}: the restated T moved {abs(T_res - prev) / T_res:.1e} since the previous call")
    if mu_truth:
        assert np.array_equal(feas, r[f"{run}_feas"]), label
        assert e_mu <= PIN_COND[name], (label, e_mu, PIN_COND[name])
    return v, T_res


@pytest.mark.parametrize("name", ["b_m15_d17", "b_rbf_long"])
def test_changed_handles(bo, monkeypatch, name):
    _set(monkeypatch, {"B200BO_SMALL_PATH": "0"})
    r = fixture(name)
    J = len(r["spec"]) - 1
    (c0, y0), X = r["spec"][0], r["X"]
    cons = [_gp(bo, name, j + 1) for j in range(J)]
    P = MB.load(name)["P"]
    # believer conditioning: a fork for the first row with room for 63 more (np re-pitched), then in place
    tgt = _fit(bo, c0, X, y0)
    _, T0 = _changed_check(bo, name, tgt, cons, "two", "fitted")
    g = tgt.condition_on_pending(P[:1], extra_rows=63)
    assert g is not tgt
    v0 = _changed_check(bo, name, g, cons, "two", "conditioned on 1 row (fork)", prev=T0)[0]
    for a, b in ((1, 8), (8, 64)):
        assert g.condition_on_pending(P[a:b]) is g
        v = _changed_check(bo, name, g, cons, "two", f"conditioned on {b} rows (in place)", prev=T0)[0]
        # alpha_ = [alpha_; 0] exactly (DESIGN.md 4.11), so A1 and every infeasible value keep their bits
        bad = ~r["two_feas"]
        assert np.array_equal(v[bad].view(np.int64), v0[bad].view(np.int64)), b
    # the append path (b200bo_gp_append through fit's incremental update) with targets off the mean, so that alpha_
    # and A1 move far
    tgt = _fit(bo, c0, X, y0)
    _changed_check(bo, name, tgt, cons, "two", "fitted")
    mu_p = _quiet(tgt.predict, P[:8])
    ys = float(np.std(y0))
    y_new = mu_p + 0.5 * ys * np.where(np.arange(8) % 2 == 0, 1.0, -1.0)
    tgt.fit(np.vstack([X, P[:8]]), np.concatenate([y0, y_new]))
    _, T1 = _changed_check(bo, name, tgt, cons, "two", "appended 8 rows", mu_truth=False, prev=T0)
    assert T1 != T0
    # NEI fantasies on the handle (the noiseless GP is the handle itself at jitter = alpha) change no bit
    tgt = _fit(bo, c0, X, y0)
    f = _mean(bo, tgt, _con(cons, r["two_lb"], r["two_ub"]))
    before = f(r["xt"])
    tgt.noiseless_fantasies(4, jitter=c0["alpha"], random_state=0)
    after = f(r["xt"])
    assert np.array_equal(before.view(np.int64), after.view(np.int64))


# ---------------------------------------------------------------------------------------------------------------
# 6. recommend() on a registered run of production size
# ---------------------------------------------------------------------------------------------------------------
def _same_gp(a, b):
    assert np.array_equal(a.X_train_, b["X"]) and np.array_equal(a._y_raw, b["y"])
    assert np.array_equal(np.asarray(a.alpha_), b["alpha"])


@pytest.mark.parametrize("name", MM.IN_SAMPLE)
def test_recommend_in_sample_is_the_best_truth_merit(bo, ref, name):
    """The reference's optimizer with every row of the problem registered (target and constraint values, the "two"
    bounds) at fixed kernels: recommend(in_sample=True) returns the row of the truth's best merit (swaps as in
    selection), the same on stale GPs (device clones fitted by recommend) and on GPs fitted on the rows (used
    read-only); the optimizer's RandomState and GPs are unchanged."""
    from scipy.optimize import NonlinearConstraint

    r = fixture(name)
    X, spec = r["X"], r["spec"]
    n, d = X.shape
    keys = [f"x{i:02d}" for i in range(d)]

    def never(**kw):
        raise AssertionError("the constraint function is never called: every value is registered")

    con = NonlinearConstraint(never, r["two_lb"], r["two_ub"])
    opt = ref.BayesianOptimization(f=None, pbounds={k: (-1.0, 2.0) for k in keys}, constraint=con, random_state=3,
                                   verbose=0)
    assert list(opt.space.keys) == keys
    (c0, y0), cons = spec[0], spec[1:]
    opt.set_gp_params(kernel=MI.sk_kernel(c0), alpha=c0["alpha"], optimizer=None)
    for m, (c, _) in zip(opt.constraint.model, cons):
        m.set_params(kernel=MI.sk_kernel(c), alpha=c["alpha"], optimizer=None)
    Y = np.column_stack([y for _, y in cons])
    for i in range(n):
        opt.register(params=dict(zip(keys, X[i])), target=float(y0[i]),
                     constraint_value=Y[i] if Y.shape[1] > 1 else float(Y[i, 0]))
    state = opt._random_state.get_state(legacy=False)
    merit = r["two_meritX"]
    best = int(np.argsort(-merit, kind="stable")[0])
    tol = 2 * max(PIN_MERIT[name], PIN_MU[name])

    def row(res):
        x = opt.space.params_to_array(res["params"])
        i = int(np.flatnonzero(np.all(X == x, axis=1))[0])
        assert i == best or abs(merit[i] - merit[best]) <= tol * abs(merit[best]), (i, best, merit[i], merit[best])
        assert res["allowed"] == bool(r["two_feasX"][i])
        return i

    stale = _quiet(bo.recommend, opt, in_sample=True, random_state=0)
    i_stale = row(stale)
    bo.enable(opt)
    opt._gp.fit(X, y0)
    for j, m in enumerate(opt.constraint.model):
        m.fit(X, Y[:, j])
    before = [dict(X=g.X_train_.copy(), y=g._y_raw.copy(), alpha=np.asarray(g.alpha_).copy())
              for g in [opt._gp] + list(opt.constraint.model)]
    fitted = _quiet(bo.recommend, opt, in_sample=True, random_state=0)
    assert row(fitted) == i_stale and fitted["params"] == stale["params"] and fitted["target"] == stale["target"]
    for g, b in zip([opt._gp] + list(opt.constraint.model), before):
        _same_gp(g, b)
    after = opt._random_state.get_state(legacy=False)
    assert np.array_equal(state["state"]["key"], after["state"]["key"]) and state["state"]["pos"] == after["state"]["pos"]
    print(f"\n{name}: recommend picks row {i_stale}, the truth's best {best} (merit {merit[best]:.6e}, "
          f"{'feasible' if r['two_feasX'][best] else 'infeasible'})")
